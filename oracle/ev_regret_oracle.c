/* TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * Plain-C restatement of the two evaluation functions recursive_eval reports besides exploitability:
 * compute_ev / compute_ev2 (subgame_solving.cc:931-982) and compute_immediate_regrets (:984-1050), on the full game tree with
 * uniform initial beliefs.  Written in the reference's operation and summation order and compiled with -ffp-contract=off
 * (recipe: oracle/ev_regret.py), so every result is bit-identical to the reference; the GPU kernels of
 * rebel_b200/csrc/ev_regret_kernels.cuh are pinned against it on the CPU tier.  Strategies are dense [N][H][A] doubles, the
 * reference's TreeStrategy. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  int D, F, A, H, liar;
} evo_game;

static evo_game game_make(int D, int F) {   /* liars_dice.h:55-57 */
  evo_game g;
  g.D = D; g.F = F; g.A = 1 + 2 * D * F; g.H = 1;
  for (int i = 0; i < D; ++i) g.H *= F;
  g.liar = g.A - 1;
  return g;
}
static int num_matches(const evo_game* g, int hand, int face) {   /* liars_dice.h:83-91: the last face is wild */
  int m = 0;
  for (int i = 0; i < g->D; ++i) { int d = hand % g->F; m += (d == face || d == g->F - 1); hand /= g->F; }
  return m;
}

typedef struct { int last_bid, player_id, children_begin, children_end, parent, depth; } evo_node;

/* unroll_tree (tree.h:51-70) of the whole game, BFS order */
static evo_node* unroll_full(const evo_game* g, int* n_out) {
  int cap = 64, n = 0;
  evo_node* t = (evo_node*)malloc(sizeof(evo_node) * cap);
  t[n++] = (evo_node){-1, 0, 0, 0, -1, 0};
  for (int i = 0; i < n; ++i) {
    int lo = t[i].last_bid < 0 ? 0 : t[i].last_bid + 1, hi = t[i].last_bid < 0 ? g->A - 1 : g->A;   /* liars_dice.h:110-115 */
    t[i].children_begin = n;
    t[i].children_end = n + hi - lo;
    for (int a = lo; a < hi; ++a) {
      if (n == cap) { cap *= 2; t = (evo_node*)realloc(t, sizeof(evo_node) * cap); }
      t[n++] = (evo_node){a, 1 - t[i].player_id, 0, 0, i, t[i].depth + 1};
    }
  }
  *n_out = n;
  return t;
}

/* compute_win_probability (:765-789, float truncation at :785) + compute_expected_terminal_values (:80-98) */
static void terminal_values(const evo_game* g, int bet, int inverse, const double* op_reach, double* values) {
  int quantity = 1 + bet / g->F, face = bet % g->F, nb = 2 * g->D + 1;   /* match counts 0 .. total_num_dice */
  double counts[64];
  for (int i = 0; i < nb; ++i) counts[i] = 0.0;
  for (int h = 0; h < g->H; ++h) counts[num_matches(g, h, face)] += op_reach[h];
  for (int i = nb - 1; i-- > 0;) counts[i] += counts[i + 1];
  for (int h = 0; h < g->H; ++h) {
    int left = quantity - num_matches(g, h, face);
    if (left < 0) left = 0;
    float p = (float)counts[left];
    values[h] = p;
  }
  double s = 0.0;
  for (int h = 0; h < g->H; ++h) s += op_reach[h];
  for (int h = 0; h < g->H; ++h) values[h] = values[h] * 2 - s;
  if (inverse) for (int h = 0; h < g->H; ++h) values[h] *= -1.0;
}

typedef struct {
  evo_game g;
  int N;
  evo_node* tree;
  double* reach[2];   /* [N][H] */
  double* values;     /* [N][H] */
} evo_ctx;

#define IDX3(c, n, h, a) ((((size_t)(n)) * (c)->g.H + (h)) * (c)->g.A + (a))
#define IDX2(c, n, h) (((size_t)(n)) * (c)->g.H + (h))

static evo_ctx* ctx_make(int D, int F) {
  evo_ctx* c = (evo_ctx*)calloc(1, sizeof(evo_ctx));
  c->g = game_make(D, F);
  c->tree = unroll_full(&c->g, &c->N);
  c->reach[0] = (double*)calloc((size_t)c->N * c->g.H, sizeof(double));
  c->reach[1] = (double*)calloc((size_t)c->N * c->g.H, sizeof(double));
  c->values = (double*)calloc((size_t)c->N * c->g.H, sizeof(double));
  return c;
}
static void ctx_free(evo_ctx* c) { free(c->tree); free(c->reach[0]); free(c->reach[1]); free(c->values); free(c); }

/* compute_reach_probabilities (:54-78) from get_initial_beliefs (subgame_solving.h:112-117) */
static void compute_reach(evo_ctx* c, const double* strategy, int player, double* reach) {
  const int H = c->g.H;
  for (int h = 0; h < H; ++h) reach[h] = 1.0 / H;
  for (int n = 1; n < c->N; ++n) {
    const evo_node* nd = &c->tree[n];
    if (c->tree[nd->parent].player_id == player)
      for (int h = 0; h < H; ++h) reach[IDX2(c, n, h)] = reach[IDX2(c, nd->parent, h)] * strategy[IDX3(c, nd->parent, h, nd->last_bid)];
    else
      memcpy(reach + IDX2(c, n, 0), reach + IDX2(c, nd->parent, 0), sizeof(double) * H);
  }
}

/* compute_ev (:931-973): sum over hands of player 0's root values under strategy1 against player 1's reach under strategy2 */
static double ev_sum(evo_ctx* c, const double* strategy1, const double* strategy2) {
  const int H = c->g.H;
  compute_reach(c, strategy2, 1, c->reach[1]);
  for (int n = c->N; n-- > 0;) {
    const evo_node* nd = &c->tree[n];
    double* value = c->values + IDX2(c, n, 0);
    if (nd->children_end == nd->children_begin) {
      terminal_values(&c->g, c->tree[nd->parent].last_bid, nd->player_id != 0, c->reach[1] + IDX2(c, n, 0), value);
      continue;
    }
    for (int h = 0; h < H; ++h) value[h] = 0.0;
    for (int ch = nd->children_begin; ch < nd->children_end; ++ch)
      for (int h = 0; h < H; ++h)
        value[h] += nd->player_id == 0 ? strategy1[IDX3(c, n, h, c->tree[ch].last_bid)] * c->values[IDX2(c, ch, h)]
                                       : c->values[IDX2(c, ch, h)];
  }
  double sum = 0;
  for (int h = 0; h < H; ++h) sum += c->values[IDX2(c, 0, h)];
  return sum;
}

/* compute_ev2 (:975-982) */
int evo_ev2(int D, int F, const double* s1, const double* s2, double* out2) {
  evo_ctx* c = ctx_make(D, F);
  out2[0] = ev_sum(c, s1, s2) / c->g.H;
  out2[1] = -ev_sum(c, s2, s1) / c->g.H;
  ctx_free(c);
  return 0;
}

/* compute_immediate_regrets (:984-1050) over n dense strategies.  The regret sums [N][H][A] are accumulated into `sums` (the
 * caller zeroes them), so a list can be passed in pieces; immediate [N][H] (may be NULL) = max over the A actions / total, 0 at
 * leaves.  Returns N. */
int evo_immediate_regrets(int D, int F, const double* strategies, int n, double* sums, int total, double* immediate) {
  evo_ctx* c = ctx_make(D, F);
  const int H = c->g.H, A = c->g.A, N = c->N;
  for (int k = 0; k < n; ++k) {
    const double* st = strategies + (size_t)k * N * H * A;
    compute_reach(c, st, 0, c->reach[0]);
    compute_reach(c, st, 1, c->reach[1]);
    for (int trav = 0; trav < 2; ++trav) {
      for (int z = 0; z < N; ++z)
        if (c->tree[z].last_bid == c->g.liar)
          terminal_values(&c->g, c->tree[c->tree[z].parent].last_bid, c->tree[z].player_id != trav, c->reach[1 - trav] + IDX2(c, z, 0),
                          c->values + IDX2(c, z, 0));
      for (int nn = N; nn-- > 0;) {
        const evo_node* nd = &c->tree[nn];
        if (nd->children_end == nd->children_begin) continue;
        double* value = c->values + IDX2(c, nn, 0);
        for (int h = 0; h < H; ++h) value[h] = 0.0;
        if (nd->player_id == trav) {
          for (int ch = nd->children_begin; ch < nd->children_end; ++ch) {
            const int a = c->tree[ch].last_bid;
            for (int h = 0; h < H; ++h) {
              sums[IDX3(c, nn, h, a)] += c->values[IDX2(c, ch, h)];
              value[h] += c->values[IDX2(c, ch, h)] * st[IDX3(c, nn, h, a)];
            }
          }
          for (int h = 0; h < H; ++h)
            for (int ch = nd->children_begin; ch < nd->children_end; ++ch) sums[IDX3(c, nn, h, c->tree[ch].last_bid)] -= value[h];
        } else {
          for (int ch = nd->children_begin; ch < nd->children_end; ++ch)
            for (int h = 0; h < H; ++h) value[h] += c->values[IDX2(c, ch, h)];
        }
      }
    }
  }
  if (immediate)
    for (int nn = 0; nn < N; ++nn)
      for (int h = 0; h < H; ++h) {
        const double* r = sums + IDX3(c, nn, h, 0);
        double m = r[0];
        for (int a = 1; a < A; ++a) if (m < r[a]) m = r[a];   /* std::max_element: the first maximum */
        immediate[IDX2(c, nn, h)] = c->tree[nn].children_end != c->tree[nn].children_begin ? m / total : 0.0;
      }
  ctx_free(c);
  return N;
}
