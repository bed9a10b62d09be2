/*
 * TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * Plain-C (fp64) restatement of the reference's self-play CFR data-generation path for
 * Liar's Dice (facebookresearch/rebel, csrc/liars_dice).  It is the CPU oracle the CUDA path in
 * rebel_b200/ is checked against.  Only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it; nothing under rebel_b200/ does.
 *
 * Parity status: PINNED.  tests/test_oracle.py checks this file against (a) every known-answer
 * value in the reference's own gtests for this path (tree_test.cc, liars_dice_test.cc,
 * subgame_solving_test.cc thresholds) and (b) outputs of the reference itself compiled from
 * a checkout of the original project (oracle/_ref, see oracle/Makefile + ref_harness.cc) — bit-exact for the zero-net
 * CFR trajectories when both are built with -ffp-contract=off — and against the committed
 * fixtures in tests/golden/ that were generated from oracle/_ref by oracle/make_golden.py.
 * Covered: game, tree, CFR (linear / vanilla / DCFR), fictitious play (linear / optimistic), terminal
 * payoffs, query rows, Net2 forward, best response / exploitability, the RlRunner walk (CFR or FP), the
 * sampled recursive strategies of recursive_eval and the evaluation entry points of rela/pybind.cc
 * (compute_strategy_recursive[_to_leaf], eval_net) — bit-identical to the compiled reference with
 * the zero net (eval_net's float32 mean: 1e-7 relative).
 *
 * Every function cites the reference file:line it follows (paths relative to
 * csrc/liars_dice/ of the original project).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#define ORC_MAX_A 64
#define ORC_MAX_H 1024

/* ------------------------------------------------------------------ game: liars_dice.h:46-155 */
typedef struct {
  int D, F, A, H, liar, wild;
} orc_game;

static int int_pow(int b, int p) { int r = 1; while (p-- > 0) r *= b; return r; }

static orc_game game_make(int D, int F) {
  orc_game g;
  g.D = D; g.F = F;
  g.A = 1 + 2 * D * F;          /* liars_dice.h:55 */
  g.H = int_pow(F, D);          /* :56 */
  g.liar = g.A - 1;             /* :57 */
  g.wild = F - 1;               /* :58 */
  return g;
}
/* liars_dice.h:83-91 */
static int game_num_matches(const orc_game* g, int hand, int face) {
  int m = 0;
  for (int i = 0; i < g->D; ++i) {
    int d = hand % g->F;
    m += (d == face || d == g->wild);
    hand /= g->F;
  }
  return m;
}
/* liars_dice.h:110-115 */
static void game_bid_range(const orc_game* g, int last_bid, int* lo, int* hi) {
  if (last_bid == -1) { *lo = 0; *hi = g->A - 1; } else { *lo = last_bid + 1; *hi = g->A; }
}
static int game_is_terminal(const orc_game* g, int last_bid) { return last_bid == g->liar; }

int orc_num_actions(int D, int F) { return game_make(D, F).A; }
int orc_num_hands(int D, int F) { return game_make(D, F).H; }
int orc_num_matches(int D, int F, int hand, int face) { orc_game g = game_make(D, F); return game_num_matches(&g, hand, face); }
void orc_bid_range(int D, int F, int last_bid, int* lo, int* hi) { orc_game g = game_make(D, F); game_bid_range(&g, last_bid, lo, hi); }
/* liars_dice.h:74-80 */
void orc_unpack_action(int D, int F, int action, int* quantity, int* face) { (void)D; *quantity = 1 + action / F; *face = action % F; }

/* ------------------------------------------------------------------ tree: tree.h:31-74 */
typedef struct {
  int last_bid, player_id, children_begin, children_end, parent, depth;
} orc_node;

/* tree.h:51-70: BFS, nodes at depth==max_depth are left childless. */
static orc_node* tree_unroll(const orc_game* g, int last_bid, int player_id, int max_depth, int* n_out) {
  int cap = 64, n = 0;
  orc_node* t = (orc_node*)malloc(sizeof(orc_node) * cap);
  t[n++] = (orc_node){last_bid, player_id, 0, 0, -1, 0};
  for (int i = 0; i < n && t[i].depth < max_depth; ++i) {
    int lo, hi;
    game_bid_range(g, t[i].last_bid, &lo, &hi);
    t[i].children_begin = n;
    t[i].children_end = n + hi - lo;
    for (int a = lo; a < hi; ++a) {
      if (n == cap) { cap *= 2; t = (orc_node*)realloc(t, sizeof(orc_node) * cap); }
      t[n++] = (orc_node){a, 1 - t[i].player_id, 0, 0, i, t[i].depth + 1};
    }
  }
  *n_out = n;
  return t;
}

int orc_unroll_tree(int D, int F, int last_bid, int player_id, int max_depth, int32_t* out, int cap_nodes) {
  orc_game g = game_make(D, F);
  int n;
  orc_node* t = tree_unroll(&g, last_bid, player_id, max_depth, &n);
  if (n > cap_nodes) { free(t); return -n; }
  for (int i = 0; i < n; ++i) {
    int32_t* r = out + 6 * i;
    r[0] = t[i].last_bid; r[1] = t[i].player_id; r[2] = t[i].children_begin;
    r[3] = t[i].children_end; r[4] = t[i].parent; r[5] = t[i].depth;
  }
  free(t);
  return n;
}

/* ------------------------------------------------------------------ terminal payoffs */
/* subgame_solving.cc:765-789.  Note the float truncation at :785. */
static void win_probability(const orc_game* g, int bet, const double* beliefs, double* values) {
  int quantity = 1 + bet / g->F, face = bet % g->F;
  int nb = 2 * g->D + 1;
  double counts[2 * 16 + 2];
  for (int i = 0; i < nb; ++i) counts[i] = 0.0;
  for (int h = 0; h < g->H; ++h) counts[game_num_matches(g, h, face)] += beliefs[h];
  for (int i = nb - 1; i-- > 0;) counts[i] += counts[i + 1];
  for (int h = 0; h < g->H; ++h) {
    int m = game_num_matches(g, h, face);
    int left = quantity - m; if (left < 0) left = 0;
    float p = (float)counts[left];
    values[h] = p;
  }
}
void orc_win_probability(int D, int F, int bet, const double* beliefs, double* out) {
  orc_game g = game_make(D, F);
  win_probability(&g, bet, beliefs, out);
}
/* subgame_solving.cc:80-98 */
static void expected_terminal_values(const orc_game* g, int last_bid, int inverse, const double* op_reach, double* values) {
  win_probability(g, last_bid, op_reach, values);
  double s = 0.0;
  for (int h = 0; h < g->H; ++h) s += op_reach[h];
  for (int h = 0; h < g->H; ++h) values[h] = values[h] * 2 - s;
  if (inverse) for (int h = 0; h < g->H; ++h) values[h] *= -1.0;
}

/* ------------------------------------------------------------------ query rows */
/* util.h:68-78 with eps = kReachSmoothingEps = 1e-80 (subgame_solving.h:34) */
static void normalize_safe_f(const double* x, int n, double eps, float* out) {
  double s = 0;
  for (int i = 0; i < n; ++i) s += x[i] + eps;
  for (int i = 0; i < n; ++i) out[i] = (float)((x[i] + eps) / s);
}
static void normalize_safe_d(double* x, int n, double eps) {
  double s = 0;
  for (int i = 0; i < n; ++i) s += x[i] + eps;
  for (int i = 0; i < n; ++i) x[i] = (x[i] + eps) / s;
}
/* subgame_solving.cc:100-123 */
static int write_query(const orc_game* g, int traverser, int last_bid, int player_id, const double* r0, const double* r1, float* buf) {
  int k = 0;
  buf[k++] = (float)player_id;
  buf[k++] = (float)traverser;
  for (int a = 0; a < g->A; ++a) buf[k++] = (float)(a == last_bid);
  normalize_safe_f(r0, g->H, 1e-80, buf + k); k += g->H;
  normalize_safe_f(r1, g->H, 1e-80, buf + k); k += g->H;
  return k;
}
int orc_query(int D, int F, int traverser, int last_bid, int player_id, const double* r0, const double* r1, float* out) {
  orc_game g = game_make(D, F);
  return write_query(&g, traverser, last_bid, player_id, r0, r1, out);
}

/* ------------------------------------------------------------------ value net: cfvpy/models.py:64-94 (Net2, fp32) */
typedef struct {
  int Q, hidden, H;
  const float *w1, *b1, *g1, *be1, *w2, *b2, *g2, *be2, *w3, *b3;
  int w3_zero;   /* every output weight is +-0: each output is exactly its bias, whatever the (finite) hidden features */
} orc_net;

static orc_net net_from_flat(const float* w, int Q, int hidden, int H) {
  orc_net n; n.Q = Q; n.hidden = hidden; n.H = H;
  n.w1 = w; w += (size_t)hidden * Q; n.b1 = w; w += hidden; n.g1 = w; w += hidden; n.be1 = w; w += hidden;
  n.w2 = w; w += (size_t)hidden * hidden; n.b2 = w; w += hidden; n.g2 = w; w += hidden; n.be2 = w; w += hidden;
  n.w3 = w; w += (size_t)H * hidden; n.b3 = w;
  n.w3_zero = 1;
  for (size_t i = 0; i < (size_t)H * hidden; ++i) n.w3_zero &= n.w3[i] == 0.0f;
  return n;
}
static void linear_f(const float* x, const float* w, const float* b, int in, int out, float* y) {
  for (int j = 0; j < out; ++j) {
    float acc = b[j];
    const float* wj = w + (size_t)j * in;
    for (int k = 0; k < in; ++k) acc += x[k] * wj[k];
    y[j] = acc;
  }
}
/* LayerNorm(eps=1e-5, affine) followed by erf-GELU (models.py:20-53,97-99) */
static void ln_gelu_f(float* x, const float* g, const float* be, int n) {
  float mean = 0, var = 0;
  for (int i = 0; i < n; ++i) mean += x[i];
  mean /= n;
  for (int i = 0; i < n; ++i) { float d = x[i] - mean; var += d * d; }
  var /= n;
  float rstd = 1.0f / sqrtf(var + 1e-5f);
  for (int i = 0; i < n; ++i) {
    float y = (x[i] - mean) * rstd * g[i] + be[i];
    x[i] = 0.5f * y * (1.0f + erff(y * 0.70710678118654752440f));
  }
}
static void net_forward(const orc_net* n, const float* queries, int rows, float* out) {
  if (n->w3_zero) {   /* acc = b3 + sum of +-0 products == b3 bit for bit: skip the hidden layers (a constant-output net) */
    for (int r = 0; r < rows; ++r) memcpy(out + (size_t)r * n->H, n->b3, sizeof(float) * n->H);
    return;
  }
  float* a = (float*)malloc(sizeof(float) * n->hidden * 2);
  float* b = a + n->hidden;
  for (int r = 0; r < rows; ++r) {
    linear_f(queries + (size_t)r * n->Q, n->w1, n->b1, n->Q, n->hidden, a);
    ln_gelu_f(a, n->g1, n->be1, n->hidden);
    linear_f(a, n->w2, n->b2, n->hidden, n->hidden, b);
    ln_gelu_f(b, n->g2, n->be2, n->hidden);
    linear_f(b, n->w3, n->b3, n->hidden, n->H, out + (size_t)r * n->H);
  }
  free(a);
}
void orc_net2_forward(const float* w, int Q, int hidden, int H, const float* queries, int rows, float* out) {
  orc_net n = net_from_flat(w, Q, hidden, H);
  net_forward(&n, queries, rows, out);
}

/* ------------------------------------------------------------------ CFR solver: subgame_solving.cc:508-715 */
typedef struct {
  orc_game g;
  int N, L, T;
  orc_node* tree;
  int* pleaf; int* term;                  /* subgame_solving.cc:186-201 */
  int num_iters, linear, dcfr; double dcfr_alpha, dcfr_beta, dcfr_gamma;
  int num_steps[2];
  double* beliefs;                        /* [2][H] */
  double *avg, *sum, *last, *regrets;     /* [N][H][A] dense, like TreeStrategy */
  double* reach[2];                       /* [N][H] */
  double* reach_buf;                      /* [N][H] */
  double* values;                         /* traverser_values [N][H] */
  double root_means[2][ORC_MAX_H]; int root_means_set[2];
  float* queries;                         /* [L][Q] */
  float* leaf_values;                     /* [L][H] */
  int has_net; orc_net net; int zero_net;
  void (*on_example)(void* ctx, const float* q, const float* v); void* ex_ctx;
} orc_cfr;

#define IDX3(s, n, h, a) ((((size_t)(n)) * (s)->g.H + (h)) * (s)->g.A + (a))
#define IDX2(s, n, h) (((size_t)(n)) * (s)->g.H + (h))

/* subgame_solving.cc:54-78 */
static void compute_reach(const orc_cfr* s, const double* strategy, const double* init, int player, double* reach) {
  int H = s->g.H;
  for (int n = 0; n < s->N; ++n) {
    if (n == 0) { memcpy(reach, init, sizeof(double) * H); continue; }
    const orc_node* nd = &s->tree[n];
    int actor = s->tree[nd->parent].player_id;
    if (player == actor) {
      for (int h = 0; h < H; ++h)
        reach[IDX2(s, n, h)] = reach[IDX2(s, nd->parent, h)] * strategy[IDX3(s, nd->parent, h, nd->last_bid)];
    } else {
      memcpy(reach + IDX2(s, n, 0), reach + IDX2(s, nd->parent, 0), sizeof(double) * H);
    }
  }
}
/* subgame_solving.cc:718-730 */
static void uniform_strategy(const orc_cfr* s, double* st) {
  memset(st, 0, sizeof(double) * s->N * s->g.H * s->g.A);
  for (int n = 0; n < s->N; ++n) {
    int lo, hi; game_bid_range(&s->g, s->tree[n].last_bid, &lo, &hi);
    int nc = s->tree[n].children_end - s->tree[n].children_begin;
    for (int h = 0; h < s->g.H; ++h)
      for (int a = lo; a < lo + nc; ++a) st[IDX3(s, n, h, a)] = 1. / nc;
  }
}

orc_cfr* orc_cfr_create(int D, int F, int last_bid, int player_id, const double* beliefs, int num_iters, int max_depth,
                        int linear_update, int dcfr, double dcfr_alpha, double dcfr_beta, double dcfr_gamma,
                        const float* net_w, int hidden) {
  orc_cfr* s = (orc_cfr*)calloc(1, sizeof(orc_cfr));
  s->g = game_make(D, F);
  s->tree = tree_unroll(&s->g, last_bid, player_id, max_depth, &s->N);
  int H = s->g.H, A = s->g.A, N = s->N;
  s->pleaf = (int*)malloc(sizeof(int) * N); s->term = (int*)malloc(sizeof(int) * N);
  for (int n = 0; n < N; ++n) {
    int nc = s->tree[n].children_end - s->tree[n].children_begin;
    if (game_is_terminal(&s->g, s->tree[n].last_bid)) s->term[s->T++] = n;
    else if (!nc) s->pleaf[s->L++] = n;
  }
  s->num_iters = num_iters; s->linear = linear_update; s->dcfr = dcfr;
  s->dcfr_alpha = dcfr_alpha; s->dcfr_beta = dcfr_beta; s->dcfr_gamma = dcfr_gamma;
  s->beliefs = (double*)malloc(sizeof(double) * 2 * H);
  memcpy(s->beliefs, beliefs, sizeof(double) * 2 * H);
  size_t dense = (size_t)N * H * A;
  s->avg = (double*)malloc(sizeof(double) * dense); s->sum = (double*)malloc(sizeof(double) * dense);
  s->last = (double*)malloc(sizeof(double) * dense); s->regrets = (double*)calloc(dense, sizeof(double));
  s->reach[0] = (double*)calloc((size_t)N * H, sizeof(double)); s->reach[1] = (double*)calloc((size_t)N * H, sizeof(double));
  s->reach_buf = (double*)calloc((size_t)N * H, sizeof(double)); s->values = (double*)calloc((size_t)N * H, sizeof(double));
  int Q = 2 + A + 2 * H;
  s->queries = (float*)calloc((size_t)(s->L ? s->L : 1) * Q, sizeof(float));
  s->leaf_values = (float*)calloc((size_t)(s->L ? s->L : 1) * H, sizeof(float));
  if (net_w) { s->has_net = 1; s->net = net_from_flat(net_w, Q, hidden, H); } else { s->zero_net = 1; }
  /* ctor, subgame_solving.cc:509-524 */
  uniform_strategy(s, s->avg);
  memcpy(s->last, s->avg, sizeof(double) * dense);
  /* get_uniform_reach_weigted_strategy, subgame_solving.cc:125-149 */
  uniform_strategy(s, s->sum);
  for (int t = 0; t < 2; ++t) {
    compute_reach(s, s->sum /* still uniform on nodes of the other player */, s->beliefs + t * H, t, s->reach_buf);
    for (int n = 0; n < N; ++n) {
      int nc = s->tree[n].children_end - s->tree[n].children_begin;
      if (!nc || s->tree[n].player_id != t) continue;
      int lo, hi; game_bid_range(&s->g, s->tree[n].last_bid, &lo, &hi);
      for (int h = 0; h < H; ++h)
        for (int a = lo; a < hi; ++a) s->sum[IDX3(s, n, h, a)] *= s->reach_buf[IDX2(s, n, h)];
    }
  }
  return s;
}
/* NOTE on the loop above: the reference computes reach for traverser 0 under the fully uniform strategy,
 * scales player-0 rows, then computes reach for traverser 1 from the partially scaled table; player-1
 * reach only reads player-1 rows (compute_reach_probabilities multiplies only where
 * player == last_action_player), which are still uniform at that point.  Same here. */

void orc_cfr_destroy(orc_cfr* s) {
  free(s->tree); free(s->pleaf); free(s->term); free(s->beliefs); free(s->avg); free(s->sum); free(s->last);
  free(s->regrets); free(s->reach[0]); free(s->reach[1]); free(s->reach_buf); free(s->values);
  free(s->queries); free(s->leaf_values); free(s);
}

/* subgame_solving.cc:253-293: leaf queries + net, then terminals */
static void precompute_all_leaf_values(orc_cfr* s, int traverser) {
  int H = s->g.H, Q = 2 + s->g.A + 2 * H;
  if (s->L) {
    for (int r = 0; r < s->L; ++r) {
      int n = s->pleaf[r];
      write_query(&s->g, traverser, s->tree[n].last_bid, s->tree[n].player_id,
                  s->reach[0] + IDX2(s, n, 0), s->reach[1] + IDX2(s, n, 0), s->queries + (size_t)r * Q);
    }
    if (s->has_net) net_forward(&s->net, s->queries, s->L, s->leaf_values);
    else memset(s->leaf_values, 0, sizeof(float) * s->L * H);
    for (int r = 0; r < s->L; ++r) {
      int n = s->pleaf[r];
      double scaler = 0;
      for (int h = 0; h < H; ++h) scaler += s->reach[1 - traverser][IDX2(s, n, h)];
      /* float tensor *= double tensor (subgame_solving.cc:268): computed in double, stored as float */
      for (int h = 0; h < H; ++h) {
        s->leaf_values[(size_t)r * H + h] = (float)((double)s->leaf_values[(size_t)r * H + h] * scaler);
        s->values[IDX2(s, n, h)] = s->leaf_values[(size_t)r * H + h];   /* :273-282 */
      }
    }
  }
  for (int i = 0; i < s->T; ++i) {   /* :285-293 */
    int n = s->term[i];
    int bid = s->tree[s->tree[n].parent].last_bid;
    expected_terminal_values(&s->g, bid, s->tree[n].player_id != traverser,
                             s->reach[1 - traverser] + IDX2(s, n, 0), s->values + IDX2(s, n, 0));
  }
}

/* subgame_solving.cc:538-575 */
static void update_regrets(orc_cfr* s, int traverser) {
  int H = s->g.H;
  compute_reach(s, s->last, s->beliefs, 0, s->reach[0]);
  compute_reach(s, s->last, s->beliefs + H, 1, s->reach[1]);
  precompute_all_leaf_values(s, traverser);
  for (int n = s->N; n-- > 0;) {
    const orc_node* nd = &s->tree[n];
    int nc = nd->children_end - nd->children_begin;
    if (!nc) continue;
    int lo, hi; game_bid_range(&s->g, nd->last_bid, &lo, &hi);
    double* value = s->values + IDX2(s, n, 0);
    for (int h = 0; h < H; ++h) value[h] = 0.0;
    if (nd->player_id == traverser) {
      for (int c = nd->children_begin, a = lo; c < nd->children_end; ++c, ++a) {
        const double* av = s->values + IDX2(s, c, 0);
        for (int h = 0; h < H; ++h) {
          s->regrets[IDX3(s, n, h, a)] += av[h];
          value[h] += av[h] * s->last[IDX3(s, n, h, a)];
        }
      }
      for (int h = 0; h < H; ++h)
        for (int a = lo; a < lo + nc; ++a) s->regrets[IDX3(s, n, h, a)] -= value[h];
    } else {
      for (int c = nd->children_begin; c < nd->children_end; ++c) {
        const double* av = s->values + IDX2(s, c, 0);
        for (int h = 0; h < H; ++h) value[h] += av[h];
      }
    }
  }
}

/* subgame_solving.cc:577-664 */
void orc_cfr_step(orc_cfr* s, int traverser) {
  int H = s->g.H, A = s->g.A;
  update_regrets(s, traverser);
  {
    double alpha = s->linear ? 2. / (s->num_steps[traverser] + 2) : 1. / (s->num_steps[traverser] + 1);
    if (!s->root_means_set[traverser]) { for (int h = 0; h < H; ++h) s->root_means[traverser][h] = 0; s->root_means_set[traverser] = 1; }
    for (int h = 0; h < H; ++h) s->root_means[traverser][h] += (s->values[IDX2(s, 0, h)] - s->root_means[traverser][h]) * alpha;
  }
  double pos = 1, neg = 1, strat = 1;
  {
    double ns = s->num_steps[traverser] + 1;
    if (s->linear) {
      pos = neg = strat = ns / (ns + 1);
    } else if (s->dcfr) {
      pos = s->dcfr_alpha >= 5 ? 1 : pow(ns, s->dcfr_alpha) / (pow(ns, s->dcfr_alpha) + 1.);
      neg = s->dcfr_beta <= -5 ? 0 : pow(ns, s->dcfr_beta) / (pow(ns, s->dcfr_beta) + 1.);
      strat = pow(ns / (ns + 1), s->dcfr_gamma);
    }
  }
  for (int n = 0; n < s->N; ++n) {   /* regret matching :619-634 */
    int nc = s->tree[n].children_end - s->tree[n].children_begin;
    if (!nc || s->tree[n].player_id != traverser) continue;
    int lo, hi; game_bid_range(&s->g, s->tree[n].last_bid, &lo, &hi);
    for (int h = 0; h < H; ++h) {
      double* row = s->last + IDX3(s, n, h, 0);
      for (int a = lo; a < hi; ++a) { double r = s->regrets[IDX3(s, n, h, a)]; row[a] = r > 1e-80 ? r : 1e-80; }
      double sum = 0; for (int a = 0; a < A; ++a) sum += row[a];
      for (int a = 0; a < A; ++a) row[a] = row[a] / sum;
    }
  }
  compute_reach(s, s->last, s->beliefs + traverser * H, traverser, s->reach_buf);   /* :636-638 */
  for (int n = 0; n < s->N; ++n) {   /* :639-661 */
    int nc = s->tree[n].children_end - s->tree[n].children_begin;
    if (!nc || s->tree[n].player_id != traverser) continue;
    int lo, hi; game_bid_range(&s->g, s->tree[n].last_bid, &lo, &hi);
    for (int h = 0; h < H; ++h) {
      for (int a = lo; a < hi; ++a) { double* r = &s->regrets[IDX3(s, n, h, a)]; *r *= (*r > 0 ? pos : neg); }
      for (int a = lo; a < hi; ++a) s->sum[IDX3(s, n, h, a)] *= strat;
      for (int a = lo; a < hi; ++a) s->sum[IDX3(s, n, h, a)] += s->reach_buf[IDX2(s, n, h)] * s->last[IDX3(s, n, h, a)];
      double sm = 0; for (int a = 0; a < A; ++a) sm += s->sum[IDX3(s, n, h, a)];
      for (int a = 0; a < A; ++a) s->avg[IDX3(s, n, h, a)] = s->sum[IDX3(s, n, h, a)] / sm;
    }
  }
  ++s->num_steps[traverser];
}

static void dump(const double* src, double* dst, size_t n) { if (dst) memcpy(dst, src, sizeof(double) * n); }

/* Same signature and semantics as ref_cfr_solve in oracle/ref_harness.cc. */
int orc_cfr_solve(int D, int F, int last_bid, int player_id, const double* beliefs, int num_iters, int max_depth,
                  int linear_update, int dcfr, double dcfr_alpha, double dcfr_beta, double dcfr_gamma,
                  const float* net_w, int hidden, int n_checkpoints, const int32_t* checkpoints,
                  double* regrets, double* last, double* sum, double* avg, double* root_means,
                  float* leaf_values_out, float* queries_out, double* traverser_values_out) {
  orc_cfr* s = orc_cfr_create(D, F, last_bid, player_id, beliefs, num_iters, max_depth, linear_update, dcfr,
                              dcfr_alpha, dcfr_beta, dcfr_gamma, net_w, hidden);
  int H = s->g.H, A = s->g.A, N = s->N, Q = 2 + A + 2 * H;
  size_t dense = (size_t)N * H * A;
  int done = 0;
  for (int c = 0; c < n_checkpoints; ++c) {
    for (; done < checkpoints[c]; ++done) orc_cfr_step(s, done % 2);
    dump(s->regrets, regrets ? regrets + c * dense : 0, dense);
    dump(s->last, last ? last + c * dense : 0, dense);
    dump(s->sum, sum ? sum + c * dense : 0, dense);
    dump(s->avg, avg ? avg + c * dense : 0, dense);
    if (root_means)
      for (int p = 0; p < 2; ++p)
        for (int h = 0; h < H; ++h) root_means[(c * 2 + p) * H + h] = s->root_means_set[p] ? s->root_means[p][h] : 0.0;
    if (leaf_values_out && s->L && done > 0) memcpy(leaf_values_out + (size_t)c * s->L * H, s->leaf_values, sizeof(float) * s->L * H);
    if (queries_out && s->L && done > 0) memcpy(queries_out + (size_t)c * s->L * Q, s->queries, sizeof(float) * s->L * Q);
    if (traverser_values_out) memcpy(traverser_values_out + (size_t)c * N * H, s->values, sizeof(double) * N * H);
  }
  orc_cfr_destroy(s);
  return N;
}

/* ------------------------------------------------------------------ fictitious play: FP, subgame_solving.cc:364-506 */
/* update_sum_strat (:391-421): the traverser's beliefs flow down through its own best-response actions. */
static void fp_update_sum_strat(orc_cfr* s, int node, int traverser, const double* br, const double* beliefs) {
  int H = s->g.H;
  const orc_node* nd = &s->tree[node];
  int nc = nd->children_end - nd->children_begin;
  if (!nc) return;
  if (nd->player_id == traverser) {
    int lo, hi; game_bid_range(&s->g, nd->last_bid, &lo, &hi);
    double* nb = (double*)malloc(sizeof(double) * H);
    for (int c = nd->children_begin, a = lo; c < nd->children_end; ++c, ++a) {
      for (int h = 0; h < H; ++h) {
        s->sum[IDX3(s, node, h, a)] += beliefs[h] * br[IDX3(s, node, h, a)];
        s->last[IDX3(s, node, h, a)] = beliefs[h] * br[IDX3(s, node, h, a)];
      }
      for (int h = 0; h < H; ++h) nb[h] = beliefs[h] * br[IDX3(s, node, h, a)];
      fp_update_sum_strat(s, c, traverser, br, nb);
    }
    free(nb);
  } else {
    for (int c = nd->children_begin; c < nd->children_end; ++c) fp_update_sum_strat(s, c, traverser, br, beliefs);
  }
}

/* FP::step (:423-460) with BRSolver::compute_br (:316-358).  `num_strategies` lives in num_steps[0] + num_steps[1];
 * s->regrets is reused for the best-response strategy. */
static void orc_fp_step(orc_cfr* s, int traverser, int optimistic) {
  int H = s->g.H, A = s->g.A;
  double* br = s->regrets;
  compute_reach(s, s->avg, s->beliefs, 0, s->reach[0]);          /* precompute_reaches (:210-218) */
  compute_reach(s, s->avg, s->beliefs + H, 1, s->reach[1]);
  precompute_all_leaf_values(s, traverser);
  for (int n = s->N; n-- > 0;) {
    const orc_node* nd = &s->tree[n];
    int nc = nd->children_end - nd->children_begin;
    if (!nc) continue;
    int lo, hi; game_bid_range(&s->g, nd->last_bid, &lo, &hi);
    double* value = s->values + IDX2(s, n, 0);
    for (int h = 0; h < H; ++h) value[h] = 0.0;
    if (nd->player_id == traverser) {
      for (int h = 0; h < H; ++h) {
        int best = lo;
        for (int c = nd->children_begin, a = lo; c < nd->children_end; ++c, ++a) {
          double nv = s->values[IDX2(s, c, h)];
          if (c == nd->children_begin || nv > value[h]) { value[h] = nv; best = a; }
        }
        for (int a = 0; a < A; ++a) br[IDX3(s, n, h, a)] = 0.;
        br[IDX3(s, n, h, best)] = 1.0;
      }
    } else {
      for (int c = nd->children_begin; c < nd->children_end; ++c)
        for (int h = 0; h < H; ++h) value[h] += s->values[IDX2(s, c, h)];
    }
  }
  int num_strategies = s->num_steps[0] + s->num_steps[1];
  int num_update = num_strategies / 2 + 1;
  {
    double alpha = s->linear ? 2. / (num_update + 1) : 1. / num_update;
    if (!s->root_means_set[traverser]) { for (int h = 0; h < H; ++h) s->root_means[traverser][h] = 0; s->root_means_set[traverser] = 1; }
    for (int h = 0; h < H; ++h) s->root_means[traverser][h] += (s->values[IDX2(s, 0, h)] - s->root_means[traverser][h]) * alpha;
  }
  fp_update_sum_strat(s, 0, traverser, br, s->beliefs + traverser * H);
  for (int n = 0; n < s->N; ++n) {
    int nc = s->tree[n].children_end - s->tree[n].children_begin;
    if (!nc || s->tree[n].player_id != traverser) continue;
    for (int h = 0; h < H; ++h) {
      double* sm = s->sum + IDX3(s, n, h, 0); double* ls = s->last + IDX3(s, n, h, 0); double* av = s->avg + IDX3(s, n, h, 0);
      if (s->linear) for (int a = 0; a < A; ++a) sm[a] *= (double)(num_update + 1) / (num_update + 2);
      if (optimistic) {            /* util.h:52-63 */
        double t0 = 0, t1 = 0;
        for (int a = 0; a < A; ++a) t0 += sm[a];
        for (int a = 0; a < A; ++a) t1 += ls[a];
        double tot = t0 + t1;
        for (int a = 0; a < A; ++a) av[a] = (sm[a] + ls[a]) / tot;
      } else {                     /* util.h:20-34 */
        double tot = 0;
        for (int a = 0; a < A; ++a) tot += sm[a];
        for (int a = 0; a < A; ++a) av[a] = sm[a] / tot;
      }
    }
  }
  ++s->num_steps[traverser];
}

/* Same signature and semantics as ref_fp_solve in oracle/ref_harness.cc. */
int orc_fp_solve(int D, int F, int last_bid, int player_id, const double* beliefs, int num_iters, int max_depth,
                 int linear_update, int optimistic, const float* net_w, int hidden, int n_checkpoints,
                 const int32_t* checkpoints, double* last, double* sum, double* avg, double* root_means) {
  orc_cfr* s = orc_cfr_create(D, F, last_bid, player_id, beliefs, num_iters, max_depth, linear_update, 0, 0, 0, 0, net_w, hidden);
  int H = s->g.H, A = s->g.A, N = s->N;
  size_t dense = (size_t)N * H * A;
  int done = 0;
  for (int c = 0; c < n_checkpoints; ++c) {
    for (; done < checkpoints[c]; ++done) orc_fp_step(s, done % 2, optimistic);
    dump(s->last, last ? last + c * dense : 0, dense);
    dump(s->sum, sum ? sum + c * dense : 0, dense);
    dump(s->avg, avg ? avg + c * dense : 0, dense);
    if (root_means)
      for (int p = 0; p < 2; ++p)
        for (int h = 0; h < H; ++h) root_means[(c * 2 + p) * H + h] = s->root_means_set[p] ? s->root_means[p][h] : 0.0;
  }
  orc_cfr_destroy(s);
  return N;
}

/* ------------------------------------------------------------------ best response / exploitability */
/* BRSolver::compute_br + compute_exploitability2, subgame_solving.cc:316-358,802-816 (full tree, no net) */
int orc_exploitability(int D, int F, const double* strategy, double* out2) {
  orc_cfr* s = (orc_cfr*)calloc(1, sizeof(orc_cfr));
  s->g = game_make(D, F);
  s->tree = tree_unroll(&s->g, -1, 0, 1000000, &s->N);
  int H = s->g.H, N = s->N;
  s->term = (int*)malloc(sizeof(int) * N); s->pleaf = (int*)malloc(sizeof(int));
  for (int n = 0; n < N; ++n) if (game_is_terminal(&s->g, s->tree[n].last_bid)) s->term[s->T++] = n;
  s->reach[0] = (double*)calloc((size_t)N * H, sizeof(double)); s->reach[1] = (double*)calloc((size_t)N * H, sizeof(double));
  s->values = (double*)calloc((size_t)N * H, sizeof(double));
  double* beliefs = (double*)malloc(sizeof(double) * 2 * H);
  for (int i = 0; i < 2 * H; ++i) beliefs[i] = 1. / H;
  for (int trav = 0; trav < 2; ++trav) {
    compute_reach(s, strategy, beliefs, 0, s->reach[0]);
    compute_reach(s, strategy, beliefs + H, 1, s->reach[1]);
    for (int i = 0; i < s->T; ++i) {
      int n = s->term[i];
      expected_terminal_values(&s->g, s->tree[s->tree[n].parent].last_bid, s->tree[n].player_id != trav,
                               s->reach[1 - trav] + IDX2(s, n, 0), s->values + IDX2(s, n, 0));
    }
    for (int n = N; n-- > 0;) {
      const orc_node* nd = &s->tree[n];
      if (nd->children_end == nd->children_begin) continue;
      double* value = s->values + IDX2(s, n, 0);
      for (int h = 0; h < H; ++h) value[h] = 0.0;
      if (nd->player_id == trav) {
        for (int c = nd->children_begin; c < nd->children_end; ++c)
          for (int h = 0; h < H; ++h) {
            double nv = s->values[IDX2(s, c, h)];
            if (c == nd->children_begin || nv > value[h]) value[h] = nv;   /* first child wins ties :336-337 */
          }
      } else {
        for (int c = nd->children_begin; c < nd->children_end; ++c)
          for (int h = 0; h < H; ++h) value[h] += s->values[IDX2(s, c, h)];
      }
    }
    double sum = 0; for (int h = 0; h < H; ++h) sum += s->values[IDX2(s, 0, h)];
    out2[trav] = sum / H;
  }
  free(beliefs); free(s->tree); free(s->term); free(s->pleaf); free(s->reach[0]); free(s->reach[1]); free(s->values); free(s);
  return 0;
}

/* ------------------------------------------------------------------ RNG: std::mt19937 + libstdc++ 13 distributions */
typedef struct { uint32_t mt[624]; int idx; } orc_mt;
static void mt_seed(orc_mt* m, uint32_t seed) {
  m->mt[0] = seed;
  for (int i = 1; i < 624; ++i) m->mt[i] = 1812433253u * (m->mt[i - 1] ^ (m->mt[i - 1] >> 30)) + (uint32_t)i;
  m->idx = 624;
}
static uint32_t mt_next(orc_mt* m) {
  if (m->idx >= 624) {
    for (int i = 0; i < 624; ++i) {
      uint32_t y = (m->mt[i] & 0x80000000u) | (m->mt[(i + 1) % 624] & 0x7fffffffu);
      m->mt[i] = m->mt[(i + 397) % 624] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
    }
    m->idx = 0;
  }
  uint32_t y = m->mt[m->idx++];
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}
/* std::uniform_int_distribution<int>(a,b) on a 32-bit URBG: Lemire "nearly divisionless"
 * (libstdc++ bits/uniform_int_dist.h _S_nd, used when the generator range is exactly 2^32-1). */
static int uniform_int(orc_mt* m, int a, int b) {
  uint32_t urange = (uint32_t)b - (uint32_t)a;
  if (urange == 0xffffffffu) return (int)(mt_next(m) + (uint32_t)a);
  uint32_t range = urange + 1;
  uint64_t product = (uint64_t)mt_next(m) * (uint64_t)range;
  uint32_t low = (uint32_t)product;
  if (low < range) {
    uint32_t threshold = (uint32_t)(-range) % range;
    while (low < threshold) { product = (uint64_t)mt_next(m) * (uint64_t)range; low = (uint32_t)product; }
  }
  return (int)((uint32_t)(product >> 32) + (uint32_t)a);
}
/* std::generate_canonical<float,24> with a 32-bit generator: one draw */
static float canonical_f(orc_mt* m) {
  float sum = (float)mt_next(m) * 1.0f;
  float r = sum / 4294967296.0f;
  if (r >= 1.0f) r = nextafterf(1.0f, 0.0f);
  return r;
}
/* std::generate_canonical<double,53>: two draws */
static double canonical_d(orc_mt* m) {
  double sum = (double)mt_next(m);
  sum += (double)mt_next(m) * 4294967296.0;
  double r = sum / 18446744073709551616.0;
  if (r >= 1.0) r = nextafter(1.0, 0.0);
  return r;
}
/* std::discrete_distribution<int>(w, w+n): normalise, partial sums, last cp forced to 1, lower_bound */
static int discrete(orc_mt* m, const double* w, int n) {
  if (n < 2) return 0;
  double sum = 0; for (int i = 0; i < n; ++i) sum += w[i];
  double cp[ORC_MAX_H > ORC_MAX_A ? ORC_MAX_H : ORC_MAX_A];
  double acc = 0;
  for (int i = 0; i < n; ++i) { acc += w[i] / sum; cp[i] = acc; }
  cp[n - 1] = 1.0;
  double p = canonical_d(m);
  int lo = 0, hi = n;
  while (lo < hi) { int mid = (lo + hi) / 2; if (cp[mid] < p) lo = mid + 1; else hi = mid; }
  return lo;
}

void orc_rng_probe(uint32_t seed, int n, int32_t* ints, float* floats, int32_t* disc) {
  orc_mt m; mt_seed(&m, seed);
  double w[5] = {0.1, 0.0, 0.4, 0.3, 0.2};
  for (int i = 0; i < n; ++i) { ints[i] = uniform_int(&m, 3, 3 + i % 11); floats[i] = canonical_f(&m); disc[i] = discrete(&m, w, 5); }
}

/* ------------------------------------------------------------------ self-play walk: recursive_solving.cc:160-246 */
typedef struct { float* q; float* v; int n, cap, Q, H; } ex_sink;
static void sink_add(ex_sink* k, const float* q, const float* v) {
  if (k->n < k->cap) { memcpy(k->q + (size_t)k->n * k->Q, q, sizeof(float) * k->Q); memcpy(k->v + (size_t)k->n * k->H, v, sizeof(float) * k->H); }
  ++k->n;
}

/* One iteration of the walk's solver: build_solver (subgame_solving.cc:1052-1063) returns CFR or FP. */
static void walk_step(orc_cfr* s, int it, int use_cfr, int optimistic) {
  if (use_cfr) orc_cfr_step(s, it % 2); else orc_fp_step(s, it % 2, optimistic);
}

/* RlRunner::step `n_games` times (stopping early after `max_subgames` solved subgames when it is > 0).  The solver is CFR
 * (linear, plain or DCFR) with use_cfr, fictitious play otherwise.  trace (optional): one row per solved subgame, [trace_cap][5]
 * int32 = game index, root last_bid, root player, act_iteration, br_sampler.  Returns the number of examples (two per subgame). */
int orc_rl_runner(int D, int F, int num_iters, int max_depth, int linear_update, float random_action_prob, int sample_leaf,
                  int seed, int n_games, const float* net_w, int hidden, float* q_out, float* v_out, int cap,
                  int use_cfr, int optimistic, int dcfr, double dcfr_alpha, double dcfr_beta, double dcfr_gamma,
                  int max_subgames, int32_t* trace, int trace_cap) {
  orc_game g = game_make(D, F);
  int H = g.H, A = g.A, Q = 2 + A + 2 * H;
  ex_sink sink = {q_out, v_out, 0, cap, Q, H};
  orc_mt gen; mt_seed(&gen, (uint32_t)seed);
  double* beliefs = (double*)malloc(sizeof(double) * 2 * H);
  double* sb = (double*)malloc(sizeof(double) * 2 * H);
  float* qrow = (float*)malloc(sizeof(float) * Q); float* vrow = (float*)malloc(sizeof(float) * H);
  if (!use_cfr) dcfr = 0;
  int solved = 0;
  for (int game_i = 0; game_i < n_games && !(max_subgames > 0 && solved >= max_subgames); ++game_i) {   /* RlRunner::step :160-182 */
    int last_bid = -1, player = 0;
    for (int i = 0; i < 2 * H; ++i) beliefs[i] = 1.0 / H;
    while (!game_is_terminal(&g, last_bid) && !(max_subgames > 0 && solved >= max_subgames)) {
      orc_cfr* s = orc_cfr_create(D, F, last_bid, player, beliefs, num_iters, max_depth, linear_update, dcfr, dcfr_alpha, dcfr_beta,
                                  dcfr_gamma, net_w, hidden);
      int act_iteration = uniform_int(&gen, 0, num_iters);
      int32_t* tr = trace && solved < trace_cap ? trace + 5 * (size_t)solved : 0;
      if (tr) { tr[0] = game_i; tr[1] = last_bid; tr[2] = player; tr[3] = act_iteration; tr[4] = -1; }
      ++solved;
      for (int it = 0; it < act_iteration; ++it) walk_step(s, it, use_cfr, optimistic);
      /* get_sampling_strategy = get_belief_propogation_strategy: CFR's last strategies, FP's average strategies (the
       * ISubgameSolver defaults, subgame_solving.h:76-83) */
      const double* sigma = use_cfr ? s->last : s->avg;
      if (sample_leaf) {   /* sample_state_to_leaf :192-246 */
        int path_n[64], path_a[64], plen = 0;
        int node = 0;
        int br_sampler = uniform_int(&gen, 0, 1);
        if (tr) tr[4] = br_sampler;
        memcpy(sb, beliefs, sizeof(double) * 2 * H);
        while (s->tree[node].children_end - s->tree[node].children_begin) {
          float eps = canonical_f(&gen);
          int pid = s->tree[node].player_id, lo, hi, action;
          game_bid_range(&g, s->tree[node].last_bid, &lo, &hi);
          if (pid == br_sampler && eps < random_action_prob) {
            action = uniform_int(&gen, lo, hi - 1);
          } else {
            int hand = discrete(&gen, sb + pid * H, H);
            action = discrete(&gen, sigma + IDX3(s, node, hand, 0), A);
          }
          for (int h = 0; h < H; ++h) sb[pid * H + h] *= sigma[IDX3(s, node, h, action)];
          normalize_safe_d(sb + pid * H, H, 1e-80);
          path_n[plen] = node; path_a[plen] = action; ++plen;
          node = s->tree[node].children_begin + action - lo;
        }
        for (int i = 0; i < plen; ++i) {   /* second pass :235-245 */
          int lo, hi; game_bid_range(&g, last_bid, &lo, &hi);
          for (int h = 0; h < H; ++h) beliefs[player * H + h] *= sigma[IDX3(s, path_n[i], h, path_a[i])];
          normalize_safe_d(beliefs + player * H, H, 1e-80);
          int child = s->tree[path_n[i]].children_begin + path_a[i] - lo;
          last_bid = s->tree[child].last_bid; player = s->tree[child].player_id;
        }
      } else {             /* sample_state_single :248-275 */
        int br_sampler = uniform_int(&gen, 0, 1);
        if (tr) tr[4] = br_sampler;
        float eps = canonical_f(&gen);
        int lo, hi, action; game_bid_range(&g, last_bid, &lo, &hi);
        if (player == br_sampler && eps < random_action_prob) {
          action = uniform_int(&gen, lo, hi - 1);
        } else {
          int hand = discrete(&gen, beliefs + player * H, H);
          action = discrete(&gen, sigma + IDX3(s, 0, hand, 0), A);
        }
        for (int h = 0; h < H; ++h) beliefs[player * H + h] *= sigma[IDX3(s, 0, h, action)];
        normalize_safe_d(beliefs + player * H, H, 1e-80);
        last_bid = action; player = 1 - player;
      }
      for (int it = act_iteration; it < num_iters; ++it) walk_step(s, it, use_cfr, optimistic);
      /* update_value_network (CFR :672-676, FP :471-474 through its BRSolver, whose reaches are those of the last step) ->
       * add_training_example :220-226 */
      for (int t = 0; t < 2; ++t) {
        write_query(&g, t, s->tree[0].last_bid, s->tree[0].player_id, s->reach[0], s->reach[1], qrow);
        for (int h = 0; h < H; ++h) vrow[h] = (float)s->root_means[t][h];
        sink_add(&sink, qrow, vrow);
      }
      orc_cfr_destroy(s);
    }
  }
  free(beliefs); free(sb); free(qrow); free(vrow);
  return sink.n;
}

/* ------------------------------------------------------------------ synthetic inputs + timed port baseline */
/* uniform_real_distribution<double>(0,1) = generate_canonical<double,53> (two draws each). */
/* ------------------------------------------------------------------ sampled recursive strategies (BASELINE config 5) */
/* std::discrete_distribution over n weights of any length (the iteration weights: n = num_iters) */
static int discrete_n(orc_mt* m, const double* w, int n) {
  if (n < 2) return 0;
  double sum = 0; for (int i = 0; i < n; ++i) sum += w[i];
  double* cp = (double*)malloc(sizeof(double) * n);
  double acc = 0;
  for (int i = 0; i < n; ++i) { acc += w[i] / sum; cp[i] = acc; }
  cp[n - 1] = 1.0;
  double p = canonical_d(m);
  int lo = 0, hi = n;
  while (lo < hi) { int mid = (lo + hi) / 2; if (cp[mid] < p) lo = mid + 1; else hi = mid; }
  free(cp);
  return lo;
}

typedef struct {
  orc_game g; const orc_node* full; int D, F, num_iters, max_depth, linear, hidden; const float* net_w;
  const double* weights; orc_mt* gen; double* out;   /* out: dense [N_full][H][A] */
} sampled_ctx;

/* compute_strategy_recursive_to_leaf with use_samplig_strategy = true (recursive_solving.cc:76-134) under the solver builder of
 * compute_sampled_strategy_recursive_to_leaf (:301-327): every subgame is solved for act_iteration ~ iteration weights and its
 * LAST strategy both fills the inner nodes and propagates the beliefs; recursion happens while the BFS pops a non-final leaf. */
static void sampled_rec(sampled_ctx* c, int node_id, const double* beliefs /*[2][H]*/) {
  const orc_node* fn = &c->full[node_id];
  if (game_is_terminal(&c->g, fn->last_bid)) return;
  const int H = c->g.H, A = c->g.A;
  const int act_iteration = discrete_n(c->gen, c->weights, c->num_iters);
  orc_cfr* s = orc_cfr_create(c->D, c->F, fn->last_bid, fn->player_id, beliefs, act_iteration, c->max_depth, c->linear, 0, 0, 0, 0,
                              c->net_w, c->hidden);
  for (int it = 0; it < act_iteration; ++it) orc_cfr_step(s, it % 2);
  int* qfull = (int*)malloc(sizeof(int) * s->N);
  int* qpart = (int*)malloc(sizeof(int) * s->N);
  double* qreach = (double*)malloc(sizeof(double) * (size_t)s->N * 2 * H);
  int head = 0, tail = 0;
  qfull[tail] = node_id; qpart[tail] = 0; memcpy(qreach, beliefs, sizeof(double) * 2 * H); ++tail;
  while (head < tail) {
    const int f = qfull[head], pn = qpart[head];
    double* reach = qreach + (size_t)head * 2 * H;
    ++head;
    memcpy(c->out + (size_t)f * H * A, s->last + IDX3(s, pn, 0, 0), sizeof(double) * H * A);
    const orc_node* pnode = &s->tree[pn];
    const orc_node* fnode = &c->full[f];
    const int pnc = pnode->children_end - pnode->children_begin, fnc = fnode->children_end - fnode->children_begin;
    int lo, hi; game_bid_range(&c->g, fnode->last_bid, &lo, &hi);
    for (int i = 0; i < pnc; ++i) {
      double* cr = qreach + (size_t)tail * 2 * H;
      memcpy(cr, reach, sizeof(double) * 2 * H);
      const int pid = fnode->player_id, action = lo + i;
      for (int h = 0; h < H; ++h) cr[pid * H + h] *= s->last[IDX3(s, pn, h, action)];
      qfull[tail] = fnode->children_begin + i; qpart[tail] = pnode->children_begin + i; ++tail;
    }
    if (pnc == 0 && fnc != 0) {
      normalize_safe_d(reach, H, 1e-80);
      normalize_safe_d(reach + H, H, 1e-80);
      sampled_rec(c, f, reach);
    }
  }
  free(qfull); free(qpart); free(qreach);
  orc_cfr_destroy(s);
}

/* Same signature and semantics as ref_sampled_strategy in oracle/ref_harness.cc. */
int orc_sampled_strategy(int D, int F, int num_iters, int max_depth, int linear_update, int seed, const float* net_w, int hidden,
                         double* strategy_out) {
  sampled_ctx c;
  c.g = game_make(D, F); c.D = D; c.F = F; c.num_iters = num_iters; c.max_depth = max_depth; c.linear = linear_update;
  c.hidden = hidden; c.net_w = net_w; c.out = strategy_out;
  int N = 0;
  orc_node* full = tree_unroll(&c.g, -1, 0, 1000000, &N);
  c.full = full;
  double* weights = (double*)malloc(sizeof(double) * (num_iters > 0 ? num_iters : 1));
  for (int i = 0; i < num_iters; ++i) weights[i] = i % 2 ? 0.0 : (i / 2. + 1);   /* :304-309 */
  c.weights = weights;
  orc_mt gen; mt_seed(&gen, (uint32_t)seed);
  c.gen = &gen;
  const int H = c.g.H;
  memset(strategy_out, 0, sizeof(double) * (size_t)N * H * c.g.A);
  double* beliefs = (double*)malloc(sizeof(double) * 2 * H);
  for (int i = 0; i < 2 * H; ++i) beliefs[i] = 1. / H;
  sampled_rec(&c, 0, beliefs);
  free(beliefs); free(weights); free(full);
  return N;
}

/* reach_probabilities of compute_stategy_stats (subgame_solving.cc:823-842): dense [2][N][H] from uniform beliefs. */
int orc_strategy_reach(int D, int F, const double* strategy, double* reach_out) {
  orc_cfr* s = (orc_cfr*)calloc(1, sizeof(orc_cfr));
  s->g = game_make(D, F);
  s->tree = tree_unroll(&s->g, -1, 0, 1000000, &s->N);
  const int H = s->g.H, N = s->N;
  double* beliefs = (double*)malloc(sizeof(double) * H);
  for (int i = 0; i < H; ++i) beliefs[i] = 1. / H;
  compute_reach(s, strategy, beliefs, 0, reach_out);
  compute_reach(s, strategy, beliefs, 1, reach_out + (size_t)N * H);
  free(beliefs); free(s->tree); free(s);
  return N;
}

/* ------------------------------------------------------------------ evaluation entry points (rela/pybind.cc:45-84) */
static void solve_all(orc_cfr* s, int use_cfr, int iters) {   /* multistep of CFR (:666-670) or FP (:462-466) */
  for (int it = 0; it < iters; ++it) { if (use_cfr) orc_cfr_step(s, it % 2); else orc_fp_step(s, it % 2, 0); }
}

typedef struct {
  orc_game g; const orc_node* full; int D, F, num_iters, max_depth, linear, use_cfr, hidden; const float* net_w; double* out;
} eval_ctx;

/* compute_strategy_recursive (recursive_solving.cc:46-74): a solver at EVERY non-terminal node; its average strategy's root row is
 * kept; the acting player's beliefs are multiplied by that row and eps-normalised for each child. */
static void strategy_recursive_rec(eval_ctx* c, int node_id, const double* beliefs) {
  const orc_node* fn = &c->full[node_id];
  if (game_is_terminal(&c->g, fn->last_bid)) return;
  const int H = c->g.H, A = c->g.A;
  orc_cfr* s = orc_cfr_create(c->D, c->F, fn->last_bid, fn->player_id, beliefs, c->num_iters, c->max_depth, c->linear, 0, 0, 0, 0,
                              c->net_w, c->hidden);
  solve_all(s, c->use_cfr, c->num_iters);
  memcpy(c->out + (size_t)node_id * H * A, s->avg, sizeof(double) * H * A);   /* get_strategy()[0] */
  orc_cfr_destroy(s);
  int lo, hi; game_bid_range(&c->g, fn->last_bid, &lo, &hi);
  double* nb = (double*)malloc(sizeof(double) * 2 * H);
  for (int child = fn->children_begin; child < fn->children_end; ++child) {
    const int action = child - fn->children_begin + lo, pid = fn->player_id;
    memcpy(nb, beliefs, sizeof(double) * 2 * H);
    for (int h = 0; h < H; ++h) nb[pid * H + h] *= c->out[((size_t)node_id * H + h) * A + action];
    normalize_safe_d(nb + pid * H, H, 1e-80);
    strategy_recursive_rec(c, child, nb);
  }
  free(nb);
}

/* compute_strategy_recursive_to_leaf with use_samplig_strategy = false (:76-134): all iterations, average strategy both as
 * the strategy and for belief propagation. */
static void strategy_to_leaf_rec(eval_ctx* c, int node_id, const double* beliefs) {
  const orc_node* fnr = &c->full[node_id];
  if (game_is_terminal(&c->g, fnr->last_bid)) return;
  const int H = c->g.H, A = c->g.A;
  orc_cfr* s = orc_cfr_create(c->D, c->F, fnr->last_bid, fnr->player_id, beliefs, c->num_iters, c->max_depth, c->linear, 0, 0, 0, 0,
                              c->net_w, c->hidden);
  solve_all(s, c->use_cfr, c->num_iters);
  int* qfull = (int*)malloc(sizeof(int) * s->N);
  int* qpart = (int*)malloc(sizeof(int) * s->N);
  double* qreach = (double*)malloc(sizeof(double) * (size_t)s->N * 2 * H);
  int head = 0, tail = 0;
  qfull[tail] = node_id; qpart[tail] = 0; memcpy(qreach, beliefs, sizeof(double) * 2 * H); ++tail;
  while (head < tail) {
    const int f = qfull[head], pn = qpart[head];
    double* reach = qreach + (size_t)head * 2 * H;
    ++head;
    memcpy(c->out + (size_t)f * H * A, s->avg + IDX3(s, pn, 0, 0), sizeof(double) * H * A);
    const orc_node* pnode = &s->tree[pn];
    const orc_node* fnode = &c->full[f];
    const int pnc = pnode->children_end - pnode->children_begin, fnc = fnode->children_end - fnode->children_begin;
    int lo, hi; game_bid_range(&c->g, fnode->last_bid, &lo, &hi);
    for (int i = 0; i < pnc; ++i) {
      double* cr = qreach + (size_t)tail * 2 * H;
      memcpy(cr, reach, sizeof(double) * 2 * H);
      const int pid = fnode->player_id, action = lo + i;
      for (int h = 0; h < H; ++h) cr[pid * H + h] *= s->avg[IDX3(s, pn, h, action)];
      qfull[tail] = fnode->children_begin + i; qpart[tail] = pnode->children_begin + i; ++tail;
    }
    if (pnc == 0 && fnc != 0) {
      normalize_safe_d(reach, H, 1e-80);
      normalize_safe_d(reach + H, H, 1e-80);
      strategy_to_leaf_rec(c, f, reach);
    }
  }
  free(qfull); free(qpart); free(qreach);
  orc_cfr_destroy(s);
}

/* eval_net (stats.cc:44-153); node order = stable sort by decreasing reach (the reference's std::sort may order exact ties
 * differently, which only permutes a float32 sum). */
typedef struct { double reach; int node; } reach_key;
static int reach_cmp(const void* a, const void* b) {
  const reach_key* x = (const reach_key*)a; const reach_key* y = (const reach_key*)b;
  if (x->reach > y->reach) return -1;
  if (x->reach < y->reach) return 1;
  return x->node - y->node;
}
static float eval_net_port(int D, int F, int mdp_depth, int fp_iters, const orc_node* full, int N, const double* net_strategy,
                           const double* full_strategy, const orc_net* net, int traverse_by_net) {
  orc_game g = game_make(D, F);
  const int H = g.H, A = g.A, Q = 2 + A + 2 * H;
  double* rn = (double*)malloc(sizeof(double) * 2 * (size_t)N * H);
  double* rt = (double*)malloc(sizeof(double) * 2 * (size_t)N * H);
  orc_strategy_reach(D, F, net_strategy, rn);
  orc_strategy_reach(D, F, full_strategy, rt);
  const double* trav = traverse_by_net ? rn : rt;
  reach_key* top = (reach_key*)malloc(sizeof(reach_key) * N);
  int nt = 0;
  for (int i = 0; i < N; ++i) {
    if ((full[i].depth == mdp_depth || full[i].depth == 2 * mdp_depth) && !game_is_terminal(&g, full[i].last_bid)) {
      double s0 = 0, s1 = 0;
      for (int h = 0; h < H; ++h) { s0 += trav[(size_t)i * H + h]; s1 += trav[((size_t)N + i) * H + h]; }
      top[nt].reach = s0 * s1; top[nt].node = i; ++nt;
    }
  }
  qsort(top, nt, sizeof(reach_key), reach_cmp);
  const float kMinReach = 1e-6f;
  while (nt > 0 && top[nt - 1].reach < kMinReach) --nt;
  float total = 0.f; int count = 0;
  double* beliefs = (double*)malloc(sizeof(double) * 2 * H);
  float* query = (float*)malloc(sizeof(float) * Q);
  float* out = (float*)malloc(sizeof(float) * H);
  for (int k = 0; k < nt; ++k) {
    const int node = top[k].node;
    for (int p = 0; p < 2; ++p) {   /* normalize_probabilities (util.h:20-34) */
      const double* r = trav + ((size_t)p * N + node) * H;
      double sum = 0; for (int h = 0; h < H; ++h) sum += r[h];
      for (int h = 0; h < H; ++h) beliefs[p * H + h] = r[h] / sum;
    }
    orc_cfr* s = orc_cfr_create(D, F, full[node].last_bid, full[node].player_id, beliefs, fp_iters, 10000, 1, 0, 0, 0, 0, NULL, 0);
    solve_all(s, /*use_cfr=*/0, fp_iters);
    for (int t = 0; t < 2; ++t) {
      write_query(&g, t, full[node].last_bid, full[node].player_id, beliefs, beliefs + H, query);
      net_forward(net, query, 1, out);
      double nv = 0, bv = 0;
      for (int h = 0; h < H; ++h) { nv += (double)out[h] * beliefs[t * H + h]; bv += s->root_means[t][h] * beliefs[t * H + h]; }
      const float d = (float)nv - (float)bv;
      total += (float)((double)d * (double)d);
      ++count;
    }
    orc_cfr_destroy(s);
  }
  free(rn); free(rt); free(top); free(beliefs); free(query); free(out);
  return count ? total / count : 0.f;
}

/* Same signature and semantics as ref_net_evaluation in oracle/ref_harness.cc. */
int orc_net_evaluation(int D, int F, int num_iters, int max_depth, int linear_update, int use_cfr, const float* net_w, int hidden,
                       int what, double* strategy_recursive, double* strategy_to_leaf, double* out4) {
  eval_ctx c;
  c.g = game_make(D, F); c.D = D; c.F = F; c.num_iters = num_iters; c.max_depth = max_depth; c.linear = linear_update;
  c.use_cfr = use_cfr; c.hidden = hidden; c.net_w = net_w;
  int N = 0;
  orc_node* full = tree_unroll(&c.g, -1, 0, 1000000, &N);
  c.full = full;
  const int H = c.g.H, A = c.g.A;
  const size_t dense = (size_t)N * H * A;
  double* beliefs = (double*)malloc(sizeof(double) * 2 * H);
  for (int i = 0; i < 2 * H; ++i) beliefs[i] = 1. / H;
  double e[2];
  if (what & 1) {
    double* out = strategy_recursive ? strategy_recursive : (double*)malloc(sizeof(double) * dense);
    memset(out, 0, sizeof(double) * dense);
    c.out = out;
    strategy_recursive_rec(&c, 0, beliefs);
    orc_exploitability(D, F, out, e);
    out4[0] = (e[0] + e[1]) / 2.0;
    if (!strategy_recursive) free(out);
  }
  if (what & 2) {
    double* out = strategy_to_leaf ? strategy_to_leaf : (double*)malloc(sizeof(double) * dense);
    memset(out, 0, sizeof(double) * dense);
    c.out = out;
    strategy_to_leaf_rec(&c, 0, beliefs);
    orc_exploitability(D, F, out, e);
    out4[1] = (e[0] + e[1]) / 2.0;
    /* full-tree solver with the same parameters (pybind.cc:69-73) */
    orc_cfr* full_solver = orc_cfr_create(D, F, -1, 0, beliefs, num_iters, 100000, linear_update, 0, 0, 0, 0, NULL, 0);
    solve_all(full_solver, use_cfr, num_iters);
    orc_net net = net_from_flat(net_w, 2 + A + 2 * H, hidden, H);
    out4[2] = eval_net_port(D, F, max_depth, num_iters, full, N, out, full_solver->avg, &net, 1);
    out4[3] = eval_net_port(D, F, max_depth, num_iters, full, N, out, full_solver->avg, &net, 0);
    orc_cfr_destroy(full_solver);
    if (!strategy_to_leaf) free(out);
  }
  free(beliefs); free(full);
  return N;
}

void orc_synthetic_beliefs(int H, int seed, double* out) {
  orc_mt m; mt_seed(&m, (uint32_t)seed);
  for (int p = 0; p < 2; ++p) {
    double s = 0;
    for (int h = 0; h < H; ++h) s += (out[p * H + h] = canonical_d(&m));
    for (int h = 0; h < H; ++h) out[p * H + h] /= s;
  }
}

/* Single-thread port baseline (kind "port"): n root subgames, build + multistep.  Returns seconds. */
double orc_bench_solve(int D, int F, int last_bid, int player_id, int num_iters, int max_depth, int n_subgames, int seed0,
                       const float* net_w, int hidden, double* root_means_out, const double* beliefs_in) {
  orc_game g = game_make(D, F);
  int H = g.H;
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  double* b = (double*)malloc(sizeof(double) * 2 * H);
  for (int i = 0; i < n_subgames; ++i) {
    if (beliefs_in) memcpy(b, beliefs_in + (size_t)i * 2 * H, sizeof(double) * 2 * H);
    else orc_synthetic_beliefs(H, seed0 + i, b);
    orc_cfr* s = orc_cfr_create(D, F, last_bid, player_id, b, num_iters, max_depth, 1, 0, 0, 0, 0, net_w, hidden);
    for (int it = 0; it < num_iters; ++it) orc_cfr_step(s, it % 2);
    if (root_means_out)
      for (int p = 0; p < 2; ++p) for (int h = 0; h < H; ++h) root_means_out[((size_t)i * 2 + p) * H + h] = s->root_means[p][h];
    orc_cfr_destroy(s);
  }
  free(b);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  return (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
}
