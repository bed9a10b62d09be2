// Device-visible plain structs shared by the CFR kernels (cfr_kernels.cu) and the C-ABI host code (cfrb_api.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cfrb {

// Terminal payoffs (subgame_solving.cc:765-789) count the opponent's hands by match count.  The reference sizes that histogram
// 2 * num_dice + 1; the CFR, best-response and regret kernels keep 9 bins (kMaxBins) and clamp the count a hand still needs to
// bin 8.  That is exact only while bin 8 stays empty, i.e. for at most 7 dice per player: cfrb_create refuses larger games.
constexpr int kMaxDice = 7;

struct TemplateDev {
  int node_off, level_off, pleaf_off, term_off;
  int N, L, T, levels;
  int qconst_off, pad_[3];
};

// Row counters of the compacted query tiles (cfr_iter_d2_kernel with the tensor-core net).  The forward half of iteration i packs
// the rows the value net must evaluate ("live") at the front of the tiles and the others ("dead") at the back, counting both in
// slot i & 1; the value net of iteration i reads live[i & 1].  The CFR launch of iteration i + 1 adds live[i & 1] to `evaluated`
// and clears slot i & 1 (its forward half fills the other slot), so both slots are zero between runs.
struct NetRows {
  int live[2], dead[2];
  int last_live;                  // live rows of the last forward half of the most recent run
  int pad_;
  unsigned long long evaluated;   // rows the value net has evaluated, summed over the handle's runs
};

template <typename real>
struct CfrDev {
  // game
  int A, H, F, Q, Qpad, Hout;
  // templates (read-only)
  const TemplateDev* tmpl;
  const int* parent; const int* child_begin; const int* nchild; const int* last_bid;
  const int* level_begin; const int* pleaf_node; const int* term_node;
  const unsigned char* matches;   // [H][F] num_matches(hand, face), liars_dice.h:83-91
  const unsigned char* tpk; int tpk_stride;   // packed byte templates (cfr_iter_d2_kernel): template i at tpk + i * tpk_stride
  const __half* qconst;           // per template [L][Qpad] fp16: constant part of the query rows (one-hot last bid, 1 at column Q)
  // wave
  const int* wave_n;              // [1] number of live subgames (of the solved set, in a self-play wave whose initial-state games share one solve)
  const int* sg_tmpl; const int* sg_player; const int* sg_row_off; const int* sg_act_iter;
  const int* sg_order;            // [K] wave positions largest template first (cfr_iter_d2_kernel's schedule) -- or nullptr = identity
  int* ticket;                    // [2] cfr_iter_d2_kernel's narrow and wide ticket counters; zero between launches
  const int* wide;                // [1] wide tickets of the wave (cfr_iter_d2_kernel, wide_count in cfr_tree.h) -- or nullptr = none
  const real* beliefs;            // [K][2][H]
  real* mu;                       // [K][2][H] root_values_means
  int* steps;                     // [K][2]
  real* R; real* Sg; real* S; real* Snap;   // [K][table_stride]
  int table_stride;
  real* vterm; int vterm_stride;  // [K][Tmax*H] terminal payoffs of the current iteration
  float* X;                       // [rows][Qpad] fp32 query rows (SIMT net) -- or nullptr
  __half* Xh;                     // fp16 query tiles in wgmma core-matrix order (tensor-core net) -- or nullptr
  float* net_out;                 // [rows][Hout] raw net outputs
  real* scaler;                   // [rows] sum of opponent reach at the pseudo-leaf
  // Compaction of the fp16 query tiles (depth-2 kernel, tensor-core net) -- or nullptr: every row at its wave position.
  NetRows* net_rows;
  int* row_src;                   // [xh_rows] wave row of each query-tile row
  int xh_rows;                    // query-tile rows allocated (a multiple of 128)
  const double* net_bound;        // [1] bound on |net output| of the current weights (cfrb_set_weights), +inf = none known
  real* scratch; size_t scratch_stride;   // global scratch (CTA groups), reals per subgame
  int nh_max, tmp_reals;                  // scratch layout: bufA[nh_max] | bufB[nh_max] | tmp[tmp_reals] | lsum[2*Lmax]
  int lmax, tmax, n1max;                  // largest pseudo-leaf / terminal / level-1 node count over the templates (depth <= 2 kernels' layouts)
  // params
  int linear, dcfr; real dcfr_alpha, dcfr_beta, dcfr_gamma;
  int use_net;
  int fp, optimistic;             // fictitious play instead of CFR (FP, subgame_solving.cc:364-506)
  int keep_sum;                   // CFR: 1 = maintain S (sum_strategies); 0 = neither read nor write it (a self-play wave, whose
                                  // loop never reads it).  FP always keeps it: its average strategy is computed from S.
  // A self-play wave whose initial-state games share one solve (sp_scan_kernel) -- or nullptr: the representative (wave position
  // *share_rep, -1 = none) leaves Sg after every iteration i in snap_hist [num_iters + 1][table_stride] at row i, from which
  // sp_share_kernel takes every initial-state game's act_iteration snapshot.
  real* snap_hist; const int* share_rep;
};

// cfr_iter_d2_kernel's wide groups use the shared memory of the CTA's second warp for kD2XchBytes of exchange ints and a copy of
// the kernel's CfrDev: they need CTAs of four warps whose group regions hold both (the host checks both, wide_warps in cfrb_api.cu).
constexpr int kD2XchBytes = 256;

// Scratch of a group (reals): bufA[N*H] | bufB[N*H] | hist[10*T] | lsum[2*L]  (hist: per-terminal match-count histogram,
// 9 bins + belief sum)
__host__ __device__ inline int cfr_tmp_reals(int N, int H, int L, int T) { (void)N; (void)H; (void)L; return 10 * (T > 0 ? T : 1); }
__host__ __device__ inline int cfr_scratch_reals(int N, int H, int L, int T) { return 2 * N * H + cfr_tmp_reals(N, H, L, T) + 2 * (L > 0 ? L : 1); }

// Depth <= 2 kernel (cfr_iter_d2_kernel): slot[N*H] | bel[2*H] | aux.  aux (bytes) serves the backward half as
// rcp[(n1max + 1) * H] reals (reciprocals of the regret-matching sums) and the forward half first as par_sum[n1max] | par_inv[n1max]
// reals followed by the fp16 belief columns qpar[n1max * H] | qown[L * H] and the leaves' query-tile rows rowpos[L] (int), then as
// the terminal histogram hist[10 * T] reals.
__host__ __device__ inline int cfr_aux_bytes_d2(int sz, int H, int L, int T, int n1max) {
  const int l1 = L > 0 ? L : 1;
  const int fwd = ((2 * n1max * sz + 15) & ~15) + (((n1max + l1) * H * 2 + 3) & ~3) + 4 * l1;
  const int bwd = (n1max + 1) * H * sz;
  const int hist = 10 * (T > 0 ? T : 1) * sz;
  int m = fwd > bwd ? fwd : bwd;
  m = m > hist ? m : hist;
  return (m + 15) & ~15;
}
__host__ __device__ inline int cfr_scratch_reals_d2(int sz, int N, int H, int L, int T, int n1max) {
  const int per16 = 16 / sz;       // every group's region starts 16-byte aligned (its template bytes are copied with 16-byte accesses)
  const int reals = N * H + 2 * H + (cfr_aux_bytes_d2(sz, H, L, T, n1max) + sz - 1) / sz;
  return (reals + per16 - 1) / per16 * per16;
}

// Full-tree best response (br_kernel.cuh).  Arrays describe ONE full-depth tree rooted at the initial state.
struct BrDev {
  int N, T, levels, H, F;
  const int* parent; const int* child_begin; const int* nchild; const int* level_begin;   // level_begin: [levels + 1]
  const int* term_node;           // [3][T]: node id, challenged bid, depth
  const unsigned char* matches;   // [H][F]
  const double* strategy;         // compact [edge = child - 1][H]
  double* scratch; size_t scratch_stride;   // per traverser: reach0[N*H] | reach1[N*H] | val[N*H] | hist[10*T]
  double* out;                    // [2]
};
void br_launch(const BrDev& p, cudaStream_t st);

// compute_ev2 of two compact full-tree strategies (ev_regret_kernels.cuh); scratch per CTA: reach1[N*H] | val[N*H] | hist[10*T].
void ev_launch(const BrDev& p, const double* s1, const double* s2, cudaStream_t st);
// Immediate-regret accumulator (ev_regret_kernels.cuh).  tree.scratch: per (strategy, traverser) reach0[N*H] | reach1[N*H] |
// hist[10*T].
struct RegretDev {
  BrDev tree;
  const int* depth; const int* act_lo;   // [N]
  int A;
  size_t s_stride;                // elements between two strategies of a batch
  double* val;                    // [S][2][N][H] traverser values
  double* acc;                    // [N][H][A] regret sums
};
// Adds S strategies (compact [S][s_stride], fp32 or fp64) to the regret sums, in order.
void regret_launch(const RegretDev& r, const float* s32, const double* s64, int S, cudaStream_t st);

// Device-resident self-play (selfplay_kernels.cuh): per-game state of K games advanced in lock-step.
constexpr int kSpMaxH = 64;       // per-thread belief copies live in local memory: larger games use the host walk
constexpr int kSpMaxPath = 16;
struct SpDev {
  int K, A, H, Q, iters, sample_leaf;
  float random_action_prob;
  // per-game state
  int* g_last_bid; int* g_player;     // [K]
  double* g_beliefs;                  // [K][2][H]   (fp64 like RlRunner::beliefs_, whatever the table dtype)
  uint32_t* mt; int* mt_idx;          // [624][K], [K]
  // tree templates (read-only; the same arrays the CFR kernels index)
  const TemplateDev* tmpl; const int* child_begin; const int* nchild; const int* last_bid;
  // wave descriptors
  int* wave;                          // [0] = number of subgames, [1] = value-net rows, [2] = subgames solved, [3] = representative,
                                      // [4] = the CFR kernel's wide tickets
  int* sg_tmpl; int* sg_player; int* sg_row_off; int* sg_act;
  int* sg_order;                      // [K] wave positions sorted by tmpl_rank (stable); when share, [solved_off, solved_off + K) the
                                      // solved ones alone (solved_off = the handle's max_subgames, so that a CUDA graph of a shared
                                      // wave stays valid when the session is re-created with another K)
  int solved_off;
  // share: the initial-state games (no bid yet, player 0, every belief bitwise 1 / H) share one solve, the one of the lowest such
  // wave position (the representative); the others are copies, which the CFR kernels skip and sp_share_kernel fills in
  int share;
  int* sg_init;                       // [K] 1 = the game is at the initial state (written only when share)
  const int* tmpl_rank;               // [A] schedule rank of each template, 0 = the costliest (schedule_ranks, cfr_tree.h)
  int table_stride;
  // the CFR kernel's wide tickets (wide_count, cfr_tree.h), which sp_scan_kernel leaves in wave[4]: the warps of its largest grid
  // (0 = none; a launch of K subgames has at most 4 ceil(K / 4)) and the test aid's setting (-1 = the rule)
  int wide_warps, wide_force;
};
void sp_launch_seed(const SpDev& p, const uint32_t* dev_seeds, cudaStream_t st);
// act_iteration draw + subgame descriptors + packed row offsets of the next wave
template <typename real> void sp_launch_begin(const SpDev& p, real* wave_beliefs, cudaStream_t st);
// training examples of the finished wave (skipped when ex_q == nullptr) and the sampling step of every game
template <typename real> void sp_launch_finish(const SpDev& p, const real* mu, const real* snap, float* ex_q, float* ex_v, cudaStream_t st);
// after the last iteration of a shared wave: the representative's results to every copy, and every initial-state game's snapshot
template <typename real> void sp_launch_share(const SpDev& p, const CfrDev<real>& d, cudaStream_t st);
// Head-to-head matches (match_kernels.cuh): S game slots playing G games between two handles (agent 0 = A, 1 = B).
// MatchDev::policy of a blueprint seat (no CFRB_MATCH_* value, so no caller's policy can name it)
constexpr int kPlyBlueprint = 3;
struct MatchDev {
  int S, G, A, H, F, max_depth, sampled, iters[2];
  uint64_t seed;
  // per slot
  int* game;                          // [S] game being played, -1 = quota done
  int* last_bid; int* player;         // [S] public node at the root of the slot's next subgames
  int* hands;                         // [S][2] dealt hand of each seat
  int* ply; int* round;               // [S] plies / subgames so far in the current game
  int* widx;                          // [S] wave index of the slot in this round (-1 = not running)
  int* act;                           // [S][2] act_iteration of each agent's current subgame
  double* bel;                        // [S][2 agents][2 players][H] fp64 beliefs
  uint32_t* mt; int* mt_idx;          // [624][S], [S]
  int* running;                       // [1] slots in this round's wave
  int* left;                          // [1] slots still holding a game after this round's walk
  // per game
  float* payoff; int* plies; int* rounds;   // [G]
  // trace of games < trace_games: per ply {agent, last bid, player, hand, action, round} and the probability of the action, per
  // subgame both agents' act_iteration and root beliefs
  int trace_games;
  int* tr_ply; double* tr_prob; int* tr_plies;             // [T][A][6], [T][A], [T]
  int* tr_act; double* tr_bel; int* tr_rounds;             // [T][A][2], [T][A][2][2][H], [T]
  // tree templates (read-only; both handles index the same ones; null in a match between two blueprints)
  const TemplateDev* tmpl; const int* child_begin; const int* nchild;
  const unsigned char* matches;       // [H][F]
  int table_stride;
  // each agent's wave descriptors and CFR step counters
  int* wave[2]; int* sg_tmpl[2]; int* sg_player[2]; int* sg_row_off[2]; int* sg_act[2]; const int* steps[2];
  // per-ply walk only (ply_kernels.cuh; the to-leaf walk leaves these unset)
  int policy[2];                      // each agent's CFRB_MATCH_* policy
  const int* level_begin;
  int* awidx[2];                      // [S] agent k's wave index of the slot in this round (-1 = k does not solve there)
  int* sub_lb[2]; int* sub_player[2]; // [S] to-leaf agent k: root of its current subgame
  int* sub_node[2]; int* sub_depth[2];   // [S] its template node and plies since that root (sub_node -1 = no subgame solved)
  double* cache[2];                   // [S][table_stride] to-leaf agent k's acting strategy in that subgame (null: every-node)
  int* solves[2];                     // [G] subgames agent k solved for game g
  // blueprint agents (cfrb_match_create3): agent k's fixed full-tree table, entry (child - 1) * H + hand, the full tree's
  // child_begin, and per slot the full-tree node the game stands at (all null for a solving agent)
  const double* bp[2]; const int* bp_child_begin[2];
  int* bp_node[2];                    // [S]
};
template <typename real>
struct MatchTabs {
  real* wave_beliefs[2];              // each handle's [K][2][H] root beliefs
  const real* table[2];               // the table each agent acts with: S (CFR average, normalised), Sg (FP average) or Snap
  int normalise[2];
};
void match_launch_deal(const MatchDev& p, cudaStream_t st);
// scan + subgame descriptors of the next round
template <typename real> void match_launch_begin(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st);
template <typename real> void match_launch_advance(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st);
// Per-ply matches (ply_kernels.cuh): one ply per round, each agent solving only where its policy needs a subgame.
void ply_launch_deal(const MatchDev& p, cudaStream_t st);
template <typename real> void ply_launch_begin(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st);
// capture: the to-leaf agents' acting strategies of this round's solves into their caches, then the ply
template <typename real> void ply_launch_advance(const MatchDev& p, const MatchTabs<real>& t, bool capture, cudaStream_t st);
// Local best response against one agent (lbr_kernels.cuh): the match's slots and games with handle 0 as the agent; index 1 of
// m's per-agent arrays is unused.  m.bel holds per slot the agent's beliefs [player][hand] (rows 0, 1) and LBR's belief over the
// agent's hand (row 2).
struct LbrDev {
  MatchDev m;
  int K;                              // subgames per round (the agent's max_subgames)
  int every_node;                     // the agent plays CFRB_MATCH_EVERY_NODE (else CFRB_MATCH_AVERAGE)
  int* nsg;                           // [S] subgames the slot holds in this round's wave (0 = waiting or done)
  int* pend;                          // [S] 1: LBR's decision at (last_bid, player) waits for the solves of its raises' children
  double* sigx;                       // [S][A][H] the agent's strategy for LBR's seat at that node, per raise (every-node: from
                                      // the what-if set-up on, the agent's belief row for LBR's seat after that raise)
  int* rr;                            // [1] rotated slot position where the next round's admission starts
  unsigned long long* deferred;       // [1] running slots left out of a round, summed over rounds
  int* solves; int* whatif;           // [G] subgames solved for game g, and how many of them were what-if solves
  double* tr_val; double* tr_beta;    // [T][A][A] LBR's action values (NaN = illegal / not LBR's ply), [T][A][H] its belief
  // against a blueprint (cfrb_match_create_lbr_blueprint; null otherwise): its table and the full tree's child_begin
  const double* bp; const int* bp_child_begin;
};
template <typename real> void lbr_launch_begin(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st);
template <typename real> void lbr_launch_advance(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st);
// against a blueprint: every running slot's game to its end, no solves
void lbr_launch_blueprint(const LbrDev& p, cudaStream_t st);
// A ReBeL agent played from outside (agent_kernels.cuh): T independent tables, each a game between the agent (one handle) and an
// external player.  A call lists n distinct tables; the kernels of that call index the per-table state through ids[0..n).
struct AgentDev {
  int T, A, H, max_depth, sampled, iters;
  int every_node;                     // 1: a subgame is solved at every node (CFRB_MATCH_EVERY_NODE), only its root row cached
  uint64_t seed;
  // per table
  int* seat; int* hand;               // [T] the agent's seat and hand
  int* last_bid; int* player; int* ply;   // [T] public node
  int* root_lb; int* root_player;     // [T] root of the current subgame
  int* node; int* depth;              // [T] node of the subgame template, plies since its root
  int* act; int* status; int* subgames;   // [T] act_iteration, 0 = no game / 1 = at an unsolved root / 2 = solved, subgames so far
  double* root_bel; double* bel;      // [T][2][H] fp64 beliefs at the subgame root (normalised) and at the node (unnormalised)
  uint32_t* mt; int* mt_idx;          // [624][T], [T]
  double* cache; int stride;          // [T][stride] acting strategy of the solved subgame, entry (child - 1) * H + hand
  // this call
  int n;
  const int* ids;                     // [n] tables of the call
  int* io;                            // [n] step: action in (-1 = the agent draws) / action played out; new games: seats
  const int* hands; const uint64_t* keys;   // [n] new games: hands and stream keys
  int* widx;                          // [n] wave index of the table's solve, -1 = none
  double* probs;                      // [n][A] step: the agent's row on its own turns, NaN on the opponent's (or nullptr)
  int* flags;                         // [n] step: bit 0 game over, bit 1 at the root of a new subgame
  double* pol;                        // [n][H][A] policy of the player to move
  // tree templates and the handle's wave descriptors
  const TemplateDev* tmpl; const int* child_begin; const int* nchild; const int* level_begin;
  int table_stride;
  int* wave; int* sg_tmpl; int* sg_player; int* sg_row_off; int* sg_act; const int* steps;
  const int* bp_child_begin;          // a blueprint agent: the full tree's child_begin (then cache is its table, stride 0); else null
};
void agent_launch_new(const AgentDev& p, cudaStream_t st);
// scan + subgame descriptors of the listed tables that stand at an unsolved root
template <typename real> void agent_launch_begin(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st);
template <typename real> void agent_launch_capture(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st);
void agent_launch_step(const AgentDev& p, cudaStream_t st);
void agent_launch_policy(const AgentDev& p, cudaStream_t st);
// Device walks (expl_kernels.cuh): one wave of a level of subgames, rooted at full-tree nodes, solved by
// one handle.  The sampled walk walks b repeats: a level lists its root groups in full-tree node order, each the b repeats of one
// root, so position pos is repeat pos % b of group pos / b.  The other walks leave its fields null / zero.  (In this field order
// ptxas keeps expl_sampled_expand_kernel free of spills.)
struct ExplDev {
  int H, A, b;
  // the full tree (BrState of the handle); the sampled walk's accumulators and strategies index its parents and size
  const int* full_child_begin; const int* full_depth; const int* full_act_lo; const int* full_parent;
  int full_nodes;
  // the handle's subgame templates
  const TemplateDev* tmpl; const int* parent; const int* child_begin; const int* nchild; const int* level_begin;
  const int* pleaf_node;
  // the handle's wave descriptors and CFR step counters
  int* sg_tmpl; int* sg_player; int* sg_act; const int* sg_row_off; const int* wave; const int* steps;
  int table_stride;
  // act_iteration of (repeat j, global level position g of its root group) = draws[j * draws_stride + level_base + g], or -1
  const int* draws; long long draws_stride; int level_base;
  // this level's roots [n_level], fp64 beliefs and reach [n_level][2][H]; the wave is positions off .. off + n - 1 (whole groups)
  const int* roots; const double* bel; const double* rch;
  int off;
  // the next level: cap positions, fill [1] of them written by the level's earlier waves
  int* next_roots; double* next_bel; double* next_rch;
  int* fill;
  long long cap;
  int* fid; int nmax;                 // [groups][nmax] scratch: full-tree node of every template node of each root group
  // float32 accumulators, compact: summed_strategy [N_full - 1][H] (entry (child - 1) * H + hand), summed_reach [N_full][H]
  float* sum_s; float* sum_r;
  // repeat last_j of the batch (-1: none) writes its sampled strategy into last [N_full - 1][H]
  double* last; int last_j;
  // with regrets tracked: every repeat j of the batch writes (float)s of its sampled strategy into rep_s + j * rep_stride,
  // compact [N_full - 1][H] (nullptr: not tracked)
  float* rep_s; size_t rep_stride;
  double* strategy;                   // the compact full-tree strategy the walk fills and the best response reads [N_full - 1][H]
  // the every-node walk (rec_expand_kernel): the full tree's child counts [N] and depth levels [levels + 1]
  const int* full_nchild; const int* full_level_begin;
};
// wave descriptors (template, player, act_iteration, root beliefs as `real`), row offsets and schedule of positions off .. off + n - 1
template <typename real> void expl_launch_begin(const ExplDev& p, const SpDev& scan, int n, real* wave_beliefs, cudaStream_t st);
// the solved wave's strategy into p.strategy, its pseudo-leaves onto the next level
template <typename real> void expl_launch_expand(const ExplDev& p, int n, const real* table, int normalise, cudaStream_t st);
// every-node walk: the solved wave's root rows into p.strategy, their non-terminal children onto the next level
template <typename real> void rec_launch_expand(const ExplDev& p, int n, const real* table, int normalise, cudaStream_t st);
// sampled walk: the solved wave's snapshot strategies into the accumulators, its pseudo-leaves (beliefs and reach) onto the next level
template <typename real> void expl_sampled_launch_expand(const ExplDev& p, int n, const real* snap, cudaStream_t st);
// strategy = (double)(sum_s / (sum_r[parent] + 1e-6f)), the final strategy of a checkpoint
void expl_sampled_launch_finalize(const ExplDev& p, cudaStream_t st);
// Full-game solver (full_game_kernels.cuh): CFR or FP on the full tree of the handle's game (BrState), fp64, one level per launch.
struct FullGameDev {
  int N, T, H, F;
  int fp, linear, dcfr, optimistic;
  double dcfr_alpha, dcfr_beta, dcfr_gamma;
  double b0;                      // root belief of every hand, 1 / H
  const int* parent; const int* child_begin; const int* nchild; const int* term_node;   // the full tree (BrDev's arrays)
  const unsigned char* matches;   // [H][F]
  double* R;                      // [N - 1][H] regrets (CFR; nullptr in FP)
  double* Sg;                     // [N - 1][H] current strategy (FP: average strategy)
  double* S;                      // [N - 1][H] sum strategy
  double* reach;                  // [N][H] reach of one player (FP: also the best-response flags)
  double* val;                    // [N][H] values (FP: also the traverser's beliefs)
  double* avg;                    // [N - 1][H] the average strategy a checkpoint evaluates (BrDev::strategy)
  int* iter;                      // [1] iterations done; the traverser of iteration i is i & 1
};
// Immediate regrets of full-tree strategies over the whole GPU (regret_grid_kernels.cuh): the full tree's arrays, four [N][H]
// tables in the handle's best-response scratch and the compact sums.
struct RegretGridDev {
  int N, T, H, F, A;
  const int* parent; const int* child_begin; const int* nchild; const int* term_node; const int* act_lo;   // BrDev's arrays
  const unsigned char* matches;   // [H][F]
  double* reach0; double* reach1; double* val0; double* val1;   // [N][H] each
  double* acc;                    // [N - 1][H] regret sums, entry (child - 1) * H + hand
};
// Adds one compact strategy [N - 1][H] (fp32 or fp64) to p.acc: about 2 launches per depth level and one for the terminals.
void regret_grid_launch(const RegretGridDev& p, const float* s32, const double* s64, const int* level_begin, int levels, int max_blocks,
                        cudaStream_t st);
// immediate [N][H] and node_sums [N] (device pointers) of the sums of `count` strategies.
void regret_grid_launch_readout(const RegretGridDev& p, double count, double* immediate, double* node_sums, int max_blocks,
                                cudaStream_t st);
// CFR constructor on the full tree (iteration counter left alone)
void full_game_launch_init(const FullGameDev& p, const int* level_begin, int levels, int max_blocks, cudaStream_t st);
// one iteration: about 2 (CFR) or 3 (FP) launches per depth level, then the counter's increment
void full_game_launch_iter(const FullGameDev& p, const int* level_begin, int levels, int max_blocks, cudaStream_t st);
// CFR's normalised sum into p.avg (FP: the host copies Sg)
void full_game_launch_average(const FullGameDev& p, const int* depth, int untouched0, int untouched1, int max_blocks, cudaStream_t st);
// FP subtree forest (fp_forest_kernels.cuh): linear FP on every full-tree subtree rooted at level d0, roots' beliefs and root value
// means bel / mu [level_begin[d0 + 1] - level_begin[d0]][2][H].  init: the FP constructor of levels d0 .. levels - 1 (iteration
// counter left alone); iter: one iteration, about 3 launches per level from d0 on, then the counter's increment.
void fp_forest_launch_init(const FullGameDev& p, const double* bel, double* mu, const int* level_begin, int levels, int d0, int max_blocks,
                           cudaStream_t st);
void fp_forest_launch_iter(const FullGameDev& p, const double* bel, double* mu, const int* level_begin, int levels, int d0, int max_blocks,
                           cudaStream_t st);
// both players' reach of a compact strategy [N - 1][H] into p.reach0 / p.reach1, then node_reach [n] and rows [n][2][H] of the
// device node list nodes [n]
void fp_forest_launch_reach(const RegretGridDev& p, const double* strategy, const int* nodes, int n, double* node_reach, double* rows,
                            const int* level_begin, int levels, int max_blocks, cudaStream_t st);
// rows [ids[i]] of a [*, width] fp32 matrix -> out[i]  (replay sampling)
void rows_launch_gather(const float* src, int width, const int* ids, int n, float* out, cudaStream_t st);

// Development check of div_by_rcp (cfr_kernels.cuh, the regret matching of cfr_iter_d2_kernel): n pseudo-random (x, b) pairs
// per call, returns the number of quotients that differ from x / b in *mismatches (device pointer).
void div_check_launch(unsigned long long seed, int blocks, unsigned long long* mismatches, cudaStream_t st);

// Launchers implemented in cfr_kernels.cu (explicitly instantiated for float and double).  `group` is 32 (one warp per
// subgame, shared-memory scratch) or 256 (one CTA per subgame, global scratch).
template <typename real> cudaError_t cfr_configure(int group, int smem_bytes);
template <typename real> void cfr_launch_init(const CfrDev<real>& p, int group, int blocks, int threads, size_t smem, cudaStream_t st,
                                              int scratch_per_group);
template <typename real> void cfr_launch_iter(const CfrDev<real>& p, int group, int blocks, int threads, size_t smem, cudaStream_t st,
                                              int iter, int do_b, int do_f, int scratch_per_group);
// Depth <= 2 specialisation (persistent warps, one subgame at a time, half the scratch); threads must be a multiple of 32 and
// <= 256.  *ctas_per_sm receives how many CTAs of `threads` threads and `smem_bytes` bytes are resident per SM for H hands.
template <typename real> cudaError_t cfr_configure_d2(int H, int threads, int smem_bytes, int* ctas_per_sm);
template <typename real> void cfr_launch_iter_d2(const CfrDev<real>& p, int blocks, int threads, size_t smem, cudaStream_t st, int iter,
                                                 int do_b, int do_f, int scratch_per_group);

}  // namespace cfrb
