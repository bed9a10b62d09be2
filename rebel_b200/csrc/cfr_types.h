// Device-visible plain structs shared by the CFR kernels (cfr_kernels.cu) and the C-ABI host code (cfrb_api.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cfrb {

struct TemplateDev {
  int node_off, level_off, pleaf_off, term_off;
  int N, L, T, levels;
  int qconst_off, pad_[3];
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
  const int* wave_n;              // [1] number of live subgames
  const int* sg_tmpl; const int* sg_player; const int* sg_row_off; const int* sg_act_iter;
  const int* sg_order;            // [K] wave positions largest template first (cfr_iter_d2_kernel's schedule) -- or nullptr = identity
  int* ticket;                    // [1] cfr_iter_d2_kernel's subgame counter; zero between launches
  const real* beliefs;            // [K][2][H]
  real* mu;                       // [K][2][H] root_values_means
  int* steps;                     // [K][2]
  real* R; real* Sg; real* S; real* Snap;   // [K][table_stride]
  int table_stride;
  real* vterm; int vterm_stride;  // [K][Tmax*H] terminal payoffs of the current iteration
  float* X;                       // [rows][Qpad] fp32 query rows (SIMT net) -- or nullptr
  __half* Xh;                     // fp16 query tiles in wgmma core-matrix order (tensor-core net) -- or nullptr
  const float* net_out;           // [rows][Hout] raw net outputs
  real* scaler;                   // [rows] sum of opponent reach at the pseudo-leaf
  real* scratch; size_t scratch_stride;   // global scratch (CTA groups), reals per subgame
  int nh_max, tmp_reals;                  // scratch layout: bufA[nh_max] | bufB[nh_max] | tmp[tmp_reals] | lsum[2*Lmax]
  int lmax, tmax, n1max;                  // largest pseudo-leaf / terminal / level-1 node count over the templates (depth <= 2 kernels' layouts)
  // params
  int linear, dcfr; real dcfr_alpha, dcfr_beta, dcfr_gamma;
  int use_net;
  int fp, optimistic;             // fictitious play instead of CFR (FP, subgame_solving.cc:364-506)
  int keep_sum;                   // CFR: 1 = maintain S (sum_strategies); 0 = neither read nor write it (a self-play wave, whose
                                  // loop never reads it).  FP always keeps it: its average strategy is computed from S.
};

// Scratch of a group (reals): bufA[N*H] | bufB[N*H] | hist[10*T] | lsum[2*L]  (hist: per-terminal match-count histogram,
// 9 bins + belief sum)
__host__ __device__ inline int cfr_tmp_reals(int N, int H, int L, int T) { (void)N; (void)H; (void)L; return 10 * (T > 0 ? T : 1); }
__host__ __device__ inline int cfr_scratch_reals(int N, int H, int L, int T) { return 2 * N * H + cfr_tmp_reals(N, H, L, T) + 2 * (L > 0 ? L : 1); }

// Depth <= 2 kernel (cfr_iter_d2_kernel): slot[N*H] | bel[2*H] | aux.  aux (bytes) serves the backward half as
// rcp[(n1max + 1) * H] reals (reciprocals of the regret-matching sums) and the forward half first as par_sum[n1max] | par_inv[n1max]
// reals followed by the fp16 belief columns qpar[n1max * H] | qown[L * H], then as the terminal histogram hist[10 * T] reals.
__host__ __device__ inline int cfr_aux_bytes_d2(int sz, int H, int L, int T, int n1max) {
  const int fwd = ((2 * n1max * sz + 15) & ~15) + (((n1max + (L > 0 ? L : 1)) * H * 2 + 15) & ~15);
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
  int* wave;                          // [0] = number of subgames, [1] = value-net rows
  int* sg_tmpl; int* sg_player; int* sg_row_off; int* sg_act;
  int* sg_order;                      // [K] wave positions sorted by tmpl_rank (stable)
  const int* tmpl_rank;               // [A] schedule rank of each template, 0 = the costliest (schedule_ranks, cfr_tree.h)
  int table_stride;
};
void sp_launch_seed(const SpDev& p, const uint32_t* dev_seeds, cudaStream_t st);
// act_iteration draw + subgame descriptors + packed row offsets of the next wave
template <typename real> void sp_launch_begin(const SpDev& p, real* wave_beliefs, cudaStream_t st);
// training examples of the finished wave (skipped when ex_q == nullptr) and the sampling step of every game
template <typename real> void sp_launch_finish(const SpDev& p, const real* mu, const real* snap, float* ex_q, float* ex_v, cudaStream_t st);
// Head-to-head matches (match_kernels.cuh): S game slots playing G games between two handles (agent 0 = A, 1 = B).
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
  // tree templates (read-only; both handles index the same ones)
  const TemplateDev* tmpl; const int* child_begin; const int* nchild;
  const unsigned char* matches;       // [H][F]
  int table_stride;
  // each agent's wave descriptors and CFR step counters
  int* wave[2]; int* sg_tmpl[2]; int* sg_player[2]; int* sg_row_off[2]; int* sg_act[2]; const int* steps[2];
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
// Local best response against one agent (lbr_kernels.cuh): the match's slots and games with handle 0 as the agent; index 1 of
// m's per-agent arrays is unused.  m.bel holds per slot the agent's beliefs [player][hand] (rows 0, 1) and LBR's belief over the
// agent's hand (row 2).
struct LbrDev {
  MatchDev m;
  int K;                              // subgames per round (the agent's max_subgames)
  int* nsg;                           // [S] subgames the slot holds in this round's wave (0 = waiting or done)
  int* pend;                          // [S] 1: LBR's decision at (last_bid, player) waits for the solves of its raises' children
  double* sigx;                       // [S][A][H] the agent's strategy for LBR's seat at that node, per raise
  int* rr;                            // [1] rotated slot position where the next round's admission starts
  unsigned long long* deferred;       // [1] running slots left out of a round, summed over rounds
  int* solves; int* whatif;           // [G] subgames solved for game g, and how many of them were what-if solves
  double* tr_val; double* tr_beta;    // [T][A][A] LBR's action values (NaN = illegal / not LBR's ply), [T][A][H] its belief
};
template <typename real> void lbr_launch_begin(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st);
template <typename real> void lbr_launch_advance(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st);
// A ReBeL agent played from outside (agent_kernels.cuh): T independent tables, each a game between the agent (one handle) and an
// external player.  A call lists n distinct tables; the kernels of that call index the per-table state through ids[0..n).
struct AgentDev {
  int T, A, H, max_depth, sampled, iters;
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
};
void agent_launch_new(const AgentDev& p, cudaStream_t st);
// scan + subgame descriptors of the listed tables that stand at an unsolved root
template <typename real> void agent_launch_begin(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st);
template <typename real> void agent_launch_capture(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st);
void agent_launch_step(const AgentDev& p, cudaStream_t st);
void agent_launch_policy(const AgentDev& p, cudaStream_t st);
// Recursive to-leaf walk (expl_kernels.cuh): one wave of a level of subgames, rooted at full-tree nodes, solved by one handle.
struct ExplDev {
  int H;
  // the full tree (BrState of the handle) and the compact full-tree strategy [N_full - 1][H] the walk fills
  const int* full_child_begin; const int* full_depth; const int* full_act_lo;
  double* strategy;
  // the handle's subgame templates
  const TemplateDev* tmpl; const int* parent; const int* child_begin; const int* nchild; const int* level_begin;
  const int* pleaf_node;
  // the handle's wave descriptors and CFR step counters
  int* sg_tmpl; int* sg_player; int* sg_act; const int* sg_row_off; const int* wave; const int* steps;
  int table_stride;
  // this level's roots [n_level] and fp64 beliefs [n_level][2][H]; the wave is entries off .. off + n - 1
  const int* roots; const double* bel;
  int off;
  // the next level: cap entries, fill [1] of them written by the level's earlier waves
  int* next_roots; double* next_bel;
  int* fill;
  int cap;
  int* fid; int nmax;                 // [K][nmax] scratch: full-tree node of every template node of each subgame
};
// wave descriptors (template, player, root beliefs as `real`), row offsets and schedule of the level's subgames off .. off + n - 1
template <typename real> void expl_launch_begin(const ExplDev& p, const SpDev& scan, int n, real* wave_beliefs, cudaStream_t st);
// the solved wave's strategy into p.strategy, its pseudo-leaves onto the next level
template <typename real> void expl_launch_expand(const ExplDev& p, int n, const real* table, int normalise, cudaStream_t st);
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
