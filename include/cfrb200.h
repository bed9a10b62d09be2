/*
 * cfrb200 — C ABI of the H100-native CFR subgame-wave solver (libcfrb200.so).
 *
 * This is the drop-in boundary beneath the reference's pybind11 module `cfvpy.rela`
 * (csrc/liars_dice/rela/pybind.cc:119-213): host orchestration (rebel_b200/csrc/rela/*.cc, the
 * re-implemented `rela` module) calls ONLY these entry points; they replace, on the GPU and for
 * thousands of subgames at a time, what one reference CPU thread does for one subgame at a time:
 *
 *   cfrb_create / cfrb_begin_wave   <-  build_solver + CFR ctor        (subgame_solving.cc:791-800, 509-534)
 *                                       unroll_tree                    (tree.h:51-70)
 *   cfrb_run                        <-  CFR::step / multistep          (subgame_solving.cc:577-670) including
 *                                       the per-iteration value-net call the reference makes through
 *                                       IValueNet::compute_values      (net_interface.h:28-32,
 *                                       rela/data_loop.h:29-48, rela/model_locker.h:85-95)
 *   cfrb_set_weights                <-  ModelLocker::updateModel       (rela/model_locker.h:69-79)
 *   cfrb_fetch                      <-  ISubgameSolver::get_strategy / get_sampling_strategy /
 *                                       get_hand_values                (subgame_solving.h:60-88)
 *   cfrb_examples                   <-  CFR::update_value_network      (subgame_solving.cc:672-676, 220-226)
 *   cfrb_tree_template              <-  unroll_tree, for bit-exact infoset-index checks (tree_test.cc)
 *   cfrb_exploitability             <-  compute_exploitability2        (subgame_solving.cc:802-816)
 *   cfrb_ev2                        <-  compute_ev2                    (subgame_solving.cc:931-982)
 *   cfrb_regrets_*                  <-  compute_immediate_regrets      (subgame_solving.cc:984-1050)
 *   cfrb_match_*                    <-  compute_[sampled_]strategy_recursive_to_leaf restricted to the path two agents play
 *                                       (recursive_solving.cc:76-134, 301-327); no counterpart in the reference
 *   cfrb_agent_*                    <-  the same policies, one agent against external players, one action per call; no
 *                                       counterpart in the reference
 *
 * Conventions: plain C, no exceptions across the boundary; every function returns 0 on success or a
 * negative CFRB_E* code (cfrb_last_error() gives the message for the calling thread); all buffers are
 * caller-owned HOST memory (pinned preferred); one handle per GPU; a handle is not thread-safe (one
 * orchestrator thread per handle).  There is NO CPU fallback: without a CUDA device cfrb_create fails.
 *
 * Layouts (all row-major; solver state crosses the boundary as fp64 like the reference's vector<double>, value-net
 * tensors as fp32 like the reference's float tensors):
 *   beliefs            [n][2][H]          root beliefs of player 0 then player 1 (Pair<vector<double>> in the reference)
 *   dense strategy     [n][Nmax][H][A]    the reference's TreeStrategy = [node][hand][action] (subgame_solving.h:39),
 *                                         padded to Nmax = cfrb_max_nodes() nodes per subgame; entries of illegal
 *                                         actions, leaves and padding are 0
 *   root_value_means   [n][2][H]          CFR::root_values_means (subgame_solving.cc:702-703)
 *   queries            [..][Q]            value-net query rows, Q = 2 + A + 2H (subgame_solving.cc:100-123)
 *   weights            flat fp32 in Net2 state_dict order (cfvpy/models.py:64-94):
 *                      body.0.weight[hid,Q] body.0.bias[hid] body.1.weight[hid] body.1.bias[hid]
 *                      body.4.weight[hid,hid] body.4.bias body.5.weight body.5.bias output.weight[H,hid] output.bias[H]
 */
#ifndef CFRB200_H_
#define CFRB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cfrb_handle cfrb_handle;

enum {
  CFRB_OK = 0,
  CFRB_EINVAL = -1,   /* bad argument */
  CFRB_ECUDA = -2,    /* CUDA runtime error (message has the cudaError string) */
  CFRB_ENODEV = -3,   /* no CUDA device / wrong architecture */
  CFRB_ESTATE = -4,   /* call sequence error (e.g. run before begin_wave, net needed but no weights) */
  CFRB_ENOMEM = -5
};

/* How the leaf value net (Net2 forward) is evaluated. */
enum {
  CFRB_NET_ZERO = 0,      /* leaf values are 0 (reference: create_zero_net, real_net.cc:30-55) */
  CFRB_NET_FP32 = 1,      /* fp32 SIMT kernel: parity path, matches libtorch fp32 to ~1e-6 */
  CFRB_NET_TC_F16 = 2,    /* wgmma tensor-core kernel: fp16 operands, fp32 accumulate/LayerNorm/GELU
                             (the reference's own `half_inference` option, selfplay.py:42-43,211).  Games of up to 16 hands
                             whose weights and two query tiles fit shared memory run the resident kernel; larger ones
                             (2x5f, 3x3f, 5x2f, 2x6f, 1x17f .. 1x32f) a kernel with the weights alone in shared memory;
                             cfrb_tc_net_supported() tells which games have one (CFRB_TC_WIDE=1 forces the second) */
  CFRB_NET_TC_F16X2 = 3,  /* same kernel with the fast GELU: y/2 (1 + tanh(poly)) with packed f32x2 FMAs and tanh.approx.f32, one
                             rounding to fp16 at the end (same accuracy as mode 2, 1 instead of 2 MUFU operations per element).
                             CFRB_X2_GELU=half selects the packed-fp16 evaluation (HFMA2 + tanh.approx.f16x2): 6 % faster, but
                             that instruction truncates towards zero and biases every activation (see DESIGN.md "P5") */
  CFRB_NET_TC_CLUSTER = 4 /* wgmma tensor-core kernel on a cluster of two CTAs that split Net2's 256 hidden features and exchange
                             LayerNorm sums and activations through distributed shared memory; mode 3's arithmetic (fp32 tanh
                             GELU).  Serves the games whose weights do not fit one SM (2x7f, 3x4f, 6x2f, 4x3f, 7x2f, 2x8f .. 2x11f,
                             3x5f, 1x33f .. 1x96f) and every game modes 2 and 3 serve; cfrb_tc_cluster_net_supported() tells which.
                             CFRB_X2_GELU and CFRB_TC_WIDE do not apply */
};

/* Subgame solver.  In FP mode cfrb_fetch's "last" is FP::last_strategies (belief x best response), "avg" is
 * FP::average_strategies (also the sampling / belief-propagation strategy, subgame_solving.h:76-83) and "regrets" is empty. */
enum {
  CFRB_SOLVER_CFR = 0,    /* CFR (subgame_solving.cc:508-715), params.use_cfr = true */
  CFRB_SOLVER_FP = 1      /* fictitious play (subgame_solving.cc:364-506), params.use_cfr = false */
};

/* Arithmetic type of the per-infoset CFR tables (regrets, strategies, reach, values). */
enum {
  CFRB_STATE_F64 = 0,     /* double, like the reference's TreeStrategy (default) */
  CFRB_STATE_F32 = 1      /* float: half the table traffic; trajectories drift from the fp64 reference sooner */
};

/* SubgameSolvingParams (subgame_solving.h:43-58) + game shape + capacity. */
typedef struct {
  int32_t num_dice;
  int32_t num_faces;
  int32_t max_depth;        /* depth of every subgame tree */
  int32_t num_iters;        /* iterations per subgame (only used for default graphs/snapshots) */
  int32_t linear_update;
  int32_t dcfr;
  double dcfr_alpha, dcfr_beta, dcfr_gamma;
  int32_t max_subgames;     /* wave capacity K */
  int32_t device;           /* CUDA ordinal */
  int32_t net_mode;         /* CFRB_NET_* */
  int32_t hidden;           /* Net2 n_hidden (256); n_layers = 2, LayerNorm on */
  int32_t state_dtype;      /* CFRB_STATE_* */
  int32_t solver;           /* CFRB_SOLVER_*: which ISubgameSolver build_solver would return (subgame_solving.cc:791-800) */
  int32_t optimistic;       /* FP only: SubgameSolvingParams::optimistic (subgame_solving.h:50, util.h:52-63) */
} cfrb_config;

/* One node of an unrolled subgame tree: UnrolledTreeNode (tree.h:31-47). */
typedef struct {
  int32_t last_bid, player_id, children_begin, children_end, parent, depth;
} cfrb_node;

const char* cfrb_last_error(void);
/* Number of CUDA devices visible (0 if none / driver missing). */
int cfrb_device_count(void);

int cfrb_create(const cfrb_config* cfg, cfrb_handle** out);
int cfrb_destroy(cfrb_handle* h);

/* Host-only (no device needed): 1 if a tensor-core value net (CFRB_NET_TC_F16 / CFRB_NET_TC_F16X2) with `hidden` units fits the
 * game on an sm_90 device, else 0 (cfrb_create then fails with CFRB_EINVAL for those modes; CFRB_NET_FP32 serves every game). */
int cfrb_tc_net_supported(int32_t num_dice, int32_t num_faces, int32_t hidden);
/* Host-only: 1 if the two-CTA cluster value net (CFRB_NET_TC_CLUSTER) with `hidden` units serves the game on an sm_90 device: hidden
 * == 256, a game cfrb_create accepts, and one CTA's half of the weights plus its exchange buffers fit the 227 KB of shared memory
 * a block may opt into.  Otherwise cfrb_create fails with CFRB_EINVAL for that mode. */
int cfrb_tc_cluster_net_supported(int32_t num_dice, int32_t num_faces, int32_t hidden);

/* Host-only: a bound B >= |output| of the tensor-core value net with these weights (cfrb_set_weights layout) over every query
 * row, +inf when none holds (a weight that is not finite); -1 for a bad shape or weight count.  The depth-2 CFR kernel leaves out of
 * the net's rows every pseudo-leaf whose opponent-reach scaler s has s * B <= 2^-151: its leaf values (float)(net * s) are +-0
 * whatever the net returns. */
double cfrb_net_output_bound(int32_t num_dice, int32_t num_faces, int32_t hidden, const float* flat, size_t n);

/* Shape queries. */
int cfrb_num_actions(const cfrb_handle* h);   /* A */
int cfrb_num_hands(const cfrb_handle* h);     /* H */
int cfrb_query_size(const cfrb_handle* h);    /* Q */
int cfrb_max_nodes(const cfrb_handle* h);     /* Nmax over all root templates */
/* Test aid: which CFR iteration kernel the handle runs, chosen by cfrb_create from the game, depth and state dtype:
 * 0 = cfr_iter_d2_kernel (depth <= 2 templates in shared memory), 1 = cfr_iter_kernel with a warp per subgame and its scratch in
 * shared memory, 2 = cfr_iter_kernel with a CTA per subgame and its scratch in global memory. */
int cfrb_debug_kernel_path(const cfrb_handle* h);

/* Host-only (no device needed): unroll_tree(game, {last_bid, player_id}, max_depth) (tree.h:51-70) through the same
 * template builder the kernels index with.  Returns the node count or a negative error; writes min(count, cap). */
int cfrb_unroll_tree(int32_t num_dice, int32_t num_faces, int32_t last_bid, int32_t player_id, int32_t max_depth,
                     cfrb_node* out, int32_t cap);

/* Tree of the subgame rooted at (last_bid, player_id) with the handle's max_depth, in the reference's BFS
 * node order.  Returns the node count (>0) or a negative error; writes min(count, cap) nodes. */
int cfrb_tree_template(const cfrb_handle* h, int32_t last_bid, int32_t player_id, cfrb_node* out, int32_t cap);

/* Install value-net weights (flat fp32, `n` floats, layout above).  `version` is remembered and returned by
 * cfrb_weights_version.  Takes effect for kernels enqueued after the call. */
int cfrb_set_weights(cfrb_handle* h, const float* flat, size_t n, uint64_t version);
uint64_t cfrb_weights_version(const cfrb_handle* h);

/* Start a wave of n <= max_subgames subgames.  Subgame k is rooted at (last_bid[k], player_id[k]) with
 * root beliefs beliefs[k][2][H]; state is initialised exactly like the CFR constructor
 * (uniform strategies, reach-weighted uniform sum, zero regrets, subgame_solving.cc:509-524,125-149).
 * act_iteration[k] (may be NULL) is the iteration count after which the sampling strategy
 * (CFR::last_strategies) of subgame k is snapshotted for RlRunner's state sampling
 * (recursive_solving.cc:168-174); -1 = no snapshot. */
int cfrb_begin_wave(cfrb_handle* h, int32_t n, const int32_t* last_bid, const int32_t* player_id,
                    const double* beliefs, const int32_t* act_iteration);

/* Re-initialise the solver state of the CURRENT wave on the device (same roots, beliefs and act_iterations; no
 * host->device traffic): what constructing fresh CFR solvers for the same subgames would do. */
int cfrb_reset_wave(cfrb_handle* h, void* cuda_stream);

/* Profiling switch: 0 = off; n > 0 = cfrb_run brackets every n-th value-net launch with a pair of CUDA events on the
 * launching stream, and cfrb_last_run_ms reports the value-net kernel time of the last run estimated from those samples
 * (mean sampled duration x number of launches).  Sampling keeps the event traffic out of the way of the measurement. */
int cfrb_set_profiling(cfrb_handle* h, int32_t on);

/* Advance every subgame of the wave by `iters` CFR iterations (iteration i has traverser i % 2,
 * CFR::multistep subgame_solving.cc:666-670), asynchronously on `cuda_stream` (a cudaStream_t; NULL = the
 * handle's own stream). */
int cfrb_run(cfrb_handle* h, int32_t iters, void* cuda_stream);
/* Block until everything enqueued by this handle has finished. */
int cfrb_sync(cfrb_handle* h);
/* Iterations done so far in the current wave. */
int cfrb_iterations_done(const cfrb_handle* h);

/* Copy results to the host (any pointer may be NULL).  Synchronises.
 *   root_value_means [n][2][H]; snapshot / last / avg / sum / regrets: dense [n][Nmax][H][A]. */
int cfrb_fetch(cfrb_handle* h, double* root_value_means, double* snapshot_strategy, double* last_strategy,
               double* avg_strategy, double* sum_strategy, double* regrets);

/* Compact fetch for host orchestration (BatchedRlRunner, evaluators): table `which` (0 snapshot, 1 last strategy, 2 sum strategy,
 * 3 regrets, 4 average strategy = ISubgameSolver::get_strategy) of every subgame as stored on the device, [n][cfrb_table_stride()] fp64 with entry (child_node - 1) * H + hand
 * holding the value of (parent node, hand, action leading to child_node).  Synchronises. */
int cfrb_table_stride(const cfrb_handle* h);
int cfrb_fetch_compact(cfrb_handle* h, int32_t which, double* out);

/* Training examples of the finished wave: for each subgame and traverser t in {0,1} the query row of the
 * subgame root as seen by t and the target root_value_means[t].  queries [n][2][Q], values [n][2][H]. */
int cfrb_examples(cfrb_handle* h, float* queries, float* values);

/* Teacher forcing (tests): overwrite solver state of the current wave from dense host arrays
 * [n][Nmax][H][A] (NULL = keep), root_value_means [n][2][H], num_steps [n][2], and set the wave's
 * iteration counter. */
int cfrb_load_state(cfrb_handle* h, const double* regrets, const double* last_strategy, const double* sum_strategy,
                    const double* root_value_means, const int32_t* num_steps, int32_t iterations_done);

/* Debug/parity taps of the most recent iteration: query rows [rows][Q] and the (unscaled) net outputs
 * [rows][H] for all pseudo-leaves of the wave in (subgame, leaf) order; returns the number of rows,
 * writes at most cap_rows.  After a self-play wave whose initial-state games shared one solve (cfrb_wave_solved < n), the rows of
 * the games that took the shared results were never written: their entries are not those of the wave (zero queries). */
int cfrb_debug_leaf_io(cfrb_handle* h, float* queries, float* net_out, double* scalers, int32_t cap_rows);

/* Debug taps of the tensor-core value net (either tensor-core mode, either kernel): re-runs it on the current query tiles and returns
 * the raw fp32 accumulators of layer 1 and layer 2 for the first 128 rows, each [128][256]. */
int cfrb_debug_net_taps(cfrb_handle* h, float* d1, float* d2);
/* Development aid: re-runs the tensor-core value net once with clock64() stamps of CTA 0 (out[2048]: thread 0 of warpgroup w
 * at [w*1024 + tile*8 + phase]; see TcArgs in leaf_mlp_tc.cuh). */
int cfrb_debug_net_trace(cfrb_handle* h, long long* out, int n);

/* Exploitability (best-response values of both players, compute_exploitability2) of a full-tree strategy
 * given as dense [N_full][H][A] fp64, evaluated on the GPU. out2 = {br0, br1}. */
int cfrb_exploitability(cfrb_handle* h, const double* full_strategy, double* out2);

/* Expected values of two full-tree strategies against each other, compute_ev2 (subgame_solving.cc:931-982): out2 = {ev0, ev1}
 * with ev0 = player 0 playing s1 against player 1 playing s2, ev1 = -(player 0 playing s2 against s1).  Dense [N_full][H][A]
 * fp64, evaluated on the GPU. */
int cfrb_ev2(cfrb_handle* h, const double* s1_dense, const double* s2_dense, double* out2);
/* Node count N_full of the full game tree (the tree cfrb_exploitability / cfrb_ev2 / cfrb_regrets_* index). */
int cfrb_full_tree_nodes(cfrb_handle* h);

/* Exploitability of the handle's recursive to-leaf average policy (compute_strategy_recursive_to_leaf, recursive_solving.cc:76-134:
 * every subgame solved for num_iters iterations, get_strategy), with the handle's weights and solver settings, without a dense
 * strategy: the subgames are solved level by level in waves of max_subgames (level l = the non-terminal nodes at depth
 * l * max_depth), their roots and beliefs built on the device, their average strategies written into the handle's compact full-tree
 * strategy, and both best responses taken on it (compute_exploitability2).  br_out2 = {br0, br1}; the exploitability is
 * (br0 + br1) / 2.  subgames, subgame_iters (may be NULL): subgames solved and their CFR iterations; seconds2 (may be NULL): host
 * wall time of the walk and of the best response.  Games with A > CFRB_TO_LEAF_MAX_ACTIONS are refused (CFRB_EINVAL), and so is
 * any call whose cfrb_to_leaf_bytes exceed the device's free memory (CFRB_ENOMEM), before anything is allocated.  Replaces the
 * handle's wave. */
int cfrb_to_leaf_exploitability(cfrb_handle* h, double* br_out2, int64_t* subgames, int64_t* subgame_iters, double* seconds2);
#define CFRB_TO_LEAF_MAX_ACTIONS 23   /* 1x11f; 2x6f (A = 25) would need more than 70 GB */
/* Host-only: device bytes cfrb_to_leaf_exploitability needs beyond the handle of this game, max_depth and max_subgames: the full
 * tree, its two compact strategies and the best-response scratch (none of which a handle that already holds its full tree
 * allocates again), and the walk's template map and two largest levels of roots and beliefs.  Games with A > 26: CFRB_EINVAL. */
int64_t cfrb_to_leaf_bytes(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t max_subgames);
/* Exploitability of the handle's every-node policy (compute_strategy_recursive, recursive_solving.cc:46-74: a subgame of depth
 * max_depth solved for num_iters iterations at every non-terminal node of the full tree, acting with the average strategy of its
 * root), with the handle's weights and solver settings, without a dense strategy: the 2^(A-1) subgames are solved level by level
 * in waves of max_subgames (level d = the C(A - 1, d) non-terminal nodes at depth d, in full-tree order), their root rows written
 * into the handle's compact full-tree strategy, each child's beliefs built on the device (the acting player's row times the child's
 * strategy, eps-normalised; the other row unchanged), and both best responses taken on the strategy (compute_exploitability2).
 * Outputs as cfrb_to_leaf_exploitability's, and refused like it: A > CFRB_TO_LEAF_MAX_ACTIONS, a handle in a live match or agent
 * and null arguments (CFRB_EINVAL), missing weights (CFRB_ESTATE), and a cfrb_recursive_bytes need above the device's free memory
 * (CFRB_ENOMEM, before anything is allocated).  Replaces the handle's wave. */
int cfrb_recursive_exploitability(cfrb_handle* h, double* br_out2, int64_t* subgames, int64_t* subgame_iters, double* seconds2);
/* Host-only: device bytes cfrb_recursive_exploitability needs beyond the handle of this game: cfrb_to_leaf_bytes' full-tree part
 * (none of which a handle that already holds its full tree allocates again) plus the walk, 2 Lmax (4 + 16 H) + 4 (two levels of
 * roots and fp64 beliefs [2][H], Lmax = C(A - 1, floor((A - 1) / 2)), and a level counter); max_subgames does not enter it.  Games
 * with A > 26: CFRB_EINVAL. */
int64_t cfrb_recursive_bytes(int32_t num_dice, int32_t num_faces, int32_t max_subgames);
/* Test aid: the compact full-tree strategy [N_full - 1][H] (entry (child - 1) * H + hand) that the last cfrb_to_leaf_exploitability
 * or cfrb_recursive_exploitability, whichever ran last, filled. */
int cfrb_to_leaf_strategy(cfrb_handle* h, double* compact);
/* Test aid: cfrb_to_leaf_exploitability, cfrb_recursive_exploitability, cfrb_to_leaf_sampled and the strategy-cache check of
 * cfrb_match_create2 (either handle's cap) see at most `bytes` free device bytes (0 = the device's own figure). */
int cfrb_debug_to_leaf_free_cap(cfrb_handle* h, int64_t bytes);
/* recursive_eval's sampled evaluation on the device, for games up to CFRB_TO_LEAF_MAX_ACTIONS: the float32 reach-weighted average
 * of num_repeats sampled recursive strategies (strategy ids seed0 .. seed0 + num_repeats - 1) and its exploitability at every
 * power of two and at num_repeats.  Replaces RecursiveEvaluator::run (recursive_eval.cc:331-369): each repeat is
 * compute_sampled_strategy_recursive_to_leaf (recursive_solving.cc:76-134, 301-327), every subgame solved up to its act_iteration,
 * the k-th draw of std::mt19937(strategy id) for the k-th subgame root in the reference's recursion order, its sampling strategy
 * at that iteration acting; summed_strategy += float(s) * float(reach) and summed_reach += float(reach) in strategy-id order
 * (:138-148, 349-355); final = summed_strategy / (summed_reach + 1e-6) (:362-363); both best responses of it
 * (compute_exploitability2, subgame_solving.cc:802-816).  The subgames of batch_repeats repeats (in [1, max_subgames]) are walked
 * level by level together, in waves of max_subgames rounded down to whole batches.  checkpoints [cap] receives the repeat counts
 * and br_out [cap][2] both best-response values at each.  ev_full (may be null): a dense full-tree strategy [N_full][H][A]; then
 * ev_out [cap][2] receives compute_ev2(ev_full, final) at each checkpoint (:368), and its compact copy ((N_full - 1) H doubles)
 * adds to the device need.  subgames the subgames solved, subgame_iters the sum of their
 * act_iterations, seconds3 the wall time of the draws, the walk and the best responses.  Returns the number of checkpoints.
 * Refused like cfrb_to_leaf_exploitability: A > CFRB_TO_LEAF_MAX_ACTIONS (CFRB_EINVAL), or a cfrb_to_leaf_sampled_bytes need above
 * the free device memory (CFRB_ENOMEM), before anything is allocated.  Replaces the handle's wave and full-tree strategy. */
int cfrb_to_leaf_sampled(cfrb_handle* h, int32_t seed0, int32_t num_repeats, int32_t batch_repeats, int32_t cap, int32_t* checkpoints,
                         double* br_out, const double* ev_full, double* ev_out, int64_t* subgames, int64_t* subgame_iters,
                         double* seconds3);
/* Host-only: device bytes cfrb_to_leaf_sampled needs beyond the handle: cfrb_to_leaf_bytes' full tree, best-response scratch and
 * template map, two levels of roots, fp64 beliefs and fp64 reach for each of batch_repeats repeats, the two float32 accumulators
 * ([N_full - 1][H] and [N_full][H]) and the act_iterations of a batch.  Games with A > 26: CFRB_EINVAL. */
int64_t cfrb_to_leaf_sampled_bytes(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t max_subgames, int32_t batch_repeats);
/* Host-only: the subgame roots of a to-leaf walk (non-terminal nodes of depth l * max_depth), R of them.  level_pos [R] (written
 * when cap >= R) gets, for the k-th root in the reference's recursion order (the order of its act_iteration draws), its position
 * in the device walk's level order over all levels; level_begin [A + 1] (may be null) gets the start of every level, R past the
 * last.  Returns R. */
int cfrb_to_leaf_recursion_order(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t* level_pos, int32_t* level_begin,
                                 int32_t cap);
/* cfrb_to_leaf_sampled with a compact baseline and immediate regrets, for games whose dense [N][H][A] tables do not fit.
 * ev_full_compact (may be NULL): the full-tree strategy compact [N_full - 1][H] fp64 (entry (child - 1) * H + hand); ev_out as in
 * cfrb_to_leaf_sampled.  track_regrets: every repeat's sampled strategy, as float32, goes into compact fp64 regret sums after its
 * batch, in repeat order (RecursiveEvaluator::run's cfrb_regrets_add, bit for bit); at checkpoint c, regret_summary[2c .. 2c+1] =
 * report_regrets' (sum of the immediate regrets of the nodes with depth < regret_depth, of the rest); at the last checkpoint
 * immediate [N_full][H] (may be NULL) gets the immediate regrets, and after the call regret_sums [N_full - 1][H] (may be NULL) the
 * raw sums and regret_count the number of strategies added.  The need check covers cfrb_to_leaf_sampled_regret_bytes more. */
int cfrb_to_leaf_sampled_ev_regrets(cfrb_handle* h, int32_t seed0, int32_t num_repeats, int32_t batch_repeats, int32_t cap,
                                    int32_t* checkpoints, double* br_out, const double* ev_full_compact, double* ev_out,
                                    int32_t track_regrets, int32_t regret_depth, double* regret_summary, double* immediate,
                                    double* regret_sums, int64_t* regret_count, int64_t* subgames, int64_t* subgame_iters,
                                    double* seconds3);
/* Host-only: the device bytes track_regrets adds to a sampled walk: 8 (N - 1) H of sums and 4 (N - 1) H per repeat of a batch.
 * A > CFRB_TO_LEAF_MAX_ACTIONS: CFRB_EINVAL. */
int64_t cfrb_to_leaf_sampled_regret_bytes(int32_t num_dice, int32_t num_faces, int32_t batch_repeats);
/* Host-only: compute_ev2 of two compact full-tree strategies [N_full - 1][H] on the handle's full tree (cfrb_ev2 without the dense
 * tables). */
int cfrb_ev2_compact(cfrb_handle* h, const double* s1, const double* s2, double* out2);
/* Test aids of the last cfrb_to_leaf_sampled: its accumulators, summed_strategy [N_full - 1][H] (entry (child - 1) * H + hand)
 * and summed_reach [N_full][H]; the last repeat's sampled strategy [N_full - 1][H] (fp64) and the act_iteration of every subgame
 * root of that repeat, [N_full] by full-tree node (-1 where no subgame is rooted). */
int cfrb_to_leaf_sampled_sums(cfrb_handle* h, float* summed_strategy, float* summed_reach);
int cfrb_to_leaf_sampled_last(cfrb_handle* h, double* compact, int32_t* act_iteration);

/* ---- Full-game solver: CFR or fictitious play on the whole game tree from the initial state (build_solver(game, params) with an
 * unlimited depth, subgame_solving.h:119-134), the same numbers as a handle whose one subgame is that tree (cfrb_begin_wave at the
 * root with uniform beliefs, cfrb_run, the average strategy of cfrb_fetch, cfrb_exploitability) bit for bit, with the tree's
 * (node, hand) entries spread over the whole device instead of one CTA and no dense [N][H][A] table anywhere, so games up to
 * A = CFRB_TO_LEAF_MAX_ACTIONS (2x5f, 5x2f, 1x10f, 1x11f) fit.  The object owns its tables, the full tree and a stream.
 * cfg: num_dice, num_faces, device, solver, linear_update, dcfr (+ alpha, beta, gamma), optimistic (FP) are read; state_dtype
 * must be CFRB_STATE_F64; max_depth, num_iters, max_subgames, net_mode and hidden are ignored.  Refused before anything is
 * allocated: A > CFRB_TO_LEAF_MAX_ACTIONS (CFRB_EINVAL, checked without a device), and a cfrb_full_game_bytes need above the
 * device's free memory (CFRB_ENOMEM).  Starts at iteration 0 in the state of the CFR constructor (subgame_solving.cc:509-524). */
typedef struct cfrb_full_game cfrb_full_game;
int cfrb_full_game_create(const cfrb_config* cfg, cfrb_full_game** out);
int cfrb_full_game_destroy(cfrb_full_game* g);
/* Host-only: device bytes of a full-game object beyond its handle: the full tree, its compact strategy pair and best-response
 * scratch (cfrb_to_leaf_bytes' tree part), the per-edge tables [N - 1][H] (CFR: regrets, current and sum strategy; FP: average and
 * sum strategy), the per-node reach and values [N][H] and the iteration counter.  solver: CFRB_SOLVER_*.  A > 26: CFRB_EINVAL. */
int64_t cfrb_full_game_bytes(int32_t num_dice, int32_t num_faces, int32_t solver);
/* Run `iters` more iterations (iteration i has traverser i % 2), each one replayed from a CUDA graph of its level launches.
 * Returns when they have finished. */
int cfrb_full_game_step(cfrb_full_game* g, int32_t iters);
/* Iterations done so far; full-tree node count N. */
int cfrb_full_game_iterations(const cfrb_full_game* g);
int cfrb_full_game_nodes(const cfrb_full_game* g);
/* Best-response values {br0, br1} of the current average strategy (compute_exploitability2); the exploitability is their mean. */
int cfrb_full_game_exploitability(cfrb_full_game* g, double* out2);
/* The current average strategy (get_strategy), compact [N - 1][H] fp64 with entry (child - 1) * H + hand. */
int cfrb_full_game_strategy(cfrb_full_game* g, double* compact);
/* Device memory the object took when it was created (the drop of the device's free memory; cudaMalloc rounds up) and the part of
 * it its handle took.  Either pointer may be NULL. */
int cfrb_full_game_memory(const cfrb_full_game* g, int64_t* total_bytes, int64_t* handle_bytes);
/* Test aid: cfrb_full_game_create sees at most `bytes` free device bytes (0 = the device's own figure); process-wide. */
int cfrb_debug_full_game_free_cap(int64_t bytes);
/* Test aid, process-wide: with byte in 0..255, every later floating-point device buffer (fp64, fp32, fp16) the library allocates
 * for a handle or another object is filled with that byte (cudaMemset, then a device-wide synchronise) before it is used, so a
 * result that depends on what fresh device memory held shows up as a difference.  Integer and struct buffers (indices, templates,
 * counters) are never filled.  -1 = off (the default).  Any other value: CFRB_EINVAL, before any device work. */
int cfrb_debug_fill_allocations(int32_t byte);
/* Immediate regrets of the full-game solve (CFR only, as the reference's full-tree solve tracks them): after
 * cfrb_full_game_track_regrets, cfrb_full_game_step adds the sampling strategy after every iteration with an even index to compact
 * fp64 sums [N - 1][H] (entry (child - 1) * H + hand), computed over the whole device.  The sums, immediate regrets and count are
 * bit-identical to cfrb_regrets_add_current after the same iterations of a one-subgame handle.  track_regrets refuses FP
 * (CFRB_EINVAL), an object that has already stepped (CFRB_ESTATE) and a cfrb_full_game_regret_bytes need above the free device
 * memory (CFRB_ENOMEM, before anything is allocated); a second call changes nothing. */
int cfrb_full_game_track_regrets(cfrb_full_game* g);
/* Host-only: the device bytes cfrb_full_game_track_regrets adds, 8 (N - 1) H.  A > CFRB_TO_LEAF_MAX_ACTIONS: CFRB_EINVAL. */
int64_t cfrb_full_game_regret_bytes(int32_t num_dice, int32_t num_faces);
/* immediate [N][H] = cfrb_regrets_fetch's max over the A action slots (0.0 for illegal ones) / count, 0 at leaves; sums [N - 1][H]
 * compact raw; node_sums [N] = per node, the sum of immediate over hands in hand order (report_regrets' inner sum, so the host
 * adds them in node order for its summary); count = strategies added.  Any pointer may be NULL.  Synchronises. */
int cfrb_full_game_regrets(cfrb_full_game* g, double* immediate, double* sums, double* node_sums, int64_t* count);

/* ---- FP subtree forest: eval_net's full-depth solves (stats.cc:118-124) of one depth at once.  Linear fictitious play without a
 * value net on every full-tree subtree rooted at the listed nodes of one depth, each root with its own beliefs: the root value means
 * of a one-subgame wave rooted at that node (cfrb_begin_wave with its last_bid, player and beliefs; solver FP, linear_update,
 * max_depth >= the subtree's depth, no net; cfrb_run(iters); cfrb_fetch's root_value_means) bit for bit, for games up to
 * A = CFRB_TO_LEAF_MAX_ACTIONS.  The object owns an FP full-game solver's tables, the full tree, a stream, the roots' beliefs and
 * means of the largest level and one CUDA graph of an iteration per root depth.  Refused before anything is allocated:
 * A > CFRB_TO_LEAF_MAX_ACTIONS (CFRB_EINVAL, checked without a device) and a cfrb_fp_forest_bytes need above the device's free
 * memory, under the cap of cfrb_debug_full_game_free_cap (CFRB_ENOMEM). */
typedef struct cfrb_fp_forest cfrb_fp_forest;
int cfrb_fp_forest_create(int32_t num_dice, int32_t num_faces, int32_t device, cfrb_fp_forest** out);
int cfrb_fp_forest_destroy(cfrb_fp_forest* f);
/* Host-only: device bytes of a forest beyond its handle: cfrb_full_game_bytes(FP) and the beliefs and means [level][2][H] of the
 * largest depth level of the full tree.  A > CFRB_TO_LEAF_MAX_ACTIONS: CFRB_EINVAL. */
int64_t cfrb_fp_forest_bytes(int32_t num_dice, int32_t num_faces);
/* Host-only: the checks cfrb_fp_forest_solve makes before it touches the device: depth in [1, A - 1], n >= 1, nodes [n] full-tree
 * node ids (BFS order) strictly ascending, all at `depth` and non-terminal; beliefs [n][2][H] finite, non-negative, every row with
 * a positive sum; iters >= 1.  CFRB_EINVAL with the reason when one fails. */
int cfrb_fp_forest_check(int32_t num_dice, int32_t num_faces, int32_t depth, int32_t n, const int32_t* nodes, const double* beliefs,
                         int32_t iters);
/* `iters` iterations (iteration i has traverser i % 2) from the FP constructor of every listed root; root_means [n][2][H] receives
 * each root's root_value_means.  Unlisted nodes of the depth are solved with uniform beliefs and change no listed result. */
int cfrb_fp_forest_solve(cfrb_fp_forest* f, int32_t depth, int32_t n, const int32_t* nodes, const double* beliefs, int32_t iters,
                         double* root_means);
/* Reach statistics of a compact full-tree strategy [N - 1][H] (entry (child - 1) * H + hand) from uniform root beliefs
 * (compute_stategy_stats, subgame_solving.cc:823-846): for the strictly ascending node list nodes [n], node_reach [n] =
 * (sum over hands of player 0's reach) x (the same of player 1's), each sum in hand order, and rows [n][2][H] both players' reach. */
int cfrb_fp_forest_reach(cfrb_fp_forest* f, const double* strategy, int32_t n, const int32_t* nodes, double* node_reach, double* rows);
/* Device memory the forest took when it was created and the part of it its handle took.  Either pointer may be NULL. */
int cfrb_fp_forest_memory(const cfrb_fp_forest* f, int64_t* total_bytes, int64_t* handle_bytes);

/* Immediate-regret accumulator on the handle's device, compute_immediate_regrets (subgame_solving.cc:984-1050) split so that a
 * list of strategies can be added in pieces: adding strategies in batches of any size gives the bits of one pass over the whole
 * list.  Reset zeroes the sums [N_full][H][A] and the count (and must precede the first add). */
int cfrb_regrets_reset(cfrb_handle* h);
/* Add n full-tree strategies, fp32 compact [n][N_full - 1][H] with entry (child_node - 1) * H + hand (the repeats of
 * recursive_eval go through a float32 tensor, recursive_eval.cc:358). */
int cfrb_regrets_add(cfrb_handle* h, const float* compact, int32_t n);
/* Add the handle's current sampling strategy (get_sampling_strategy, read in place on the device).  Subgame 0 of the wave must be
 * the full game tree (max_depth covering the whole game, rooted at the initial state); otherwise CFRB_EINVAL. */
int cfrb_regrets_add_current(cfrb_handle* h);
/* immediate [N_full][H] = max over the A actions of the sums / count (0 at leaves); sums [N_full][H][A] raw, for reductions over
 * processes; count = strategies added.  Any pointer may be NULL.  Synchronises. */
int cfrb_regrets_fetch(cfrb_handle* h, double* immediate, double* sums, int64_t* count);

/* Counters for bench.py: kernels launched by this handle since creation, and leaf rows of the wave. */
int64_t cfrb_kernel_launches(const cfrb_handle* h);
int64_t cfrb_wave_leaf_rows(const cfrb_handle* h);
/* Value-net rows evaluated by this handle since creation (the wave's leaf rows minus those left out as dead, over all iterations);
 * counted where the depth-2 kernel feeds a tensor-core net, CFRB_EINVAL elsewhere. */
int64_t cfrb_net_rows_evaluated(const cfrb_handle* h);
/* Timing marks (benchmarks): record CUDA event `slot` (0..7) on `cuda_stream` (NULL = the handle's stream); device time
 * between two recorded marks (waits for the second). */
int cfrb_mark(cfrb_handle* h, int32_t slot, void* cuda_stream);
int cfrb_mark_elapsed_ms(cfrb_handle* h, int32_t a, int32_t b, float* ms);
int cfrb_mark_wait(cfrb_handle* h, int32_t slot);          /* block until the mark has been reached */
void* cfrb_handle_stream(cfrb_handle* h);                  /* the handle's own cudaStream_t (what NULL stream arguments mean) */
/* Overwrite a scratch buffer of `bytes` on the stream (pass more than the 50 MB of an H100's L2 to evict it between timed steps). */
int cfrb_l2_flush(cfrb_handle* h, size_t bytes, void* cuda_stream);
/* Device time in ms of the most recent cfrb_run, and of its value-net kernels only (CUDA events on
 * the launching stream; valid after cfrb_sync). */
int cfrb_last_run_ms(cfrb_handle* h, float* total_ms, float* net_ms);

/* ---- Device-resident self-play: RlRunner::step (recursive_solving.cc:160-275) for n_games games in lock-step, without host
 * round trips.  Replaces, per wave, RlRunner's act_iteration draw (:168-169), sample_state_to_leaf / sample_state_single
 * (:192-275), normalize_beliefs_inplace (:41-44) and CFR::update_value_network (subgame_solving.cc:672-676).  Game g owns a
 * std::mt19937 seeded with seeds[g] on the device and consumes it in the reference's draw order, so it replays
 * RlRunner(seed = seeds[g]) as long as the solver's strategies agree.  random_action_prob / sample_leaf are
 * RecursiveSolvingParams' fields (recursive_solving.h:31-38). */
int cfrb_selfplay_create(cfrb_handle* h, int32_t n_games, const uint32_t* seeds, float random_action_prob, int32_t sample_leaf);
/* One step of the loop, enqueued asynchronously on `cuda_stream` (NULL = the handle's stream):
 *   1. if a wave is pending: its 2 * n_games training examples are written to the DEVICE buffers dev_ex_q [2n][Q] /
 *      dev_ex_v [2n][H] (both NULL = drop them) and every game samples its next public state (a finished game restarts);
 *   2. if start_next != 0: act_iteration draws, subgame descriptors, CFR constructor and num_iters iterations of the next wave.
 * Returns the number of example rows written (0 or 2 * n_games) or a negative error.
 * A CFR wave started here does not maintain the sum strategy, which the loop never reads.  The readers of it (cfrb_fetch's avg /
 * sum, cfrb_fetch_compact 2 / 4, cfrb_load_state) first rebuild it bit for bit by solving the wave again on the handle's stream,
 * which costs about one wave; they return CFRB_EINVAL instead when cfrb_set_weights has been called since the wave was solved. */
int cfrb_selfplay_wave(cfrb_handle* h, float* dev_ex_q, float* dev_ex_v, int32_t start_next, void* cuda_stream);
/* Block until the examples written by the most recent cfrb_selfplay_wave are complete (the wave it started keeps running). */
int cfrb_selfplay_wait_examples(cfrb_handle* h);
/* Game states (public state and beliefs [n][2][H]) copied to the host; any pointer may be NULL.  Synchronises.  Returns n_games. */
int cfrb_selfplay_state(cfrb_handle* h, int32_t* last_bid, int32_t* player, double* beliefs);
/* Save and restore a self-play session, so that a stopped run continues bit for bit.  The image is a versioned header (magic,
 * format version, num_dice, num_faces, n_games, num_hands, sample_leaf, the bits of random_action_prob, the wave count) followed by
 * every game's beliefs, mt19937 state and index, last bid and player, in host byte order.
 * cfrb_selfplay_export writes the image to `out` (cap bytes) and returns its size; out == NULL only reports the size.  It
 * synchronises.  CFRB_ESTATE without a session or while a wave is pending: drain first with cfrb_selfplay_wave(..., start_next=0).
 * cfrb_selfplay_import installs an image into the session of cfrb_selfplay_create with the same n_games.  The image is checked on
 * the host before the device is touched; a header field that differs from the session (named in the message), a buffer of the
 * wrong size, an mt index outside [0, 624], a player other than 0 / 1, a last bid the walk cannot produce, or a negative or
 * non-finite belief returns CFRB_EINVAL and leaves the session unchanged.  An accepted image is installed between two device-wide
 * synchronisations, so it is ordered after every wave drained on any stream and before the next one.  Afterwards no wave is pending and the handle holds no
 * wave (as after cfrb_create), so readers of a solved wave find none until the next cfrb_selfplay_wave. */
int64_t cfrb_selfplay_export(cfrb_handle* h, void* out, size_t cap);
int cfrb_selfplay_import(cfrb_handle* h, const void* in, size_t bytes);
/* Test aid: the division-free quotient of the regret-matching step (reciprocal of the node's sum + two fused multiply-add
 * corrections, csrc/cfr_kernels.cuh) against IEEE division on blocks x 256 x 4096 pseudo-random operand pairs. */
int cfrb_debug_div_check(cfrb_handle* h, uint64_t seed, int32_t blocks, uint64_t* mismatches);
/* Test aid: the packed-half GELU of the value-net epilogue on every fp16 input: out[i] = fp16 bits of f(fp16 with bit pattern i), i < 65536;
 * what 0 = tanh.approx.f16x2, 1 / 2 = GELU(2 x) computed from x = y / 2 the way the packed-half / fp32-tanh epilogue does (tests pin the arithmetic model of
 * oracle/ref_harness.cc against it). */
int cfrb_debug_gelu_table(cfrb_handle* h, int32_t what, uint16_t* out);
/* Roots (last_bid, player_id) of the subgames of the current wave — also of a wave built on the device by cfrb_selfplay_wave
 * (synchronises then).  Writes min(n, cap) entries, returns n. */
int cfrb_wave_roots(cfrb_handle* h, int32_t* last_bid, int32_t* player_id, int32_t cap);
/* The order in which the depth <= 2 CFR kernel starts the current wave's subgames: wave positions, costliest subgame first
 * (waves of cfrb_begin_wave and cfrb_selfplay_wave), else 0 .. n-1.  Synchronises.  Writes min(n, cap) entries, returns n. */
int cfrb_wave_order(cfrb_handle* h, int32_t* order, int32_t cap);
/* Host only: that order for n subgames rooted at last_bid[] of the game's depth-max_depth trees, and cost[k] (may be NULL), the
 * schedule cost of subgame k: (nodes - 1) x hands table items + pseudo-leaves. */
int cfrb_schedule_order(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t n, const int32_t* last_bid, int32_t* order,
                        int64_t* cost);
/* Test aid: run the depth <= 2 CFR kernel on at most max_ctas CTAs (0 = as many as are resident at once), so that every warp
 * solves many subgames per launch.  Returns the number of CTAs resident at once. */
int cfrb_debug_d2_grid(cfrb_handle* h, int32_t max_ctas);
/* Test aid: wide tickets of the depth <= 2 CFR kernel in the waves that start from now on, the schedule's first m subgames each
 * solved by a whole CTA instead of one warp: -1 = the wave's own rule (default), 0 = none, m > 0 = m (at most the subgames the wave
 * solves).  Waves without a schedule (matches, local best responses, agents) stay narrow. */
int cfrb_debug_d2_wide(cfrb_handle* h, int32_t m);
/* Test aid: the wide tickets the current wave's depth-2 kernel takes (0 when it takes none). */
int cfrb_wave_wide(cfrb_handle* h);
/* Test aid: share = 0 makes the next self-play waves solve every game on its own, instead of solving the games at the initial
 * state (no bid yet, player 0, every belief bitwise 1 / num_hands) once and giving every other one the results (default 1). */
int cfrb_debug_selfplay_share(cfrb_handle* h, int32_t share);
/* The number of subgames the current wave's last solve ran: its size, less all but one of its initial-state games when it is a
 * self-play wave whose initial-state games shared one solve.  A rerun of the wave (cfrb_reset_wave, the rebuild of its sum
 * strategy) solves every game.  Synchronises then. */
int cfrb_wave_solved(cfrb_handle* h);
/* Test aid: skip = 0 makes the value net evaluate every pseudo-leaf row, dead or not, from the next cfrb_set_weights on. */
int cfrb_debug_skip_dead_rows(cfrb_handle* h, int32_t skip);
/* Block until the work enqueued on `cuda_stream` (NULL = the handle's stream) has finished. */
int cfrb_stream_wait(cfrb_handle* h, void* cuda_stream);

/* ---- Head-to-head matches: two agents (an agent = one handle: its solver, iterations, CFR/FP settings and value net) play
 * n_games games of the handles' game against each other on the device, n_slots at a time, one thread per game between waves.
 * Each agent plays its recursive to-leaf strategy restricted to the path played: compute_strategy_recursive_to_leaf
 * (recursive_solving.cc:76-134, policy AVERAGE: all num_iters iterations, get_strategy() acts and propagates beliefs) or
 * compute_sampled_strategy_recursive_to_leaf without root_only (:301-327, policy SAMPLED: per subgame act_iteration ~ weight
 * i/2 + 1 on even i < num_iters, the sampling strategy snapshotted at act_iteration acts and propagates beliefs).  It solves
 * the subgame rooted at the current public node from its own beliefs at the game root and at every pseudo-leaf of its previous
 * subgame, acts for the hand dealt to its seat, and updates both players' beliefs with its own strategy at every node
 * (unnormalised inside a subgame, normalize_beliefs_inplace at its leaves, :41-44).
 * Deals: each seat's hand uniform over the H hands; games 2i and 2i+1 share the hands and swap the agents' seats (agent A sits
 * in seat 0 in even games).  Payoff to A: +1 / -1 at the liar call (the bidder wins iff both hands hold at least the bid's
 * quantity of its face, the last face being wild).  Every draw of game g comes from mt19937 streams keyed by (seed, g) (the
 * deal by (seed, g / 2)), so results do not depend on n_slots.  Slot s plays games s, s + n_slots, ... to their ends.
 * While a match is live its handles serve only the match; afterwards a handle's "current wave" (cfrb_fetch, cfrb_wave_roots,
 * ...) is the last wave the match enqueued, which is empty once every game had finished before it. */
enum {
  CFRB_MATCH_AVERAGE = 0,
  CFRB_MATCH_SAMPLED = 1,
  /* compute_strategy_recursive (recursive_solving.cc:46-74; the policy compute_exploitability_with_net and
   * cfrb_recursive_exploitability measure) restricted to the path played: at EVERY node the agent solves the subgame rooted
   * there from its own beliefs (all num_iters iterations) and acts with the average strategy of that subgame's root.  After each
   * action it multiplies the mover's belief row by its root row and eps-normalises that row (normalize_beliefs_inplace); the
   * other row is unchanged.  Matches with it play one ply per round (cfrb_match_create2). */
  CFRB_MATCH_EVERY_NODE = 2
};
enum { CFRB_MATCH_TRACE_GAMES = 256 };   /* games < min(n_games, this) are traced (cfrb_match_trace) */
typedef struct cfrb_match cfrb_match;
/* a, b: two distinct handles with the same game, max_depth, device and state dtype, max_subgames >= n_slots, no live self-play
 * session or match.  n_games even.  Each violation returns CFRB_EINVAL with a message. */
int cfrb_match_create(cfrb_handle* a, cfrb_handle* b, int32_t n_slots, int32_t n_games, uint64_t seed, int32_t policy, cfrb_match** out);
/* Agent a plays policy_a and agent b policy_b, any pair of the three policies (every-node against to-leaf, AVERAGE against
 * SAMPLED, ...); cfrb_match_create(..., p, ...) is cfrb_match_create2(..., p, p, ...).  A pair of equal to-leaf policies plays
 * the to-leaf walk above, bit for bit.  Any other pair plays the per-ply walk: a round is ONE ply of every running game.  In it
 * each agent solves one wave of the slots where its policy needs a subgame (an every-node agent: every running slot; a to-leaf
 * agent: the slots at the game root or at a pseudo-leaf of its previous subgame), then the mover's agent acts and both agents
 * update their own beliefs.  A to-leaf agent's acting strategy of each solve is copied into a per-slot fp64 cache right after
 * the solve: n_slots x E x H x 8 bytes per to-leaf agent (E: the edges of the largest depth-max_depth template; about 0.7 GB for
 * 8192 slots at 2x6f), see cfrb_match_cache_bytes.  It is refused with CFRB_ENOMEM and its byte count when it exceeds the free
 * device memory (or either handle's cfrb_debug_to_leaf_free_cap), before anything is allocated.  Draws of game g come from its
 * (seed, g) streams in a fixed order per ply (agent a's act_iteration when it starts a SAMPLED subgame, then b's, then the
 * action), so results do not depend on n_slots.  In a per-ply match cfrb_match_trace's rounds are plies: act_iterations[r][k] is
 * -1 when agent k solved with AVERAGE or EVERY_NODE at ply r, its draw for a SAMPLED solve, and -2 when it did not solve (it
 * plays on inside its to-leaf subgame); root_beliefs[r][k] are agent k's beliefs at ply r in every case.  cfrb_match_results'
 * solves and subgame_iters count each agent's actual solves.  Validation as cfrb_match_create's, plus a bad policy value. */
int cfrb_match_create2(cfrb_handle* a, cfrb_handle* b, int32_t n_slots, int32_t n_games, uint64_t seed, int32_t policy_a,
                       int32_t policy_b, cfrb_match** out);
/* Host-only: device bytes of the strategy caches cfrb_match_create2 allocates for a match of this game, max_depth, n_slots and
 * pair of policies (0 for the to-leaf walk and for two every-node agents). */
int64_t cfrb_match_cache_bytes(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t n_slots, int32_t policy_a,
                               int32_t policy_b);
/* Enqueue max_rounds rounds on `cuda_stream` (NULL = a's stream); a round is one wave of num_iters iterations per agent (the
 * subgames of every running game, built on the device) and one walk.  Returns max_rounds, or 0 once every game has finished
 * (learned from the previous call's rounds, without further work). */
int cfrb_match_run(cfrb_match* m, int32_t max_rounds, void* cuda_stream);
/* Synchronises.  payoff_a [n_games] (0 for a game not finished yet), plies [n_games]; solves = subgames solved by both agents;
 * subgame_iters = CFR / FP iterations run for them.  Any pointer may be NULL. */
int cfrb_match_results(cfrb_match* m, float* payoff_a, int32_t* plies, int64_t* solves, int64_t* subgame_iters);
/* Synchronises.  solves [2]: subgames agent a and agent b solved (an LBR match: the agent's, and 0 for LBR). */
int cfrb_match_agent_solves(cfrb_match* m, int64_t* solves);
/* Synchronises.  Trace of one game < min(n_games, CFRB_MATCH_TRACE_GAMES); returns its number of plies P (<= A).
 *   ply_records [A][6]  per ply: agent that acted (0 = a), last bid before the action, acting player (seat), its hand, action,
 *                       subgame (round) index within the game
 *   probs [A]           fp64 probability of that action in the acting agent's strategy
 *   act_iterations [A][2], root_beliefs [A][2][2][H]: per subgame r < *n_rounds, each agent's act_iteration (-1 = AVERAGE) and
 *                       root beliefs [player][hand] (fp64, before the conversion to the state dtype)
 * Any pointer may be NULL. */
int cfrb_match_trace(cfrb_match* m, int32_t game, int32_t* ply_records, double* probs, int32_t* act_iterations, double* root_beliefs,
                     int32_t* n_rounds);
int cfrb_match_destroy(cfrb_match* m);

/* ---- Blueprints: fixed full-tree strategies as players.  A blueprint is a compact fp64 table [N - 1][H] over the full game
 * tree (entry (child - 1) * H + hand, the layout of cfrb_full_game_strategy, cfrb_to_leaf_strategy and cfrb_ev2_compact) held on
 * one device with the full tree's child_begin [N] and the game's match counts [H][F].  It never solves: at a public node it acts
 * with the row of that node's edges for its hand.  Games with A > CFRB_TO_LEAF_MAX_ACTIONS have none (CFRB_EINVAL, checked
 * without a device).  A blueprint is read-only; it must outlive every match that plays it, and any number of matches may. */
typedef struct cfrb_blueprint cfrb_blueprint;
/* Host-only: device bytes of a blueprint, 8 (N - 1) H + 4 N + H F with N = 2^A - 1 full-tree nodes (2x4f: 17 MB, 2x5f: 0.43 GB,
 * 5x2f: 0.55 GB, 1x11f: 0.77 GB). */
int64_t cfrb_blueprint_bytes(int32_t num_dice, int32_t num_faces);
/* Host-only: the checks of cfrb_blueprint_create on a host table, each refused with CFRB_EINVAL and a message naming the first
 * bad node and hand (full-tree BFS order, hands innermost): a non-finite or negative entry, or a (node, hand) row whose sum over
 * the node's children is more than 1e-6 away from 1. */
int cfrb_blueprint_check(int32_t num_dice, int32_t num_faces, const double* compact);
/* Upload a host table to `device` after cfrb_blueprint_check's checks.  A cfrb_blueprint_bytes need above the device's free
 * memory is refused with CFRB_ENOMEM before anything is allocated. */
int cfrb_blueprint_create(int32_t device, int32_t num_dice, int32_t num_faces, const double* compact, cfrb_blueprint** out);
/* The solver's current average strategy, copied on its device: bit for bit what cfrb_full_game_strategy returns. */
int cfrb_blueprint_from_full_game(cfrb_full_game* g, cfrb_blueprint** out);
/* The full-tree strategy the handle's last to-leaf or every-node walk filled, copied on its device: bit for bit what
 * cfrb_to_leaf_strategy returns.  CFRB_ESTATE when the handle holds none. */
int cfrb_blueprint_from_handle(cfrb_handle* h, cfrb_blueprint** out);
/* Synchronises.  The table, compact [N - 1][H]. */
int cfrb_blueprint_strategy(const cfrb_blueprint* b, double* compact);
int cfrb_blueprint_destroy(cfrb_blueprint* b);

/* One seat of cfrb_match_create3: a handle playing `policy` (CFRB_MATCH_*), or a blueprint (h NULL; policy is not read). */
typedef struct cfrb_match_agent {
  cfrb_handle* h;
  cfrb_blueprint* bp;
  int32_t policy;
} cfrb_match_agent;
/* A match in which either seat, or both, may be a blueprint.  Without a blueprint it is cfrb_match_create2(a.h, b.h, ...,
 * a.policy, b.policy).  With one it plays the per-ply walk of cfrb_match_create2: a blueprint solves nothing and keeps no beliefs;
 * it holds the full-tree node of each game (the root at the deal, child_begin[node] + j after action j) and acts there with its
 * table's row.  Its draws are the action draws of the game's (seed, g) stream at the point where any other policy draws, and it
 * draws no act_iteration, so a blueprint holding the table an AVERAGE or EVERY_NODE agent acts with plays that agent's games bit
 * for bit.  A match of two blueprints needs no handle: it runs walk kernels only, on a stream of its own.  The agents must play
 * the same game on the same device; a handle agent is refused as in cfrb_match_create2 (capacity, live session or match, bad
 * policy, its strategy cache above the free memory: CFRB_ENOMEM).  cfrb_match_run / _results / _agent_solves / _trace /
 * _destroy apply: a blueprint's solves are 0, its act_iterations trace entry is -2 on every ply and its traced beliefs stay
 * uniform. */
int cfrb_match_create3(const cfrb_match_agent* a, const cfrb_match_agent* b, int32_t n_slots, int32_t n_games, uint64_t seed,
                       cfrb_match** out);
/* Local best response against a blueprint: LBR's rule is exactly cfrb_match_create_lbr's, with sigma(child(a)) and every update of
 * beta read from the blueprint's table, so there are no what-if solves and no solves at all.  A round plays every running slot's
 * game to its end (walk kernels only, on a stream of the match's own).  Seats, deals and the agent's draws are a match's; a
 * blueprint holding the table of an AVERAGE or EVERY_NODE agent's walked policy gives cfrb_match_create_lbr2's payoffs and LBR
 * trace for that agent bit for bit.  cfrb_match_run / _results / _trace / _lbr_trace / _lbr_counts / _destroy apply: solves and
 * whatif_solves are 0, and every traced ply has round 0. */
int cfrb_match_create_lbr_blueprint(cfrb_blueprint* bp, int32_t n_slots, int32_t n_games, uint64_t seed, cfrb_match** out);

/* ---- Local best response (Lisy & Bowling, 2017): a lower bound on one agent's exploitability on any game.  The agent (one
 * handle) plays as in a CFRB_MATCH_AVERAGE match against LBR, which best-responds one decision at a time: with its fp64 belief
 * beta over the agent's hand (uniform, times the agent's strategy after every agent action, renormalised) it plays the argmax
 * (ties: the smallest action) of
 *   liar (b >= 0):  sum_h beta[h] (b true ? -1 : +1)
 *   raise a:        sum_h beta[h] sum_{a' legal after a, liar last} sigma(child(a), h, a') (a' liar ? (a true ? +1 : -1)
 *                                                                                     : (a' true ? -1 : +1))
 * (a bid is true for agent hand h when LBR's and h's matches of its face reach its quantity; every raise of the agent is
 * assumed to be called).  sigma(child(a)) comes from the agent's current subgame, or, when child(a) is a pseudo-leaf of it,
 * from the root of the agent's subgame at child(a) solved from its beliefs propagated through its own strategy ("what-if"
 * solves, one per raise; the chosen one is the agent's next subgame).  Seats, deals and the agent's draws are those of
 * cfrb_match_create: the agent sits in seat 0 in even games.  A round solves at most max_subgames subgames: running games ask
 * for 1 subgame (game start, pseudo-leaf) or m (an LBR decision with m raises) and are admitted round-robin; the others wait.
 * cfrb_match_run / _results / _trace / _destroy apply: payoff_a is the agent's payoff (LBR's is its negative), solves counts
 * every subgame solved, what-if ones included; in the trace agent 1 is LBR (probability 1, act_iteration and root beliefs 0).
 * agent: max_subgames >= A - 1, no live self-play session or match; n_games even.  Each violation returns CFRB_EINVAL.
 * cfrb_match_create_lbr(...) is cfrb_match_create_lbr2(..., CFRB_MATCH_AVERAGE, ...). */
int cfrb_match_create_lbr(cfrb_handle* agent, int32_t n_slots, int32_t n_games, uint64_t seed, cfrb_match** out);
/* LBR against the agent playing `policy`: CFRB_MATCH_AVERAGE (the walk above, bit for bit) or CFRB_MATCH_EVERY_NODE.  The
 * every-node agent plays as in a per-ply cfrb_match_create2 match: it solves at every node of the path, whoever moves, and acts
 * and updates the mover's belief row with that subgame's root row.  The LBR rule is unchanged; sigma(child(a)) is always the
 * root row of a what-if solve at child(a).  At an LBR decision at node X with m > 0 legal raises a slot takes two rounds:
 *   phase 1   one subgame rooted at X from the agent's beliefs (its root row is how the agent updates LBR's row)
 *   phase 2   m what-if subgames rooted at the children: the agent's own row, and LBR's row times X's root row for that raise,
 *             eps-normalised
 * then LBR decides.  After a raise the chosen what-if is the agent's subgame at child(a), not solved again: the agent acts from
 * its root row, and the slot waits for phase 1 at LBR's next decision.  At bid A - 2 LBR has no raise and calls without a
 * solve; an agent moving first solves at the game root and acts.  Counts: solves = phase 1 + what-if + game-root solves, i.e.
 * per game the sum over LBR decisions with m > 0 of (1 + m), plus 1 where the agent moves first; whatif_solves (cfrb_match_lbr_counts)
 * = the sum of m.  In cfrb_match_trace a round is a node of the path where the agent solved a subgame it acts or updates
 * beliefs from (the game root when it moves first, each phase 1, each chosen what-if): root_beliefs are its beliefs there, and
 * each ply carries the round of its node (LBR's call after bid A - 2: the round of the agent's ply before it).
 * CFRB_MATCH_SAMPLED (LBR would respond to a drawn snapshot the agent's opponent cannot see, so the payoff bounds nothing) and
 * unknown values return CFRB_EINVAL with a message; other validation as cfrb_match_create_lbr's. */
int cfrb_match_create_lbr2(cfrb_handle* agent, int32_t n_slots, int32_t n_games, uint64_t seed, int32_t policy, cfrb_match** out);
/* Synchronises.  For a traced game: per ply where LBR acted, values [A][A] (fp64 value of every action, NaN where illegal and on
 * the agent's plies) and beliefs [A][H] (beta before the decision, 0 on the agent's plies).  Returns the number of plies. */
int cfrb_match_lbr_trace(cfrb_match* m, int32_t game, double* values, double* beliefs);
/* Synchronises.  what-if subgames solved, and running slots that waited a round for capacity (summed over rounds). */
int cfrb_match_lbr_counts(cfrb_match* m, int64_t* whatif_solves, int64_t* deferred_slot_rounds);

/* ---- A ReBeL agent played from outside: one handle's agent at n_tables independent tables, each a game against an external
 * player (a person, another program's bot, a tournament harness), advanced one action per call.  At every table the agent plays
 * as in a cfrb_match_* match: compute_strategy_recursive_to_leaf (policy CFRB_MATCH_AVERAGE),
 * compute_sampled_strategy_recursive_to_leaf without root_only (CFRB_MATCH_SAMPLED, recursive_solving.cc:76-134, 301-327) or
 * compute_strategy_recursive (CFRB_MATCH_EVERY_NODE, :46-74) restricted to the path played.  An every-node agent stands at an
 * unsolved subgame root at every node: each step or policy at a table first solves the subgame at the table's current node,
 * whoever is to move, and the cache holds that root row; after every action (its own or an observed opponent's) the mover's row
 * is multiplied by the agent's root row and eps-normalised.  The to-leaf policies:  It solves the subgame rooted at the current public node from its own beliefs at the game root
 * and at every pseudo-leaf of its previous subgame, acts for its hand, and updates both players' beliefs with its own strategy,
 * whoever acts (unnormalised inside a subgame, normalize_beliefs_inplace at its leaves, :41-44).  An opponent action the agent's
 * strategy gives probability 0 is applied all the same: it zeroes that row's beliefs and the eps-normalisation at the next
 * subgame root decides, as in the reference.
 * Deals and seats belong to the caller: the agent only ever sees its own hand.  The payoff is the caller's business too.
 * Table t's random draws (act_iteration, the agent's actions) come from mt19937(match_stream_seed(seed, key, 3)) where key is the
 * game's key, so a game's draws depend only on (seed, key): not on the table, the batch, or the order of the calls.
 * step / policy solve every listed table that stands at an unsolved subgame root in ONE wave of the handle (its CUDA graph of
 * num_iters iterations), packed in list order.  Since wave positions change from call to call, each solved subgame's acting
 * strategy (the normalised average of CFR, the average of FP, or the act_iteration snapshot) is copied into a per-table fp64
 * cache right after the solve; everything later reads the cache only.
 * Every call checks the whole batch on the host first and then synchronises; a table's error (id out of range or repeated, a hand
 * outside [0, H), an action that is not above the last bid or a liar call before any bid, -1 on the opponent's turn, a table with
 * no running game) returns CFRB_EINVAL with the table id in the message and leaves every table of the call unchanged.
 * h: max_subgames >= n_tables, no live self-play session or match; while the agent lives the handle serves only it (it counts as
 * in a live match).  The caller keeps the handle and destroys it after the agent. */
typedef struct cfrb_agent cfrb_agent;
int cfrb_agent_create(cfrb_handle* h, int32_t n_tables, uint64_t seed, int32_t policy, cfrb_agent** out);
/* An agent that plays a blueprint: step, policy and state answer from its table at the full-tree node of each table, its draws
 * are the (seed, key) streams of cfrb_agent_create's agents, and it never solves (subgames 0, act_iteration -1, root beliefs
 * uniform, counts 0).  A blueprint holding an AVERAGE agent's walked to-leaf policy answers as that agent, bit for bit.  It has
 * no handle and runs on a stream of its own; the blueprint must outlive it. */
int cfrb_agent_create_blueprint(cfrb_blueprint* bp, int32_t n_tables, uint64_t seed, cfrb_agent** out);
/* Start (or restart) a game at each listed table: the agent sits in seat seats[i] (0 moves first) with hand hands[i].  keys[i]
 * keys the game's stream; keys NULL: the number of games this agent had started before, counted in list order. */
int cfrb_agent_new_games(cfrb_agent* a, int32_t n, const int32_t* ids, const int32_t* seats, const int32_t* hands, const uint64_t* keys);
/* One action at each listed table.  actions[i] in: the action to apply (normally the opponent's; on the agent's own turn it
 * overrides the agent's choice, e.g. to replay a logged game), or -1 = the agent draws its action for its hand (its turn only);
 * out: the action played.  probs [n][A] (may be NULL): on the agent's turns its probability row for its hand (0 on illegal
 * actions), NaN on the opponent's.  done[i] = 1 when the action was the liar call (the table's game is over). */
int cfrb_agent_step(cfrb_agent* a, int32_t n, const int32_t* ids, int32_t* actions, double* probs, int32_t* done);
/* The agent's strategy for the player to move at each listed table, out [n][H][A] (0 on illegal actions). */
int cfrb_agent_policy(cfrb_agent* a, int32_t n, const int32_t* ids, double* out);
/* Any pointer may be NULL.  Public node (last bid, player to move, plies so far), subgames solved in the current game, the
 * act_iteration of the current subgame (-1: AVERAGE), and its root beliefs [n][2][H] (fp64, before the conversion to the state
 * dtype; at a table that waits for a solve, the beliefs of the subgame it will solve). */
int cfrb_agent_state(cfrb_agent* a, int32_t n, const int32_t* ids, int32_t* last_bid, int32_t* player, int32_t* ply, int32_t* subgames,
                     int32_t* act_iteration, double* root_beliefs);
/* Subgames solved since creation and the iterations run for them. */
int cfrb_agent_counts(cfrb_agent* a, int64_t* solves, int64_t* subgame_iters);
/* Device time in ms of the solves (subgame initialisation and iterations, CUDA events) since creation. */
int cfrb_agent_solve_ms(cfrb_agent* a, double* ms);
int cfrb_agent_destroy(cfrb_agent* a);

/* ---- Device-resident example rows: storage of the replay buffer (rela/prioritized_replay.h:224-506 keeps one pair of host
 * tensors per example; here the rows of the ring live in HBM as two [capacity][dim] fp32 matrices and never visit the host on
 * their way from the generator kernels to the trainer's batch).  Bookkeeping (head, size, priorities, blocking) stays with the
 * caller. */
typedef struct cfrb_rows cfrb_rows;
int cfrb_rows_create(int32_t device, int64_t capacity_rows, int32_t q_dim, int32_t v_dim, cfrb_rows** out);
int cfrb_rows_destroy(cfrb_rows* r);
int cfrb_rows_device(const cfrb_rows* r);
/* Store n rows at ring position `slot` (wraps around).  kind 0: q / v are host pointers; kind 1: device pointers on CUDA
 * device src_device (peer copy when that is another GPU).  Returns when the rows are in place. */
int cfrb_rows_write(cfrb_rows* r, int64_t slot, int32_t n, const float* q, const float* v, int32_t kind, int32_t src_device);
/* n rows starting at `slot` (wraps around) to host memory (save / extract). */
int cfrb_rows_read(cfrb_rows* r, int64_t slot, int32_t n, float* q, float* v);
/* Batch assembly (PrioritizedReplay::sample -> makeBatch, rela/types.cc:19-41): rows ids[0..n) gathered into out_q [n][q_dim] /
 * out_v [n][v_dim] on out_device (CUDA ordinal, -1 = host memory).  On the ring's own device the gather kernel runs on
 * `cuda_stream` (the consumer's stream). */
int cfrb_rows_gather(cfrb_rows* r, const int32_t* ids, int32_t n, float* out_q, float* out_v, int32_t out_device, void* cuda_stream);
/* Device scratch for the hand-over of one wave's examples from a generator handle to a row store. */
int cfrb_dev_alloc(int32_t device, size_t bytes, void** out);
int cfrb_dev_free(int32_t device, void* p);
int cfrb_dev_to_host(int32_t device, void* dst, const void* src, size_t bytes);

/* ---- Value-net training: one optimisation step of the reference trainer (cfvpy/selfplay.py:409-438) for the net the kernels
 * evaluate, Net2(n_hidden=256, n_layers=2, use_layer_norm=True), on a batch of n <= max_batch examples: forward (Linear ->
 * LayerNorm(eps 1e-5) -> erf GELU, twice, then Linear), the loss averaged over the H outputs and then over the batch
 * (selfplay.py:135-149), backward through every parameter, clip_grad_norm_ (selfplay.py:636-651: total = 2-norm of the
 * per-parameter 2-norms, gradients scaled by max_norm / (total + 1e-6) when that is < 1; max_norm <= 0 = no clipping) and
 * torch.optim.Adam with its defaults (betas 0.9 / 0.999, eps 1e-8, no weight decay, bias correction).  fp32 operands and
 * accumulation, no atomics: the same state and batch give the same bits on every run, eagerly or replayed from a CUDA graph.
 * The trainer owns its parameters, gradients, Adam moments, step count and scratch on one device; a trainer is not thread-safe,
 * and since steps and losses share its scratch, all calls on one trainer must be ordered: enqueue them on one stream, or order
 * the streams (events) yourself.
 * Parameters and moments cross the boundary as flat fp32 buffers in the cfrb_set_weights layout. */
typedef struct cfrb_trainer cfrb_trainer;
enum {
  CFRB_LOSS_HUBER = 0,   /* (|x| > 1)(2|x| - 1) + (|x| <= 1) x^2 of x = values - net(query) */
  CFRB_LOSS_MSE = 1      /* x^2 */
};
/* Parameters, moments and step count start at zero (cfrb_trainer_set_state installs a net). */
int cfrb_trainer_create(int32_t device, int32_t num_dice, int32_t num_faces, int32_t max_batch, cfrb_trainer** out);
int cfrb_trainer_destroy(cfrb_trainer* t);
/* Number of floats of the flat parameter buffer (= of each Adam moment). */
int64_t cfrb_trainer_num_params(const cfrb_trainer* t);
/* Host buffers of cfrb_trainer_num_params floats; m / v NULL = zero moments.  step = Adam steps already taken.  Synchronises
 * the device. */
int cfrb_trainer_set_state(cfrb_trainer* t, const float* params, const float* m, const float* v, int64_t step);
/* Any pointer may be NULL.  Synchronises the device. */
int cfrb_trainer_get_state(cfrb_trainer* t, float* params, float* m, float* v, int64_t* step);
/* One step on the batch dev_q [n][Q], dev_v [n][H] (row-major fp32, memory of the trainer's device), enqueued on `cuda_stream`
 * (a cudaStream_t; NULL = the legacy default stream) with no host<->device copy and no synchronisation.  lr is the learning rate
 * of this step (the host halves it on its schedule).  dev_out (device memory, may be NULL) receives {loss, pre-clip grad norm,
 * loss of row 0, .., loss of row n-1} (row loss = mean over the H outputs) once the stream gets there.  Arguments are checked
 * before anything is enqueued: a refused call leaves the trainer unchanged. */
int cfrb_trainer_step(cfrb_trainer* t, const float* dev_q, const float* dev_v, int32_t n, double lr, double max_norm, int32_t loss_kind,
                      void* cuda_stream, float* dev_out);
/* Forward pass and loss only (validation sets), on `cuda_stream`: dev_out [2 + n] receives {loss, unused, row losses}. */
int cfrb_trainer_loss(cfrb_trainer* t, const float* dev_q, const float* dev_v, int32_t n, int32_t loss_kind, void* cuda_stream,
                      float* dev_out);
/* Loss and pre-clip grad norm of the most recent cfrb_trainer_step.  Synchronises the device. */
int cfrb_trainer_last(cfrb_trainer* t, float* loss, float* grad_norm);
/* Test aid: the gradients of the most recent step after clipping, flat [cfrb_trainer_num_params].  Synchronises the device. */
int cfrb_trainer_debug_grads(cfrb_trainer* t, float* out);

/* ---- One process per GPU: the two hand-overs the reference performs through shared host memory inside ONE process become NCCL
 * collectives over NVLink, issued by this library on device buffers (no torch.distributed, no host bounce):
 *   ModelLocker::updateModel (rela/model_locker.h:69-79)         -> cfrb_comm_broadcast_weights
 *   PrioritizedReplay::add   (rela/prioritized_replay.h:247-261) -> cfrb_comm_gather_rows into the trainer rank's device rows
 *   recursive_eval's float32 accumulation (recursive_eval.cc:343-363) -> cfrb_comm_reduce_sum
 * The 128-byte id is created on one rank (cfrb_comm_unique_id) and handed to the others by the launcher (e.g. through the
 * torchrun store); every function is a collective: all ranks of the communicator call it, in the same order. */
typedef struct cfrb_comm cfrb_comm;
int cfrb_comm_unique_id(uint8_t* out128);
int cfrb_comm_create(const uint8_t* id128, int32_t rank, int32_t world, int32_t device, cfrb_comm** out);
int cfrb_comm_destroy(cfrb_comm* c);
int cfrb_comm_rank(const cfrb_comm* c);
int cfrb_comm_world(const cfrb_comm* c);
/* flat fp32 weights (cfrb_set_weights layout): read from the root's host buffer, delivered to every other rank.  cuda_stream NULL:
 * the communicator's own stream, the call waits and the other ranks' flat_host is filled.  Otherwise the H2D copy (root), the
 * ncclBroadcast and the D2H copy (others) are only ENQUEUED on that stream (a generator loop puts them between two waves); the
 * other ranks pass flat_host = NULL and read the weights with cfrb_comm_broadcast_fetch once the stream has passed that point. */
int cfrb_comm_broadcast_weights(cfrb_comm* c, float* flat_host, size_t n, int32_t root, void* cuda_stream);
int cfrb_comm_broadcast_fetch(cfrb_comm* c, float* out_host, size_t n);
/* every rank contributes n rows from DEVICE buffers dev_q [n][q_dim], dev_v [n][v_dim]; on the root they arrive in rank order in
 * the DEVICE buffers recv_q [world * n][q_dim], recv_v [world * n][v_dim] (ignored elsewhere).  cuda_stream NULL: the communicator's
 * own stream, the call waits; otherwise the send / recv are only ENQUEUED on that stream — a generator loop puts them between two
 * waves on its handle's stream, where the GPU has nothing else to run and they cost microseconds instead of competing with a
 * wave's kernels for SMs. */
int cfrb_comm_gather_rows(cfrb_comm* c, const float* dev_q, const float* dev_v, int32_t n, int32_t q_dim, int32_t v_dim, float* recv_q,
                          float* recv_v, int32_t root, void* cuda_stream);
/* agreement between generator loops that must issue the same collectives in the same order ("stop after this wave", "the trainer
 * rank has weights version v"): every rank contributes n <= 4 ints, all ranks obtain the element-wise maximum; enqueued on
 * cuda_stream like cfrb_comm_gather_rows, read with cfrb_comm_vote_result once that point is reached. */
int cfrb_comm_vote(cfrb_comm* c, const int32_t* values, int32_t n, void* cuda_stream);
int cfrb_comm_vote_result(cfrb_comm* c, int32_t* out, int32_t n);
/* in-place float32 sum over the ranks of a DEVICE buffer, result on the root. */
int cfrb_comm_reduce_sum(cfrb_comm* c, float* dev_buf, size_t n, int32_t root);

#ifdef __cplusplus
}
#endif
#endif /* CFRB200_H_ */
