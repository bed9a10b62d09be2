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
  CFRB_NET_TC_F16X2 = 3   /* same kernel with the fast GELU: y/2 (1 + tanh(poly)) with packed f32x2 FMAs and tanh.approx.f32, one
                             rounding to fp16 at the end (same accuracy as mode 2, 1 instead of 2 MUFU operations per element).
                             CFRB_X2_GELU=half selects the packed-fp16 evaluation (HFMA2 + tanh.approx.f16x2): 6 % faster, but
                             that instruction truncates towards zero and biases every activation (see DESIGN.md "P5") */
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

/* Shape queries. */
int cfrb_num_actions(const cfrb_handle* h);   /* A */
int cfrb_num_hands(const cfrb_handle* h);     /* H */
int cfrb_query_size(const cfrb_handle* h);    /* Q */
int cfrb_max_nodes(const cfrb_handle* h);     /* Nmax over all root templates */

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
 * writes at most cap_rows. */
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
/* Test aid: the compact full-tree strategy [N_full - 1][H] (entry (child - 1) * H + hand) the last cfrb_to_leaf_exploitability
 * filled. */
int cfrb_to_leaf_strategy(cfrb_handle* h, double* compact);
/* Test aid: cfrb_to_leaf_exploitability sees at most `bytes` free device bytes (0 = the device's own figure). */
int cfrb_debug_to_leaf_free_cap(cfrb_handle* h, int64_t bytes);

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
  CFRB_MATCH_SAMPLED = 1
};
enum { CFRB_MATCH_TRACE_GAMES = 256 };   /* games < min(n_games, this) are traced (cfrb_match_trace) */
typedef struct cfrb_match cfrb_match;
/* a, b: two distinct handles with the same game, max_depth, device and state dtype, max_subgames >= n_slots, no live self-play
 * session or match.  n_games even.  Each violation returns CFRB_EINVAL with a message. */
int cfrb_match_create(cfrb_handle* a, cfrb_handle* b, int32_t n_slots, int32_t n_games, uint64_t seed, int32_t policy, cfrb_match** out);
/* Enqueue max_rounds rounds on `cuda_stream` (NULL = a's stream); a round is one wave of num_iters iterations per agent (the
 * subgames of every running game, built on the device) and one walk.  Returns max_rounds, or 0 once every game has finished
 * (learned from the previous call's rounds, without further work). */
int cfrb_match_run(cfrb_match* m, int32_t max_rounds, void* cuda_stream);
/* Synchronises.  payoff_a [n_games] (0 for a game not finished yet), plies [n_games]; solves = subgames solved by both agents;
 * subgame_iters = CFR / FP iterations run for them.  Any pointer may be NULL. */
int cfrb_match_results(cfrb_match* m, float* payoff_a, int32_t* plies, int64_t* solves, int64_t* subgame_iters);
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
 * agent: max_subgames >= A - 1, no live self-play session or match; n_games even.  Each violation returns CFRB_EINVAL. */
int cfrb_match_create_lbr(cfrb_handle* agent, int32_t n_slots, int32_t n_games, uint64_t seed, cfrb_match** out);
/* Synchronises.  For a traced game: per ply where LBR acted, values [A][A] (fp64 value of every action, NaN where illegal and on
 * the agent's plies) and beliefs [A][H] (beta before the decision, 0 on the agent's plies).  Returns the number of plies. */
int cfrb_match_lbr_trace(cfrb_match* m, int32_t game, double* values, double* beliefs);
/* Synchronises.  what-if subgames solved, and running slots that waited a round for capacity (summed over rounds). */
int cfrb_match_lbr_counts(cfrb_match* m, int64_t* whatif_solves, int64_t* deferred_slot_rounds);

/* ---- A ReBeL agent played from outside: one handle's agent at n_tables independent tables, each a game against an external
 * player (a person, another program's bot, a tournament harness), advanced one action per call.  At every table the agent plays
 * as in a cfrb_match_* match: compute_strategy_recursive_to_leaf (policy CFRB_MATCH_AVERAGE) or
 * compute_sampled_strategy_recursive_to_leaf without root_only (CFRB_MATCH_SAMPLED, recursive_solving.cc:76-134, 301-327)
 * restricted to the path played.  It solves the subgame rooted at the current public node from its own beliefs at the game root
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
