// libcfrb200.so — C ABI implementation (include/cfrb200.h) of the H100 CFR wave solver.
// Plain CUDA runtime; no torch, no CPU fallback: every entry point that computes needs the device.
#include "../../include/cfrb200.h"

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <array>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "cfr_types.h"
#include "cfr_tree.h"
#include "leaf_mlp_simt.cuh"
#include "leaf_mlp_tc.cuh"
#include "leaf_mlp_tc_wide.cuh"
#include "train_kernels.cuh"

namespace {
inline bool is_tc(int net_mode) { return net_mode == CFRB_NET_TC_F16 || net_mode == CFRB_NET_TC_F16X2; }

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t e__ = (call);                                                                      \
    if (e__ != cudaSuccess)                                                                        \
      return fail(CFRB_ECUDA, std::string(#call) + ": " + cudaGetErrorString(e__) + " @" + __FILE__ + ":" + \
                                  std::to_string(__LINE__));                                       \
  } while (0)

// Device memory of `n` elements, freed with its owner.  alloc() frees what the buffer held before.
template <class T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), n(std::exchange(o.n, 0)) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { free(); p = std::exchange(o.p, nullptr); n = std::exchange(o.n, 0); }
    return *this;
  }
  ~DevBuf() { free(); }
  cudaError_t alloc(size_t count) {
    free();
    const cudaError_t e = cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
    if (e == cudaSuccess) n = count;
    else p = nullptr;
    return e;
  }

 private:
  void free() { if (p) cudaFree(p); p = nullptr; n = 0; }
};
static_assert(!std::is_copy_constructible_v<DevBuf<int>>);

// Any other CUDA (or NCCL) handle, destroyed with its owner.  put() hands the slot to a create call.
template <class T, auto Destroy>
class Owner {
 public:
  Owner() = default;
  explicit Owner(T v) : v_(v) {}
  Owner(const Owner&) = delete;
  Owner& operator=(const Owner&) = delete;
  Owner(Owner&& o) noexcept : v_(std::exchange(o.v_, T{})) {}
  Owner& operator=(Owner&& o) noexcept {
    if (this != &o) { destroy(); v_ = std::exchange(o.v_, T{}); }
    return *this;
  }
  ~Owner() { destroy(); }
  T* put() { destroy(); return &v_; }
  T get() const { return v_; }
  operator T() const { return v_; }

 private:
  void destroy() { if (v_) Destroy(v_); v_ = T{}; }
  T v_{};
};
template <class T> using Pinned = Owner<T*, cudaFreeHost>;
using Event = Owner<cudaEvent_t, cudaEventDestroy>;
using Stream = Owner<cudaStream_t, cudaStreamDestroy>;
using Graph = Owner<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Owner<cudaGraphExec_t, cudaGraphExecDestroy>;

inline int round_up(int x, int m) { return (x + m - 1) / m * m; }

// Which tensor-core value net serves a game: the resident kernel (leaf_mlp_tc.cuh: weights and two query tiles in shared
// memory, at most 16 outputs) where it fits and is not overridden, else the wide kernel (leaf_mlp_tc_wide.cuh: weights only,
// query fragments loaded from global memory, nout = roundup(H, 16) outputs).  Returns false when neither fits; `why` then
// holds the byte arithmetic.  `smem_limit` is the device's opt-in shared memory per block.
struct TcPlan { bool wide = false; int nout = cfrb::tc::kNout, smem_bytes = 0; };
bool tc_plan(int H, int Qpad, int smem_limit, bool force_wide, TcPlan* plan, std::string* why) {
  const cfrb::tc::BlobLayout R(Qpad);
  if (!force_wide && H <= cfrb::tc::kNout && R.smem_bytes <= smem_limit) {
    plan->wide = false; plan->nout = cfrb::tc::kNout; plan->smem_bytes = R.smem_bytes;
    return true;
  }
  const int nout = round_up(H, 16);
  const cfrb::tc::WideLayout W(Qpad, nout);
  if (nout <= 48 && Qpad / 16 <= cfrb::tc::kWideMaxKSteps && W.smem_bytes <= smem_limit) {
    plan->wide = true; plan->nout = nout; plan->smem_bytes = W.smem_bytes;
    return true;
  }
  if (why)
    *why = "tensor-core value net does not fit this game: num_hands " + std::to_string(H) + ", padded query width " +
           std::to_string(Qpad) + ", output layer " + std::to_string(nout) + " (at most 48); weights W1 256 x " +
           std::to_string(Qpad) + " x 2 B + W2 131072 B + W3 " + std::to_string(nout) + " x 256 x 2 B + biases / LayerNorm " +
           std::to_string(W.blob_bytes - W.off_b2) + " B = " + std::to_string(W.smem_bytes) + " B of shared memory (with the "
           "mbarrier) > " + std::to_string(smem_limit) + " B per block; use CFRB_NET_FP32";
  return false;
}

// Typed (fp32 / fp64) part of the solver state.
template <typename Real>
struct WaveState {
  using real = Real;
  DevBuf<real> beliefs, mu, R, Sg, S, Snap, vterm, scaler, scratch;
  cfrb::CfrDev<real> dev{};
};

}  // namespace

struct cfrb_handle {
  cfrb_config cfg{};
  cfrb::GameShape g;
  std::vector<cfrb::TreeTemplate> tmpl;   // index = root_bid + 1
  int Nmax = 0, Lmax = 0, Tmax = 0;
  int Qpad = 0, Hout = 0;
  bool f64 = true;
  int group = 32;          // threads per subgame group (32 = warp, 256 = CTA with global scratch)
  int groups_per_cta = 8;
  int scratch_per_group = 0;  // reals
  // depth <= 2 kernel (all templates have at most three levels): own scratch layout and CTA shape
  bool d2 = false;
  int max_levels = 0;
  int d2_groups_per_cta = 8;
  int d2_scratch_per_group = 0;
  size_t d2_smem = 0;      // dynamic shared memory of a depth-2 CTA
  int d2_ctas = 0;         // CTAs of the depth-2 kernel resident at once on the device: its persistent grid
  int d2_grid_cap = 0;     // test aid (cfrb_debug_d2_grid): at most this many CTAs, 0 = no cap
  std::vector<int> tmpl_rank;   // schedule rank of each template (schedule_ranks)
  bool sorted = false;     // d_sg_order holds the current wave's schedule; otherwise the depth-2 kernel takes wave order
  int n1max = 0;           // bound on the level-1 nodes of a template (the depth-2 scratch layout)
  int table_stride = 0;
  int num_sms = 0;
  Stream own_stream;
  Event ev_a, ev_b;
  int profiling = 0;          // 0 off, n: bracket every n-th value-net launch with CUDA events
  int net_launch_idx = 0, net_launches_run = 0;
  std::vector<Event> net_ev;   // pairs around value-net launches (profiling mode)
  int net_ev_used = 0;
  // CUDA graphs of whole cfrb_run calls (2 launches per iteration would otherwise be enqueued one by one by the host)
  struct GraphEntry { int first, count, prof, has_rows, sorted, keep_sum; GraphExec exec; int launches, net_launches, ev_used; };
  std::vector<GraphEntry> graphs;
  std::vector<std::array<int, 6>> graph_seen;   // keys requested once: a graph is only built for a key that comes back
  bool capturing = false;           // launch geometry independent of the wave size while a graph is being captured / replayed
  // device: templates
  DevBuf<cfrb::TemplateDev> d_tmpl;
  DevBuf<int> d_parent, d_child_begin, d_nchild, d_last_bid, d_level_begin, d_pleaf_node, d_term_node;
  DevBuf<unsigned char> d_matches;
  // full-depth tree for cfrb_exploitability / cfrb_ev2 / the regret accumulator, built on first use
  struct BrState {
    bool ready = false;
    cfrb::TreeTemplate t;
    DevBuf<int> parent, child_begin, nchild, level_begin, term_node, depth, act_lo;
    DevBuf<double> strategy, strategy2, scratch, out;
    size_t scratch_stride = 0;
  } br;
  // immediate-regret accumulator (cfrb_regrets_*): sums [N_full][H][A] and the number of strategies added
  struct RegretState {
    bool ready = false;
    int cap = 0;                     // strategies per batch
    DevBuf<double> acc, val, scratch;
    DevBuf<float> s32;
    int64_t count = 0;
  } rg;
  DevBuf<__half> d_qconst;
  DevBuf<unsigned char> d_tpk;   // byte-packed templates for the depth <= 2 kernel
  int tpk_stride = 0;
  // device: wave (untyped part)
  DevBuf<int> d_wave;      // [0] = n, [1] = rows
  DevBuf<int> d_sg_tmpl, d_sg_player, d_sg_row_off, d_sg_act, d_steps;
  DevBuf<int> d_sg_order, d_tmpl_rank, d_ticket;   // the depth-2 kernel's schedule, template ranks, subgame counter
  DevBuf<float> d_X, d_out, d_dbg;
  long long* dbg_trace = nullptr;   // set only inside cfrb_debug_net_trace
  int x2_gelu = 2;                  // GELU variant of CFRB_NET_TC_F16X2 (leaf_mlp_tc.cuh kGelu): 2 = fp32 tanh, 1 = packed half
  TcPlan tc;                        // which tensor-core kernel serves the game (tc_plan)
  DevBuf<__half> d_Xh;
  WaveState<float> sf;
  WaveState<double> sd;
  // device: weights
  DevBuf<float> d_w;
  DevBuf<uint8_t> d_blob;
  // weight upload without stalling the generator pipeline: two pinned staging buffers, stream-ordered copies on own_stream
  Pinned<uint8_t> w_stage[2];
  size_t w_stage_bytes = 0;
  Event w_ev[2];
  int w_slot = 0;
  cudaEvent_t w_last = nullptr;      // completion of the most recent upload (waited for by runs on other streams)
  cfrb::NetDev net{};
  bool have_weights = false;
  uint64_t weights_version = 0;
  uint64_t weight_uploads = 0;       // cfrb_set_weights calls so far
  // The current wave is a CFR self-play wave, solved without the sum table S (the self-play loop never reads it).  Readers of S
  // rebuild it first (materialise_sum), which needs the weights that wave was solved with: upload count sum_uploads.
  bool sum_dropped = false;
  uint64_t sum_uploads = 0;
  // host mirror of the wave
  int n = 0, rows = 0, iters_done = 0;
  std::vector<int> h_tmpl, h_player, h_row_off, h_last_bid;
  std::vector<double> h_beliefs;
  int64_t launches = 0;
  float last_total_ms = 0.f, last_net_ms = 0.f;
  // device-resident self-play (cfrb_selfplay_*): game states, generator streams
  struct SelfPlay {
    bool ready = false, pending = false;    // pending: a wave has been run whose games have not been advanced yet
    int K = 0;
    DevBuf<int> last_bid, player, mt_idx;
    DevBuf<double> beliefs;
    DevBuf<uint32_t> mt, seeds;
    cfrb::SpDev dev{};
    int64_t waves = 0;
    Event ev_examples;    // recorded behind the example / advance kernels of the last finished wave
    bool ev_recorded = false;
  } sp;
  Event marks[8];                      // cfrb_mark: timing events
  DevBuf<unsigned char> flush_buf;     // cfrb_l2_flush
  bool rows_on_device = false;   // the wave was built on the device: its row count / roots exist only there
  bool mirror_stale = false;     // ... and the host mirror (h_tmpl, h_beliefs, rows) has not been pulled yet
  bool in_match = false;         // an agent of a live cfrb_match: its waves are built by the match
  int64_t to_leaf_free_cap = 0;  // test aid (cfrb_debug_to_leaf_free_cap): cfrb_to_leaf_exploitability sees at most this many free bytes
};

// Calls f with the handle's typed (fp64 or fp32) solver state.
template <class F>
static decltype(auto) with_state(cfrb_handle* h, F&& f) { return h->f64 ? f(h->sd) : f(h->sf); }
// The same for the two agents of a match, which share their state dtype (cfrb_match_create checks it).
template <class F>
static decltype(auto) with_state(cfrb_handle* a, cfrb_handle* b, F&& f) { return a->f64 ? f(a->sd, b->sd) : f(a->sf, b->sf); }

using cfrb::TemplateDev;

// ------------------------------------------------------------------------------------------ typed helpers
// Device reals -> host doubles or floats, element by element (one copy when the types agree).
template <typename real, typename out_t>
static int pull_reals(const real* src, size_t n, out_t* out) {
  if constexpr (std::is_same_v<real, out_t>) {
    CK(cudaMemcpy(out, src, n * sizeof(real), cudaMemcpyDeviceToHost));
  } else {
    std::vector<real> tmp(n);
    CK(cudaMemcpy(tmp.data(), src, n * sizeof(real), cudaMemcpyDeviceToHost));
    std::copy(tmp.begin(), tmp.end(), out);
  }
  return CFRB_OK;
}
// Host doubles -> device reals, converted on the host; returns once stream `st` has copied them.
template <typename real>
static int push_reals(const double* src, size_t n, real* dst, cudaStream_t st) {
  const std::vector<real> tmp(src, src + n);
  CK(cudaMemcpyAsync(dst, tmp.data(), n * sizeof(real), cudaMemcpyHostToDevice, st));
  CK(cudaStreamSynchronize(st));
  return CFRB_OK;
}

template <typename real>
static int alloc_state(cfrb_handle* h, WaveState<real>& s, int max_optin) {
  const auto& g = h->g;
  const int K = h->cfg.max_subgames;
  const size_t tab = (size_t)K * h->table_stride;
  const size_t rows_cap = (size_t)K * std::max(h->Lmax, 1);
  CK(s.beliefs.alloc((size_t)K * 2 * g.H)); CK(s.mu.alloc((size_t)K * 2 * g.H));
  CK(s.R.alloc(tab)); CK(s.Sg.alloc(tab)); CK(s.S.alloc(tab)); CK(s.Snap.alloc(tab));
  const int vterm_stride = round_up(std::max(h->Tmax, 1) * g.H, 4);     // 16-byte aligned rows
  CK(s.vterm.alloc((size_t)K * vterm_stride + 8)); CK(s.scaler.alloc(rows_cap + 8));
  CK(cudaMemset(s.vterm.p, 0, ((size_t)K * vterm_stride + 8) * sizeof(real)));
  CK(cudaMemset(s.scaler.p, 0, (rows_cap + 8) * sizeof(real)));
  CK(cudaMemset(s.Snap.p, 0, tab * sizeof(real)));
  CK(cudaMemset(s.S.p, 0, tab * sizeof(real)));   // self-play waves leave S alone: its entries outside a wave's trees stay defined
  const size_t per_group_bytes = (size_t)h->scratch_per_group * sizeof(real);
  if (per_group_bytes * 2 <= (size_t)max_optin) {
    h->group = 32;
    // 2 CTAs per SM, as many warps per CTA as fit in ~85 % of the shared memory (the rest stays L1 for the read-only
    // template arrays), capped by the register file (64 registers x 32 warps) and the 512-thread block
    const size_t budget = (size_t)max_optin * 85 / 100 / 2;
    h->groups_per_cta = (int)std::max<size_t>(1, std::min<size_t>(16, budget / per_group_bytes));
    const int smem_bytes = (int)(per_group_bytes * h->groups_per_cta);
    CK(cfrb::cfr_configure<real>(32, smem_bytes));
    if (h->max_levels <= 3 && h->tpk_stride > 0) {
      // 32 warps per SM (register file: 64 registers x 32 warps) as 8 CTAs of 4 warps; each CTA has 1 KB of shared memory reserved
      // by the runtime.  The grid is at most the resident CTAs (d2_ctas): persistent warps, costliest subgame first
      h->d2 = true;
      h->d2_scratch_per_group = cfrb::cfr_scratch_reals_d2((int)sizeof(real), h->Nmax, h->g.H, h->Lmax, h->Tmax, h->n1max);
      const size_t d2_bytes = (size_t)h->d2_scratch_per_group * sizeof(real) + h->tpk_stride;
      const size_t cta_budget = ((size_t)228 * 1024 - 8 * 1024) / 8;
      h->d2_groups_per_cta = (int)std::max<size_t>(1, std::min<size_t>(4, cta_budget / d2_bytes));
      h->d2_smem = d2_bytes * h->d2_groups_per_cta;
      int ctas_per_sm = 0;
      CK(cfrb::cfr_configure_d2<real>(g.H, 32 * h->d2_groups_per_cta, (int)h->d2_smem, &ctas_per_sm));
      h->d2_ctas = std::max(1, ctas_per_sm) * h->num_sms;
    }
  } else {
    h->group = 256;
    h->groups_per_cta = 1;
    CK(s.scratch.alloc((size_t)K * h->scratch_per_group));
  }
  cfrb::CfrDev<real>& d = s.dev;
  d.A = g.A; d.H = g.H; d.F = g.F; d.Q = g.Q; d.Qpad = h->Qpad; d.Hout = h->Hout;
  d.tmpl = h->d_tmpl.p; d.parent = h->d_parent.p; d.child_begin = h->d_child_begin.p; d.nchild = h->d_nchild.p;
  d.last_bid = h->d_last_bid.p; d.level_begin = h->d_level_begin.p; d.pleaf_node = h->d_pleaf_node.p;
  d.term_node = h->d_term_node.p; d.matches = h->d_matches.p; d.qconst = h->d_qconst.p;
  d.tpk = h->d_tpk.p; d.tpk_stride = h->tpk_stride;
  d.wave_n = h->d_wave.p; d.sg_tmpl = h->d_sg_tmpl.p; d.sg_player = h->d_sg_player.p; d.sg_row_off = h->d_sg_row_off.p;
  d.sg_act_iter = h->d_sg_act.p; d.beliefs = s.beliefs.p; d.mu = s.mu.p; d.steps = h->d_steps.p;
  d.sg_order = nullptr; d.ticket = h->d_ticket.p;
  d.R = s.R.p; d.Sg = s.Sg.p; d.S = s.S.p; d.Snap = s.Snap.p; d.table_stride = h->table_stride;
  d.vterm = s.vterm.p; d.vterm_stride = vterm_stride;
  d.lmax = std::max(h->Lmax, 1); d.tmax = std::max(h->Tmax, 1); d.n1max = h->n1max;
  d.X = h->cfg.net_mode == CFRB_NET_FP32 ? h->d_X.p : nullptr;
  d.Xh = is_tc(h->cfg.net_mode) ? h->d_Xh.p : nullptr;
  d.net_out = h->d_out.p; d.scaler = s.scaler.p;
  d.scratch = h->group == 32 ? nullptr : s.scratch.p; d.scratch_stride = h->scratch_per_group;
  d.nh_max = h->Nmax * g.H; d.tmp_reals = cfrb::cfr_tmp_reals(h->Nmax, g.H, h->Lmax, h->Tmax);
  d.linear = h->cfg.linear_update; d.dcfr = h->cfg.dcfr;
  d.dcfr_alpha = (real)h->cfg.dcfr_alpha; d.dcfr_beta = (real)h->cfg.dcfr_beta; d.dcfr_gamma = (real)h->cfg.dcfr_gamma;
  d.use_net = h->cfg.net_mode != CFRB_NET_ZERO;
  d.fp = h->cfg.solver == CFRB_SOLVER_FP; d.optimistic = h->cfg.optimistic;
  d.keep_sum = 1;
  return CFRB_OK;
}

// The kernel parameters of the current wave.
template <typename real>
static cfrb::CfrDev<real> wave_dev(const cfrb_handle* h, const WaveState<real>& s) {
  cfrb::CfrDev<real> d = s.dev;
  d.keep_sum = !h->sum_dropped;
  return d;
}

static int launch_init(cfrb_handle* h, cudaStream_t st) {
  const int blocks = (h->n + h->groups_per_cta - 1) / h->groups_per_cta;
  with_state(h, [&](auto& s) {
    using real = typename std::decay_t<decltype(s)>::real;
    const size_t smem = h->group == 32 ? (size_t)h->scratch_per_group * sizeof(real) * h->groups_per_cta : 0;
    cfrb::cfr_launch_init<real>(wave_dev(h, s), h->group, blocks, 32 * h->groups_per_cta, smem, st, h->scratch_per_group);
  });
  ++h->launches;
  CK(cudaGetLastError());
  return CFRB_OK;
}

template <typename real>
static int launch_iter(cfrb_handle* h, WaveState<real>& s, cudaStream_t st, int iter, int do_b, int do_f) {
  const int nsg = h->capturing ? h->cfg.max_subgames : h->n;   // surplus groups return at once (k >= *wave_n)
  cfrb::CfrDev<real> d = wave_dev(h, s);
  if (h->d2) {
    // persistent warps: no more CTAs than are resident at once (the warps then take the wave's subgames from a counter)
    int blocks = std::min((nsg + h->d2_groups_per_cta - 1) / h->d2_groups_per_cta, h->d2_ctas);
    if (h->d2_grid_cap > 0) blocks = std::min(blocks, h->d2_grid_cap);
    d.sg_order = h->sorted ? h->d_sg_order.p : nullptr;
    cfrb::cfr_launch_iter_d2<real>(d, blocks, 32 * h->d2_groups_per_cta, h->d2_smem, st, iter, do_b, do_f, h->d2_scratch_per_group);
  } else {
    const int blocks = (nsg + h->groups_per_cta - 1) / h->groups_per_cta;
    const size_t smem = h->group == 32 ? (size_t)h->scratch_per_group * sizeof(real) * h->groups_per_cta : 0;
    cfrb::cfr_launch_iter<real>(d, h->group, blocks, 32 * h->groups_per_cta, smem, st, iter, do_b, do_f, h->scratch_per_group);
  }
  ++h->launches;
  CK(cudaGetLastError());
  return CFRB_OK;
}

// compact [E][H] (edge = child-1) <-> dense [Nmax][H][A]
static void to_dense(const cfrb_handle* h, int k, const double* compact, double* dense) {
  const auto& t = h->tmpl[h->h_tmpl[k]];
  const int H = h->g.H, A = h->g.A;
  std::memset(dense, 0, sizeof(double) * (size_t)h->Nmax * H * A);
  for (int n = 0; n < t.N; ++n)
    for (int j = 0; j < t.nchild[n]; ++j) {
      const int c = t.child_begin[n] + j, a = t.act_lo[n] + j;
      for (int hd = 0; hd < H; ++hd) dense[((size_t)n * H + hd) * A + a] = compact[(size_t)(c - 1) * H + hd];
    }
}
template <typename real>
static void from_dense(const cfrb_handle* h, int k, const double* dense, real* compact) {
  const auto& t = h->tmpl[h->h_tmpl[k]];
  const int H = h->g.H, A = h->g.A;
  for (int n = 0; n < t.N; ++n)
    for (int j = 0; j < t.nchild[n]; ++j) {
      const int c = t.child_begin[n] + j, a = t.act_lo[n] + j;
      for (int hd = 0; hd < H; ++hd) compact[(size_t)(c - 1) * H + hd] = (real)dense[((size_t)n * H + hd) * A + a];
    }
}

// The table holding a handle's average strategy (ISubgameSolver::get_strategy): FP keeps it in Sg; CFR's is the normalised sum
// S (subgame_solving.cc:659-660), so it needs normalising.
template <typename real>
struct AvgTable { real* p; bool normalise; };
template <typename real>
static AvgTable<real> avg_table(const cfrb_handle* h, WaveState<real>& s) {
  const bool fp = h->cfg.solver == CFRB_SOLVER_FP;
  return {fp ? s.Sg.p : s.S.p, !fp};
}

// Normalises the current wave's compact sums `tab` [n][table_stride] into average strategies, in place.  The average of a player
// stays the uniform initial strategy until that player's first update (CFR ctor, subgame_solving.cc:516-518; the normalised sum is
// only written in step(), :659-660).
static int normalise_avg(cfrb_handle* h, double* tab) {
  std::vector<int> steps((size_t)h->n * 2);
  CK(cudaMemcpy(steps.data(), h->d_steps.p, steps.size() * sizeof(int), cudaMemcpyDeviceToHost));
  const int H = h->g.H;
  for (int k = 0; k < h->n; ++k) {
    const auto& t = h->tmpl[h->h_tmpl[k]];
    double* tk = tab + (size_t)k * h->table_stride;
    for (int nn = 0; nn < t.N; ++nn) {
      const int nc = t.nchild[nn];
      if (!nc) continue;
      const bool untouched = steps[2 * k + (h->h_player[k] ^ (t.depth[nn] & 1))] == 0;
      for (int hd = 0; hd < H; ++hd) {
        double sum = 0;
        for (int j = 0; j < nc; ++j) sum += tk[(size_t)(t.child_begin[nn] + j - 1) * H + hd];
        for (int j = 0; j < nc; ++j) {
          double& v = tk[(size_t)(t.child_begin[nn] + j - 1) * H + hd];
          v = (sum > 0 && !untouched) ? v / sum : 1.0 / nc;
        }
      }
    }
  }
  return CFRB_OK;
}

// Rebuilds the sum table of a wave solved without it (sum_dropped): replays the wave from cfr_init with S kept, on the handle's
// stream, from the wave's own descriptors (roots, players, beliefs, act_iterations, row offsets, schedule), which stay on the device
// until the next wave is built.  The solve is deterministic, so R, Sg, Snap, mu and the step counters are rewritten with the bits
// they hold, and S comes out as a wave that kept it would have left it.  Refused when the value-net weights have been replaced since
// the wave was solved: the replay would solve a different wave.
static int materialise_sum(cfrb_handle* h) {
  if (!h->sum_dropped) return CFRB_OK;
  if (h->weight_uploads != h->sum_uploads)
    return fail(CFRB_EINVAL, "the sum strategy of this self-play wave was not kept, and it cannot be rebuilt: the value-net weights "
                             "have been replaced (cfrb_set_weights) since the wave was solved");
  const int iters = h->iters_done;
  h->sum_dropped = false;
  h->iters_done = 0;
  int rc = launch_init(h, h->own_stream);
  if (!rc) rc = cfrb_run(h, iters, h->own_stream);
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->own_stream));
  return CFRB_OK;
}

// The current wave's compact tables [n][table_stride] as doubles.  which: 0 = Snap, 1 = Sg, 2 = S, 3 = R, 4 = the average
// strategy (avg_table, normalised where it is a sum).
static int pull_table(cfrb_handle* h, int which, double* out) {
  if (which == 2 || which == 4) {
    const int rc = materialise_sum(h);
    if (rc) return rc;
  }
  bool normalise = false;
  int rc = with_state(h, [&](auto& s) {
    const auto avg = avg_table(h, s);
    normalise = which == 4 && avg.normalise;
    const auto* src = which == 0 ? s.Snap.p : which == 1 ? s.Sg.p : which == 2 ? s.S.p : which == 4 ? avg.p : s.R.p;
    return pull_reals(src, (size_t)h->n * h->table_stride, out);
  });
  if (!rc && normalise) rc = normalise_avg(h, out);
  return rc;
}

template <typename real>
static int load_state_t(cfrb_handle* h, WaveState<real>& s, const double* regrets, const double* last_strategy,
                        const double* sum_strategy, const double* root_value_means) {
  const int n = h->n, H = h->g.H, A = h->g.A;
  const size_t dense_sz = (size_t)h->Nmax * H * A;
  std::vector<real> tmp((size_t)n * h->table_stride);
  auto push = [&](const double* dense, real* ddst) -> int {
    CK(cudaMemcpy(tmp.data(), ddst, tmp.size() * sizeof(real), cudaMemcpyDeviceToHost));
    for (int k = 0; k < n; ++k) from_dense<real>(h, k, dense + (size_t)k * dense_sz, tmp.data() + (size_t)k * h->table_stride);
    CK(cudaMemcpy(ddst, tmp.data(), tmp.size() * sizeof(real), cudaMemcpyHostToDevice));
    return CFRB_OK;
  };
  int rc;
  if (regrets && (rc = push(regrets, s.R.p))) return rc;
  if (last_strategy && (rc = push(last_strategy, s.Sg.p))) return rc;
  if (sum_strategy && (rc = push(sum_strategy, s.S.p))) return rc;
  if (root_value_means) return push_reals(root_value_means, (size_t)n * 2 * H, s.mu.p, nullptr);
  return CFRB_OK;
}

// A wave built on the device (cfrb_selfplay_wave) has no host mirror of its subgame descriptors; the inspection entry points
// (fetch / examples / load_state / reset, used by tests and evaluators, not by the self-play loop) pull it on demand.
static int sync_mirror(cfrb_handle* h) {
  if (!h->rows_on_device || !h->mirror_stale) return CFRB_OK;
  CK(cudaDeviceSynchronize());
  const int n = h->n;
  int wave[2] = {0, 0};
  CK(cudaMemcpy(wave, h->d_wave.p, sizeof(wave), cudaMemcpyDeviceToHost));
  h->rows = wave[1];
  h->h_tmpl.resize(n); h->h_player.resize(n); h->h_row_off.resize(n); h->h_last_bid.resize(n);
  CK(cudaMemcpy(h->h_tmpl.data(), h->d_sg_tmpl.p, n * sizeof(int), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h->h_player.data(), h->d_sg_player.p, n * sizeof(int), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(h->h_row_off.data(), h->d_sg_row_off.p, n * sizeof(int), cudaMemcpyDeviceToHost));
  for (int k = 0; k < n; ++k) h->h_last_bid[k] = h->h_tmpl[k] - 1;
  h->h_beliefs.resize((size_t)n * 2 * h->g.H);
  int rc = with_state(h, [&](auto& s) { return pull_reals(s.beliefs.p, h->h_beliefs.size(), h->h_beliefs.data()); });
  if (rc) return rc;
  h->mirror_stale = false;
  return CFRB_OK;
}

extern "C" {

const char* cfrb_last_error(void) { return g_err.c_str(); }

int cfrb_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int cfrb_destroy(cfrb_handle* h) {
  if (!h) return CFRB_OK;
  cudaSetDevice(h->cfg.device);
  if (h->own_stream) cudaStreamSynchronize(h->own_stream);
  delete h;
  return CFRB_OK;
}

static int create_impl(const cfrb_config* cfg, cfrb_handle* h) {
  h->cfg = *cfg;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(CFRB_ENODEV, "no CUDA device visible: libcfrb200 has no CPU fallback");
  }
  if (cfg->device < 0 || cfg->device >= ndev) return fail(CFRB_EINVAL, "device ordinal out of range");
  CK(cudaSetDevice(cfg->device));
  if (cfg->num_dice < 1 || cfg->num_faces < 1 || cfg->max_depth < 1 || cfg->max_subgames < 1)
    return fail(CFRB_EINVAL, "num_dice, num_faces, max_depth, max_subgames must be >= 1");
  if (cfg->net_mode < CFRB_NET_ZERO || cfg->net_mode > CFRB_NET_TC_F16X2) return fail(CFRB_EINVAL, "bad net_mode");
  if (cfg->state_dtype != CFRB_STATE_F64 && cfg->state_dtype != CFRB_STATE_F32) return fail(CFRB_EINVAL, "bad state_dtype");
  if (cfg->solver != CFRB_SOLVER_CFR && cfg->solver != CFRB_SOLVER_FP) return fail(CFRB_EINVAL, "bad solver");
  if (cfg->net_mode != CFRB_NET_ZERO && cfg->hidden != 256) return fail(CFRB_EINVAL, "only hidden == 256 is built");
  h->f64 = cfg->state_dtype == CFRB_STATE_F64;
  h->g = cfrb::GameShape(cfg->num_dice, cfg->num_faces);
  const auto& g = h->g;
  if (g.A > 1024 || g.H > 4096) return fail(CFRB_EINVAL, "game too large");
  // ---- templates: root_bid in {-1, 0 .. A-2}
  std::vector<TemplateDev> td;
  std::vector<int> parent, child_begin, nchild, last_bid, level_begin, pleaf_node, term_node;
  std::vector<__half> qconst;
  const int Qpad = round_up(g.Q + 1, 16);
  for (int rb = -1; rb <= g.A - 2; ++rb) {
    h->tmpl.push_back(cfrb::build_template(g, rb, cfg->max_depth));
    const auto& t = h->tmpl.back();
    TemplateDev d;
    d.node_off = (int)child_begin.size(); d.level_off = (int)level_begin.size();
    d.pleaf_off = (int)pleaf_node.size(); d.term_off = (int)term_node.size();
    d.N = t.N; d.L = t.L; d.T = t.T; d.levels = t.levels;
    d.qconst_off = (int)qconst.size();
    for (int n : t.pleaf_node)
      for (int q = 0; q < Qpad; ++q)   // one-hot of the leaf's last bid (subgame_solving.cc:111-113) and the constant 1 at column Q
        qconst.push_back(__float2half_rn((q >= 2 && q < 2 + g.A && q - 2 == t.last_bid[n]) || q == g.Q ? 1.f : 0.f));
    td.push_back(d);
    parent.insert(parent.end(), t.parent.begin(), t.parent.end());
    child_begin.insert(child_begin.end(), t.child_begin.begin(), t.child_begin.end());
    nchild.insert(nchild.end(), t.nchild.begin(), t.nchild.end());
    last_bid.insert(last_bid.end(), t.last_bid.begin(), t.last_bid.end());
    level_begin.insert(level_begin.end(), t.level_begin.begin(), t.level_begin.end());
    level_begin.push_back(t.N);   // sentinel: "children of the last level" is an empty range
    pleaf_node.insert(pleaf_node.end(), t.pleaf_node.begin(), t.pleaf_node.end());
    term_node.insert(term_node.end(), t.term_node.begin(), t.term_node.end());
    for (int n : t.term_node) term_node.push_back(t.last_bid[t.parent[n]]);   // challenged bid
    for (int n : t.term_node) term_node.push_back(t.depth[n]);
    h->max_levels = std::max(h->max_levels, t.levels);
    h->Nmax = std::max(h->Nmax, t.N); h->Lmax = std::max(h->Lmax, t.L); h->Tmax = std::max(h->Tmax, t.T);
  }
  std::vector<unsigned char> matches((size_t)g.H * g.F);
  for (int hd = 0; hd < g.H; ++hd)
    for (int f = 0; f < g.F; ++f) matches[(size_t)hd * g.F + f] = (unsigned char)g.num_matches(hd, f);

  // byte-packed copies of the templates for cfr_iter_d2_kernel (one coalesced copy into shared memory per subgame and launch):
  // header {N, L, T, levels, n1e, n2e, -, -, qconst_off:int32, -} | parent[N] child_begin[N] nchild[N] last_bid+1[N] pleaf[L]
  // term[3][T] matches[H*F]; only built when every count fits a byte (all depth <= 2 trees of the supported games do)
  std::vector<unsigned char> tpk;
  if (h->max_levels <= 3 && h->Nmax <= 255 && g.A <= 254) {
    size_t mx = 0;
    for (const auto& t : h->tmpl) mx = std::max(mx, (size_t)16 + 4 * (size_t)t.N + t.L + 3 * (size_t)t.T + (size_t)g.H * g.F);
    h->tpk_stride = round_up((int)mx, 16);
    tpk.assign((size_t)h->tpk_stride * h->tmpl.size(), 0);
    for (size_t i = 0; i < h->tmpl.size(); ++i) {
      const auto& t = h->tmpl[i];
      unsigned char* b = tpk.data() + i * h->tpk_stride;
      b[0] = (unsigned char)t.N; b[1] = (unsigned char)t.L; b[2] = (unsigned char)t.T; b[3] = (unsigned char)t.levels;
      b[4] = (unsigned char)(t.levels >= 2 ? t.level_begin[2] : t.level_begin[1]);
      b[5] = (unsigned char)(t.levels >= 3 ? t.level_begin[3] : b[4]);
      std::memcpy(b + 8, &td[i].qconst_off, sizeof(int));
      unsigned char* q = b + 16;
      for (int n = 0; n < t.N; ++n) q[n] = (unsigned char)(t.parent[n] < 0 ? 0 : t.parent[n]);
      q += t.N;
      for (int n = 0; n < t.N; ++n) q[n] = (unsigned char)t.child_begin[n];
      q += t.N;
      for (int n = 0; n < t.N; ++n) q[n] = (unsigned char)t.nchild[n];
      q += t.N;
      for (int n = 0; n < t.N; ++n) q[n] = (unsigned char)(t.last_bid[n] + 1);
      q += t.N;
      for (int r = 0; r < t.L; ++r) q[r] = (unsigned char)t.pleaf_node[r];
      q += t.L;
      for (int z = 0; z < t.T; ++z) {
        q[z] = (unsigned char)t.term_node[z];
        q[t.T + z] = (unsigned char)t.last_bid[t.parent[t.term_node[z]]];     // challenged bid (:287); a terminal is never the root
        q[2 * t.T + z] = (unsigned char)t.depth[t.term_node[z]];
      }
      q += 3 * t.T;
      std::memcpy(q, matches.data(), matches.size());
    }
  }
  auto up = [&](auto& buf, const auto& v) -> cudaError_t {
    cudaError_t e = buf.alloc(v.size());
    if (e != cudaSuccess) return e;
    return cudaMemcpy(buf.p, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
  };
  CK(up(h->d_tpk, tpk));
  CK(up(h->d_tmpl, td)); CK(up(h->d_parent, parent)); CK(up(h->d_child_begin, child_begin)); CK(up(h->d_nchild, nchild));
  CK(up(h->d_last_bid, last_bid)); CK(up(h->d_level_begin, level_begin)); CK(up(h->d_pleaf_node, pleaf_node));
  CK(up(h->d_term_node, term_node)); CK(up(h->d_matches, matches)); CK(up(h->d_qconst, qconst));
  h->tmpl_rank = cfrb::schedule_ranks(h->tmpl, g.H);
  CK(up(h->d_tmpl_rank, h->tmpl_rank));

  // ---- sizes
  const int K = cfg->max_subgames;
  h->Qpad = round_up(g.Q + 1, 16);   // one spare column carries the constant 1 that feeds bias 1 through the tensor cores
  h->Hout = round_up(g.H, 4);                                     // value-net output rows padded to 16 bytes
  h->table_stride = round_up(std::max(1, (h->Nmax - 1) * g.H), 4);   // every subgame's tables start 16-byte aligned
  h->n1max = g.A;
  h->scratch_per_group = cfrb::cfr_scratch_reals(h->Nmax, g.H, h->Lmax, h->Tmax);
  int max_optin = 0;
  CK(cudaDeviceGetAttribute(&max_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device));
  CK(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, cfg->device));
  CK(h->d_wave.alloc(2));
  CK(h->d_sg_tmpl.alloc(K)); CK(h->d_sg_player.alloc(K)); CK(h->d_sg_row_off.alloc(K)); CK(h->d_sg_act.alloc(K));
  CK(h->d_steps.alloc((size_t)K * 2));
  CK(h->d_sg_order.alloc(K)); CK(h->d_ticket.alloc(1));
  CK(cudaMemset(h->d_ticket.p, 0, sizeof(int)));
  const size_t rows_cap = (size_t)K * std::max(h->Lmax, 1);
  CK(h->d_X.alloc(cfg->net_mode == CFRB_NET_FP32 ? rows_cap * h->Qpad : 1));
  CK(h->d_out.alloc(rows_cap * h->Hout));
  CK(cudaMemset(h->d_wave.p, 0, 2 * sizeof(int)));
  CK(cudaMemset(h->d_out.p, 0, rows_cap * h->Hout * sizeof(float)));
  if (is_tc(cfg->net_mode)) {
    // CFRB_TC_WIDE=1: the wide kernel also on games the resident kernel serves (tests, measurements)
    const char* fw = std::getenv("CFRB_TC_WIDE");
    std::string why;
    if (!tc_plan(g.H, h->Qpad, max_optin, fw && *fw == '1', &h->tc, &why)) return fail(CFRB_EINVAL, why);
    const size_t tiles = (rows_cap + cfrb::tc::kTileM - 1) / cfrb::tc::kTileM;
    CK(h->d_Xh.alloc(tiles * cfrb::tc::kTileM * h->Qpad));
    CK(cudaMemset(h->d_Xh.p, 0, tiles * cfrb::tc::kTileM * h->Qpad * sizeof(__half)));
    CK(h->d_dbg.alloc(2 * cfrb::tc::kTileM * cfrb::tc::kHid));
    // the limit is per kernel and process-wide: raised to the device's opt-in maximum (see cfr_configure in cfr_kernels.cu)
    const int sm = std::max(h->tc.smem_bytes, max_optin);
    if (h->tc.wide) {
      CK(cfrb::tc::wide_configure(h->tc.nout, sm));
    } else {
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<false, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<true, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
      CK(cudaFuncSetAttribute(cfrb::tc::leaf_mlp_tc_kernel<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, sm));
    }
    // CFRB_NET_TC_F16X2's GELU: fp32 tanh (default) or the packed-half evaluation (CFRB_X2_GELU=half), see leaf_mlp_tc.cuh
    if (const char* e = std::getenv("CFRB_X2_GELU")) h->x2_gelu = std::string(e) == "half" ? 1 : 2;
  }
  CK(cudaFuncSetAttribute(cfrb::leaf_mlp_fp32_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                          (int)cfrb::leaf_mlp_fp32_smem(256)));
  int rc = with_state(h, [&](auto& s) { return alloc_state(h, s, max_optin); });
  if (rc) return rc;
  CK(cudaStreamCreateWithFlags(h->own_stream.put(), cudaStreamNonBlocking));
  CK(cudaEventCreate(h->ev_a.put())); CK(cudaEventCreate(h->ev_b.put()));
  return CFRB_OK;
}

int cfrb_create(const cfrb_config* cfg, cfrb_handle** out) {
  if (!cfg || !out) return fail(CFRB_EINVAL, "null argument");
  *out = nullptr;
  auto h = std::make_unique<cfrb_handle>();
  const int rc = create_impl(cfg, h.get());
  if (rc != CFRB_OK) return rc;
  *out = h.release();
  return CFRB_OK;
}

int cfrb_tc_net_supported(int32_t num_dice, int32_t num_faces, int32_t hidden) {
  if (num_dice < 1 || num_faces < 1 || hidden != 256) return 0;
  long hands = 1;
  for (int i = 0; i < num_dice && hands <= 4096; ++i) hands *= num_faces;
  if (hands > 4096 || 2L * num_dice * num_faces + 1 > 1024) return 0;     // beyond what cfrb_create accepts at all
  const cfrb::GameShape g(num_dice, num_faces);
  TcPlan plan;
  return tc_plan(g.H, round_up(g.Q + 1, 16), cfrb::tc::kSmemOptinSm90, false, &plan, nullptr) ? 1 : 0;
}

int cfrb_num_actions(const cfrb_handle* h) { return h->g.A; }
int cfrb_num_hands(const cfrb_handle* h) { return h->g.H; }
int cfrb_query_size(const cfrb_handle* h) { return h->g.Q; }
int cfrb_max_nodes(const cfrb_handle* h) { return h->Nmax; }

static void export_tree(const cfrb::TreeTemplate& t, int player_id, cfrb_node* out, int cap) {
  for (int n = 0; n < t.N && n < cap; ++n) {
    out[n].last_bid = t.last_bid[n];
    out[n].player_id = player_id ^ (t.depth[n] & 1);
    // like the reference, a processed node with an empty bid range (terminal above the depth limit) keeps
    // children_begin == children_end == (tree size at that moment); unprocessed nodes keep 0/0 (tree.h:59-62)
    out[n].children_begin = t.child_begin[n];
    out[n].children_end = t.child_begin[n] + t.nchild[n];
    out[n].parent = t.parent[n];
    out[n].depth = t.depth[n];
  }
}

int cfrb_unroll_tree(int32_t num_dice, int32_t num_faces, int32_t last_bid, int32_t player_id, int32_t max_depth,
                     cfrb_node* out, int32_t cap) {
  if (num_dice < 1 || num_faces < 1 || max_depth < 0) return fail(CFRB_EINVAL, "bad game shape");
  cfrb::GameShape g(num_dice, num_faces);
  if (last_bid < -1 || last_bid >= g.A) return fail(CFRB_EINVAL, "bad root bid");
  const auto t = cfrb::build_template(g, last_bid, max_depth);
  export_tree(t, player_id, out, cap);
  return t.N;
}

int cfrb_tree_template(const cfrb_handle* h, int32_t last_bid, int32_t player_id, cfrb_node* out, int32_t cap) {
  if (!h || last_bid < -1 || last_bid > h->g.A - 2) return fail(CFRB_EINVAL, "bad root bid");
  const auto& t = h->tmpl[last_bid + 1];
  export_tree(t, player_id, out, cap);
  return t.N;
}

int cfrb_set_weights(cfrb_handle* h, const float* flat, size_t n, uint64_t version) {
  if (!h || !flat) return fail(CFRB_EINVAL, "null argument");
  const int hid = h->cfg.hidden, Q = h->g.Q, H = h->g.H, Qp = h->Qpad;
  const size_t expect = (size_t)hid * Q + 3 * hid + (size_t)hid * hid + 3 * hid + (size_t)H * hid + H;
  if (n != expect) return fail(CFRB_EINVAL, "weight count mismatch: expected " + std::to_string(expect) + " got " + std::to_string(n));
  CK(cudaSetDevice(h->cfg.device));
  const float* w1 = flat; const float* b1 = w1 + (size_t)hid * Q; const float* g1 = b1 + hid; const float* be1 = g1 + hid;
  const float* w2 = be1 + hid; const float* b2 = w2 + (size_t)hid * hid; const float* g2 = b2 + hid; const float* be2 = g2 + hid;
  const float* w3 = be2 + hid; const float* b3 = w3 + (size_t)H * hid;
  // Stream-ordered upload: the packed weights are built in a pinned staging buffer and copied on the handle's stream, i.e.
  // after the waves already enqueued there (ModelLocker::updateModel waits for in-flight forwards; here nothing waits — the
  // generator's software pipeline keeps running) and before everything enqueued later.
  const size_t total_fp32 = (size_t)Qp * hid + 3 * hid + (size_t)hid * hid + 3 * hid + (size_t)hid * h->Hout + h->Hout;
  // tensor-core blob: the resident kernel's layout, or the wide kernel's (W3 with tc.nout rows); with 16 outputs the two agree
  const cfrb::tc::WideLayout L(Qp, h->tc.nout);
  const size_t need = is_tc(h->cfg.net_mode) ? (size_t)L.blob_bytes : total_fp32 * sizeof(float);
  if (h->w_stage_bytes < need) {
    CK(cudaStreamSynchronize(h->own_stream));
    for (int i = 0; i < 2; ++i) {
      CK(cudaMallocHost((void**)h->w_stage[i].put(), need));
      if (!h->w_ev[i]) CK(cudaEventCreateWithFlags(h->w_ev[i].put(), cudaEventDisableTiming));
    }
    h->w_stage_bytes = need;
  }
  const int slot = h->w_slot;
  h->w_slot ^= 1;
  CK(cudaEventSynchronize(h->w_ev[slot]));        // the copy that last used this staging buffer (two uploads ago) is long done
  std::memset(h->w_stage[slot], 0, need);
  if (is_tc(h->cfg.net_mode)) {
    // tensor-core blob: fp16 weights in wgmma K-major core-matrix order + fp32 {bias, gamma, beta} per feature
    struct { uint8_t* p; uint8_t* data() { return p; } } blob{h->w_stage[slot].get()};
    __half* hw1 = reinterpret_cast<__half*>(blob.data() + L.off_w1);
    __half* hw2 = reinterpret_cast<__half*>(blob.data() + L.off_w2);
    __half* hw3 = reinterpret_cast<__half*>(blob.data() + L.off_w3);
    // LayerNorm without the mean (leaf_mlp_tc.cuh).  Subtracting from every column of W (and from the bias) its
    // mean over the 256 output features makes the features of y = W x + b sum to zero for every x, which is all the mean
    // subtraction of LayerNorm does; the epilogue then only needs sum y^2.  Done in double, before the fp16 rounding.
    std::vector<double> m1(Q + 1, 0.0), m2(hid + 1, 0.0);
    for (int k = 0; k < Q; ++k) { for (int j = 0; j < hid; ++j) m1[k] += w1[(size_t)j * Q + k]; m1[k] /= hid; }
    for (int j = 0; j < hid; ++j) m1[Q] += b1[j];
    m1[Q] /= hid;
    for (int k = 0; k < hid; ++k) { for (int j = 0; j < hid; ++j) m2[k] += w2[(size_t)j * hid + k]; m2[k] /= hid; }
    for (int j = 0; j < hid; ++j) m2[hid] += b2[j];
    m2[hid] /= hid;
    for (int j = 0; j < hid; ++j) for (int k = 0; k < Q; ++k) hw1[cfrb::tc::umma_kmajor_offset_halves(j, k, hid)] = __float2half_rn((float)(w1[(size_t)j * Q + k] - m1[k]));
    for (int j = 0; j < hid; ++j) hw1[cfrb::tc::umma_kmajor_offset_halves(j, Q, hid)] = __float2half_rn((float)(b1[j] - m1[Q]));   // bias 1 x constant-1 column
    float* fb2 = reinterpret_cast<float*>(blob.data() + L.off_b2);      // bias 2, rounded to fp16 like bias 1 in W1
    for (int j = 0; j < hid; ++j) fb2[j] = __half2float(__float2half_rn((float)(b2[j] - m2[hid])));
    for (int j = 0; j < hid; ++j) for (int k = 0; k < hid; ++k) hw2[cfrb::tc::umma_kmajor_offset_halves(j, k, hid)] = __float2half_rn((float)(w2[(size_t)j * hid + k] - m2[k]));
    for (int j = 0; j < H; ++j) for (int k = 0; k < hid; ++k) hw3[cfrb::tc::umma_kmajor_offset_halves(j, k, h->tc.nout)] = __float2half_rn(w3[(size_t)j * hid + k]);
    float* ln1 = reinterpret_cast<float*>(blob.data() + L.off_ln1);
    float* ln2 = reinterpret_cast<float*>(blob.data() + L.off_ln2);
    // the GELU of CFRB_NET_TC_F16X2 evaluates the activation from y / 2: gamma / 2 and beta / 2 are stored
    const float lnscale = h->cfg.net_mode == CFRB_NET_TC_F16X2 ? 0.5f : 1.f;
    for (int j = 0; j < hid; ++j) {
      // per feature pair (j even): {gamma_j, gamma_j+1, beta_j, beta_j+1}: one 16-byte load per column pair of the epilogue
      const int o = (j >> 1) * 4 + (j & 1);
      ln1[o] = lnscale * g1[j]; ln1[o + 2] = lnscale * be1[j];
      ln2[o] = lnscale * g2[j]; ln2[o + 2] = lnscale * be2[j];
    }
    std::copy(b3, b3 + H, reinterpret_cast<float*>(blob.data() + L.off_b3));
    if (!h->d_blob.p) CK(h->d_blob.alloc(L.blob_bytes));
    CK(cudaMemcpyAsync(h->d_blob.p, blob.data(), L.blob_bytes, cudaMemcpyHostToDevice, h->own_stream));
  } else {
    // transposed k-major fp32 weights for the SIMT kernel
    const size_t total = (size_t)Qp * hid + 3 * hid + (size_t)hid * hid + 3 * hid + (size_t)hid * h->Hout + h->Hout;
    struct { float* p; float& operator[](size_t i) { return p[i]; } float* begin() { return p; } float* data() { return p; } } pk{reinterpret_cast<float*>(h->w_stage[slot].get())};
    size_t o = 0;
    const size_t o_w1 = o; for (int k = 0; k < Q; ++k) for (int j = 0; j < hid; ++j) pk[o_w1 + (size_t)k * hid + j] = w1[(size_t)j * Q + k];
    o += (size_t)Qp * hid;
    const size_t o_b1 = o; std::copy(b1, b1 + hid, pk.begin() + o); o += hid;
    const size_t o_g1 = o; std::copy(g1, g1 + hid, pk.begin() + o); o += hid;
    const size_t o_be1 = o; std::copy(be1, be1 + hid, pk.begin() + o); o += hid;
    const size_t o_w2 = o; for (int k = 0; k < hid; ++k) for (int j = 0; j < hid; ++j) pk[o_w2 + (size_t)k * hid + j] = w2[(size_t)j * hid + k];
    o += (size_t)hid * hid;
    const size_t o_b2 = o; std::copy(b2, b2 + hid, pk.begin() + o); o += hid;
    const size_t o_g2 = o; std::copy(g2, g2 + hid, pk.begin() + o); o += hid;
    const size_t o_be2 = o; std::copy(be2, be2 + hid, pk.begin() + o); o += hid;
    const size_t o_w3 = o; for (int k = 0; k < hid; ++k) for (int j = 0; j < H; ++j) pk[o_w3 + (size_t)k * h->Hout + j] = w3[(size_t)j * hid + k];
    o += (size_t)hid * h->Hout;
    const size_t o_b3 = o; std::copy(b3, b3 + H, pk.begin() + o);
    if (!h->d_w.p) CK(h->d_w.alloc(total));
    CK(cudaMemcpyAsync(h->d_w.p, pk.data(), total * sizeof(float), cudaMemcpyHostToDevice, h->own_stream));
    cfrb::NetDev& nd = h->net;
    nd.Qpad = Qp; nd.hidden = hid; nd.Hout = h->Hout;
    nd.w1t = h->d_w.p + o_w1; nd.b1 = h->d_w.p + o_b1; nd.g1 = h->d_w.p + o_g1; nd.be1 = h->d_w.p + o_be1;
    nd.w2t = h->d_w.p + o_w2; nd.b2 = h->d_w.p + o_b2; nd.g2 = h->d_w.p + o_g2; nd.be2 = h->d_w.p + o_be2;
    nd.w3t = h->d_w.p + o_w3; nd.b3 = h->d_w.p + o_b3;
  }
  CK(cudaEventRecord(h->w_ev[slot], h->own_stream));
  h->w_last = h->w_ev[slot];
  h->have_weights = true;
  h->weights_version = version;
  ++h->weight_uploads;
  return CFRB_OK;
}

uint64_t cfrb_weights_version(const cfrb_handle* h) { return h ? h->weights_version : 0; }

int cfrb_begin_wave(cfrb_handle* h, int32_t n, const int32_t* last_bid, const int32_t* player_id, const double* beliefs,
                    const int32_t* act_iteration) {
  if (!h || (n > 0 && (!last_bid || !player_id || !beliefs))) return fail(CFRB_EINVAL, "null argument");
  if (n < 0 || n > h->cfg.max_subgames) return fail(CFRB_EINVAL, "n exceeds max_subgames");
  CK(cudaSetDevice(h->cfg.device));
  const int H = h->g.H;
  std::vector<int> tm(n), pl(n), ro(n), act(n, -1);
  int rows = 0;
  for (int k = 0; k < n; ++k) {
    if (last_bid[k] < -1 || last_bid[k] > h->g.A - 2) return fail(CFRB_EINVAL, "subgame root bid out of range (terminal or invalid)");
    if (player_id[k] != 0 && player_id[k] != 1) return fail(CFRB_EINVAL, "player_id must be 0 or 1");
    tm[k] = last_bid[k] + 1;
    pl[k] = player_id[k];
    ro[k] = rows;
    rows += h->tmpl[tm[k]].L;
    if (act_iteration) act[k] = act_iteration[k];
  }
  std::vector<int> order(n);
  cfrb::schedule_order(h->tmpl_rank, tm.data(), n, order.data());
  h->n = n; h->rows = rows; h->iters_done = 0; h->rows_on_device = false; h->sp.pending = false; h->sorted = true;
  h->sum_dropped = false;
  h->h_tmpl = tm; h->h_player = pl; h->h_row_off = ro;
  h->h_last_bid.assign(last_bid, last_bid + n);
  h->h_beliefs.assign(beliefs, beliefs + (size_t)n * 2 * H);
  cudaStream_t st = h->own_stream;
  CK(cudaStreamSynchronize(st));
  const int wave[2] = {n, rows};
  CK(cudaMemcpyAsync(h->d_wave.p, wave, sizeof(wave), cudaMemcpyHostToDevice, st));
  if (n) {
    CK(cudaMemcpyAsync(h->d_sg_tmpl.p, tm.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->d_sg_player.p, pl.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->d_sg_row_off.p, ro.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->d_sg_act.p, act.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(h->d_sg_order.p, order.data(), n * sizeof(int), cudaMemcpyHostToDevice, st));
    int rc = with_state(h, [&](auto& s) { return push_reals(h->h_beliefs.data(), h->h_beliefs.size(), s.beliefs.p, st); });
    if (rc) return rc;
    rc = launch_init(h, st);
    if (rc) return rc;
  }
  CK(cudaStreamSynchronize(st));   // host staging vectors above go out of scope
  return CFRB_OK;
}

// Inside a stream capture a plain cudaEventRecord only marks a dependency; cudaEventRecordExternal makes it an event-record
// NODE, whose timestamps can be synchronised on and read after every launch of the graph.
static cudaError_t record_event(cfrb_handle* h, cudaEvent_t ev, cudaStream_t st) {
  return h->capturing ? cudaEventRecordWithFlags(ev, st, cudaEventRecordExternal) : cudaEventRecord(ev, st);
}

// At least `count` events for timing value-net launches (profiling mode).
static int reserve_net_events(cfrb_handle* h, int count) {
  while ((int)h->net_ev.size() < count) {
    Event e;
    CK(cudaEventCreate(e.put()));
    h->net_ev.push_back(std::move(e));
  }
  return CFRB_OK;
}

static int launch_net(cfrb_handle* h, cudaStream_t st, float* dbg1, float* dbg2) {
  if (h->cfg.net_mode == CFRB_NET_ZERO || (h->rows == 0 && !h->rows_on_device)) return CFRB_OK;
  const bool sample = h->profiling > 0 && (h->net_launch_idx % h->profiling) == 0;
  ++h->net_launch_idx;
  if (sample) {
    const int rc = reserve_net_events(h, h->net_ev_used + 2);
    if (rc) return rc;
    CK(record_event(h, h->net_ev[h->net_ev_used], st));
  }
  if (is_tc(h->cfg.net_mode)) {
    cfrb::tc::TcArgs a{h->d_blob.p, h->d_Xh.p, h->d_wave.p + 1, h->d_out.p, h->Qpad, h->g.H, h->Hout, dbg1, dbg2, nullptr};
    const int tiles = (h->rows + cfrb::tc::kTileM - 1) / cfrb::tc::kTileM;
    const int grid = (h->capturing || h->rows_on_device) ? h->num_sms : std::min(tiles, h->num_sms);   // surplus CTAs return at once
    const bool x2 = h->cfg.net_mode == CFRB_NET_TC_F16X2;
    a.trace = h->dbg_trace;
    const bool dbg = dbg1 || dbg2 || a.trace;
    // programmatic dependent launch: the kernel fetches its weights while the CFR kernel before it drains
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(grid); lc.blockDim = dim3(cfrb::tc::kThreads); lc.stream = st;
    lc.dynamicSmemBytes = h->tc.smem_bytes;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    lc.attrs = at; lc.numAttrs = dbg ? 0 : 1;
    const int gelu = x2 ? h->x2_gelu : 0;
    if (h->tc.wide) CK(cfrb::tc::wide_launch(lc, a, h->tc.nout, gelu, dbg));
    else if (dbg && gelu == 1) CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<true, 1>, a));
    else if (dbg && gelu == 2) CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<true, 2>, a));
    else if (dbg) CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<true, 0>, a));
    else if (gelu == 1) CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<false, 1>, a));
    else if (gelu == 2) CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<false, 2>, a));
    else CK(cudaLaunchKernelEx(&lc, cfrb::tc::leaf_mlp_tc_kernel<false, 0>, a));
  } else {
    // a wave built on the device: worst-case grid, CTAs beyond the device-side row count return at once
    const int64_t rows_host = h->rows_on_device ? (int64_t)h->n * std::max(h->Lmax, 1) : h->rows;
    const int blocks = (int)((rows_host + cfrb::kMlpRows - 1) / cfrb::kMlpRows);
    cfrb::leaf_mlp_fp32_kernel<256><<<blocks, 256, cfrb::leaf_mlp_fp32_smem(256), st>>>(h->net, h->d_X.p, h->d_wave.p + 1, h->d_out.p);
  }
  ++h->launches;
  CK(cudaGetLastError());
  if (sample) {
    CK(record_event(h, h->net_ev[h->net_ev_used + 1], st));
    h->net_ev_used += 2;
  }
  return CFRB_OK;
}

int cfrb_reset_wave(cfrb_handle* h, void* cuda_stream) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  h->iters_done = 0;
  h->sum_dropped = false;   // a wave the host runs again keeps its sum
  if (h->n == 0) return CFRB_OK;
  return launch_init(h, cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream);
}

int cfrb_set_profiling(cfrb_handle* h, int32_t on) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  h->profiling = on < 0 ? 0 : on;
  return CFRB_OK;
}

static int enqueue_run(cfrb_handle* h, cudaStream_t st, int first, int last) {
  CK(record_event(h, h->ev_a, st));
  h->net_ev_used = 0;
  h->net_launch_idx = 0;
  for (int i = first; i <= last; ++i) {
    const int do_b = i > first, do_f = i < last;
    int rc = with_state(h, [&](auto& s) { return launch_iter(h, s, st, i, do_b, do_f); });
    if (rc) return rc;
    if (do_f) { rc = launch_net(h, st, nullptr, nullptr); if (rc) return rc; }
  }
  CK(record_event(h, h->ev_b, st));
  h->net_launches_run = h->net_launch_idx;
  return CFRB_OK;
}

int cfrb_run(cfrb_handle* h, int32_t iters, void* cuda_stream) {
  if (!h || iters < 0) return fail(CFRB_EINVAL, "bad argument");
  if (h->cfg.net_mode != CFRB_NET_ZERO && !h->have_weights && h->Lmax > 0)
    return fail(CFRB_ESTATE, "value-net weights not set (cfrb_set_weights) but the subgame trees have non-final leaves");
  if (h->n == 0 || iters == 0) return CFRB_OK;
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
  if (st != h->own_stream && h->w_last) CK(cudaStreamWaitEvent(st, h->w_last, 0));   // weights are uploaded on the handle's own stream
  const int first = h->iters_done, last = first + iters;
  // Long runs are replayed from a CUDA graph: one host call instead of 2 * iters kernel launches, so a busy or slow host
  // thread cannot starve the GPU.  The graph bakes in the iteration indices and a wave-size-independent launch geometry; it
  // is keyed by (first iteration, count, profiling period, "the wave has value-net rows", "the wave has a schedule", "the wave keeps
  // the sum table").  The fp32 parity net sizes its grid by the row count and stays on the eager path, like short runs.
  static const bool no_graph = [] { const char* e = std::getenv("CFRB_NO_GRAPH"); return e && *e == '1'; }();
  const bool graphable = !no_graph && iters >= 64 && h->cfg.net_mode != CFRB_NET_FP32;
  if (graphable) {
    const int has_rows = h->rows > 0 || h->rows_on_device, sorted = h->sorted, keep_sum = !h->sum_dropped;
    cfrb_handle::GraphEntry* g = nullptr;
    for (auto& e : h->graphs)
      if (e.first == first && e.count == iters && e.prof == h->profiling && e.has_rows == has_rows && e.sorted == sorted &&
          e.keep_sum == keep_sum) { g = &e; break; }
    if (!g) {
      // capture + instantiation of ~2 * iters nodes costs ~0.1 s: only worth it for a key that repeats (waves of a self-play
      // loop, bench steps), not for one-off run lengths (e.g. the evaluator's per-chunk act_iteration maxima)
      const std::array<int, 6> key{first, iters, h->profiling, has_rows, sorted, keep_sum};
      bool seen = false;
      for (const auto& k : h->graph_seen) seen |= k == key;
      if (!seen) {
        if (h->graph_seen.size() >= 64) h->graph_seen.erase(h->graph_seen.begin());
        h->graph_seen.push_back(key);
      }
      if (seen) {
      if (h->profiling > 0) {   // events are created outside the capture
        const int rc = reserve_net_events(h, 2 * (iters / h->profiling + 2));
        if (rc) return rc;
      }
      const int64_t l0 = h->launches;
      GraphExec exec;
      h->capturing = true;
      cudaError_t ce = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
      int rc = CFRB_OK;
      if (ce == cudaSuccess) {
        rc = enqueue_run(h, st, first, last);
        Graph graph;
        ce = cudaStreamEndCapture(st, graph.put());
        if (rc == CFRB_OK && ce == cudaSuccess) ce = cudaGraphInstantiate(exec.put(), graph, 0);
      }
      h->capturing = false;
      const int captured = (int)(h->launches - l0);
      h->launches = l0;
      if (rc == CFRB_OK && ce == cudaSuccess && exec) {
        if (h->graphs.size() >= 8) h->graphs.erase(h->graphs.begin());
        h->graphs.push_back({first, iters, h->profiling, has_rows, sorted, keep_sum, std::move(exec), captured, h->net_launches_run,
                             h->net_ev_used});
        g = &h->graphs.back();
      } else {
        cudaGetLastError();   // the stream could not be captured (e.g. a legacy stream): run eagerly
      }
      }
    }
    if (g) {
      CK(cudaGraphLaunch(g->exec, st));
      h->launches += g->launches;
      h->net_launches_run = g->net_launches;
      h->net_ev_used = g->ev_used;
      h->iters_done = last;
      return CFRB_OK;
    }
  }
  int rc = enqueue_run(h, st, first, last);
  if (rc) return rc;
  h->iters_done = last;
  return CFRB_OK;
}

int cfrb_sync(cfrb_handle* h) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  return CFRB_OK;
}

int cfrb_iterations_done(const cfrb_handle* h) { return h ? h->iters_done : 0; }

int cfrb_fetch(cfrb_handle* h, double* root_value_means, double* snapshot_strategy, double* last_strategy, double* avg_strategy,
               double* sum_strategy, double* regrets) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  { int rc = sync_mirror(h); if (rc) return rc; }
  const int n = h->n;
  if (n == 0) return CFRB_OK;
  int rc = CFRB_OK;
  if (root_value_means && (rc = with_state(h, [&](auto& s) { return pull_reals(s.mu.p, (size_t)n * 2 * h->g.H, root_value_means); })))
    return rc;
  // The compact tables, expanded.  The average comes out as normalising the dense rows would give it: both sums add the legal
  // actions in the same order, and an illegal action only adds an exact +0.0 before or after them.
  const size_t dense_sz = (size_t)h->Nmax * h->g.H * h->g.A;
  std::vector<double> compact((size_t)n * h->table_stride);
  auto pull = [&](int which, double* dense) -> int {
    int rc = pull_table(h, which, compact.data());
    if (rc) return rc;
    for (int k = 0; k < n; ++k) to_dense(h, k, compact.data() + (size_t)k * h->table_stride, dense + (size_t)k * dense_sz);
    return CFRB_OK;
  };
  if (snapshot_strategy && (rc = pull(0, snapshot_strategy))) return rc;
  const bool fp = h->cfg.solver == CFRB_SOLVER_FP;   // FP: Sg = average_strategies, R = last_strategies
  if (last_strategy && (rc = pull(fp ? 3 : 1, last_strategy))) return rc;
  if (avg_strategy && (rc = pull(4, avg_strategy))) return rc;
  if (sum_strategy && (rc = pull(2, sum_strategy))) return rc;
  if (regrets && fp) std::fill(regrets, regrets + (size_t)n * dense_sz, 0.0);
  if (regrets && !fp && (rc = pull(3, regrets))) return rc;
  return CFRB_OK;
}

int cfrb_table_stride(const cfrb_handle* h) { return h ? h->table_stride : 0; }

int cfrb_fetch_compact(cfrb_handle* h, int32_t which, double* out) {
  if (!h || !out || which < 0 || which > 4) return fail(CFRB_EINVAL, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  { int rc = sync_mirror(h); if (rc) return rc; }
  if (h->n == 0) return CFRB_OK;
  return pull_table(h, which, out);
}

int cfrb_examples(cfrb_handle* h, float* queries, float* values) {
  if (!h || !queries || !values) return fail(CFRB_EINVAL, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  { int rc = sync_mirror(h); if (rc) return rc; }
  const int n = h->n, H = h->g.H, A = h->g.A, Q = h->g.Q;
  if (n == 0) return CFRB_OK;
  // std::copy_n into a float tensor, subgame_solving.cc:224
  int rc = with_state(h, [&](auto& s) { return pull_reals(s.mu.p, (size_t)n * 2 * H, values); });
  if (rc) return rc;
  // query of node 0 as seen by traverser t (write_query_to, subgame_solving.cc:104-123); root reach == beliefs
  for (int k = 0; k < n; ++k) {
    const double* b = h->h_beliefs.data() + (size_t)k * 2 * H;
    for (int t = 0; t < 2; ++t) {
      float* q = queries + ((size_t)k * 2 + t) * Q;
      q[0] = (float)h->h_player[k];
      q[1] = (float)t;
      for (int a = 0; a < A; ++a) q[2 + a] = (a == h->h_last_bid[k]) ? 1.f : 0.f;
      for (int p = 0; p < 2; ++p) {
        double s = 0;
        for (int hd = 0; hd < H; ++hd) s += b[p * H + hd] + 1e-80;
        for (int hd = 0; hd < H; ++hd) q[2 + A + p * H + hd] = (float)((b[p * H + hd] + 1e-80) / s);
      }
    }
  }
  return CFRB_OK;
}

int cfrb_load_state(cfrb_handle* h, const double* regrets, const double* last_strategy, const double* sum_strategy,
                    const double* root_value_means, const int32_t* num_steps, int32_t iterations_done) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  { int rc = sync_mirror(h); if (rc) return rc; }
  { int rc = materialise_sum(h); if (rc) return rc; }   // the tables it does not replace, S among them, stay the wave's
  int rc = with_state(h, [&](auto& s) { return load_state_t(h, s, regrets, last_strategy, sum_strategy, root_value_means); });
  if (rc) return rc;
  if (num_steps) CK(cudaMemcpy(h->d_steps.p, num_steps, (size_t)h->n * 2 * sizeof(int), cudaMemcpyHostToDevice));
  h->iters_done = iterations_done;
  return CFRB_OK;
}

int cfrb_debug_leaf_io(cfrb_handle* h, float* queries, float* net_out, double* scalers, int32_t cap_rows) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  { int rc = sync_mirror(h); if (rc) return rc; }
  const int rows = std::min<int>(h->rows, cap_rows), Q = h->g.Q;
  if (rows > 0 && queries && is_tc(h->cfg.net_mode)) {
    const int tiles = (rows + cfrb::tc::kTileM - 1) / cfrb::tc::kTileM;
    std::vector<__half> x((size_t)tiles * cfrb::tc::kTileM * h->Qpad);
    CK(cudaMemcpy(x.data(), h->d_Xh.p, x.size() * sizeof(__half), cudaMemcpyDeviceToHost));
    for (int r = 0; r < rows; ++r)
      for (int q = 0; q < Q; ++q)
        queries[(size_t)r * Q + q] = __half2float(x[(size_t)(r >> 7) * cfrb::tc::kTileM * h->Qpad +
                                                    cfrb::tc::umma_kmajor_offset_halves(r & 127, q, cfrb::tc::kTileM)]);
  } else if (rows > 0 && queries && h->cfg.net_mode == CFRB_NET_FP32) {
    std::vector<float> x((size_t)rows * h->Qpad);
    CK(cudaMemcpy(x.data(), h->d_X.p, x.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int r = 0; r < rows; ++r) std::memcpy(queries + (size_t)r * Q, x.data() + (size_t)r * h->Qpad, Q * sizeof(float));
  }
  if (rows > 0 && net_out) {
    std::vector<float> o((size_t)rows * h->Hout);
    CK(cudaMemcpy(o.data(), h->d_out.p, o.size() * sizeof(float), cudaMemcpyDeviceToHost));
    for (int r = 0; r < rows; ++r) std::memcpy(net_out + (size_t)r * h->g.H, o.data() + (size_t)r * h->Hout, h->g.H * sizeof(float));
  }
  if (rows > 0 && scalers) {
    int rc = with_state(h, [&](auto& s) { return pull_reals(s.scaler.p, rows, scalers); });
    if (rc) return rc;
  }
  return h->rows;
}

int cfrb_debug_net_trace(cfrb_handle* h, long long* out, int n) {
  if (!h || !is_tc(h->cfg.net_mode)) return fail(CFRB_EINVAL, "trace exists only for the tensor-core value net");
  if (!h->have_weights || h->rows == 0) return fail(CFRB_ESTATE, "no weights or no leaf rows");
  if (n < 2048) return fail(CFRB_EINVAL, "trace buffer must hold 2048 stamps");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  DevBuf<long long> d;
  CK(d.alloc(2048));
  CK(cudaMemset(d.p, 0, 2048 * sizeof(long long)));
  const int prof = h->profiling;
  h->profiling = 0;
  h->dbg_trace = d.p;
  int rc = launch_net(h, h->own_stream, nullptr, nullptr);
  h->dbg_trace = nullptr;
  h->profiling = prof;
  if (!rc && cudaStreamSynchronize(h->own_stream) != cudaSuccess) rc = fail(CFRB_ECUDA, "trace launch failed");
  if (!rc) cudaMemcpy(out, d.p, 2048 * sizeof(long long), cudaMemcpyDeviceToHost);
  return rc;
}

int cfrb_debug_net_taps(cfrb_handle* h, float* d1, float* d2) {
  if (!h || !is_tc(h->cfg.net_mode)) return fail(CFRB_EINVAL, "taps exist only for the tensor-core value net");
  if (!h->have_weights || h->rows == 0) return fail(CFRB_ESTATE, "no weights or no leaf rows");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const size_t n = (size_t)cfrb::tc::kTileM * cfrb::tc::kHid;
  const int prof = h->profiling;
  h->profiling = 0;
  int rc = launch_net(h, h->own_stream, h->d_dbg.p, h->d_dbg.p + n);
  h->profiling = prof;
  if (rc) return rc;
  CK(cudaStreamSynchronize(h->own_stream));
  if (d1) CK(cudaMemcpy(d1, h->d_dbg.p, n * sizeof(float), cudaMemcpyDeviceToHost));
  if (d2) CK(cudaMemcpy(d2, h->d_dbg.p + n, n * sizeof(float), cudaMemcpyDeviceToHost));
  return CFRB_OK;
}

// The full-depth tree rooted at the initial state (unroll_tree(game), tree.h:51-70) on the device, built on first use.
static int full_tree_setup(cfrb_handle* h, const char* who) {
  auto& b = h->br;
  const auto& g = h->g;
  if (b.ready) return CFRB_OK;
  if (g.A > 26) return fail(CFRB_EINVAL, std::string(who) + ": full tree too large (2^A - 1 nodes)");
  b.t = cfrb::build_template(g, -1, 1 << 30);
  const auto& t = b.t;
  std::vector<int> term(t.term_node.begin(), t.term_node.end());
  for (int n : t.term_node) term.push_back(t.last_bid[t.parent[n]]);   // challenged bid (:287)
  for (int n : t.term_node) term.push_back(t.depth[n]);
  auto up = [&](auto& buf, const auto& v) -> cudaError_t {
    cudaError_t e = buf.alloc(v.size());
    if (e != cudaSuccess) return e;
    return cudaMemcpy(buf.p, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice);
  };
  CK(up(b.parent, t.parent)); CK(up(b.child_begin, t.child_begin)); CK(up(b.nchild, t.nchild));
  CK(up(b.level_begin, t.level_begin)); CK(up(b.term_node, term)); CK(up(b.depth, t.depth)); CK(up(b.act_lo, t.act_lo));
  b.scratch_stride = (size_t)3 * t.N * g.H + (size_t)10 * std::max(t.T, 1);
  CK(b.scratch.alloc(2 * b.scratch_stride));
  CK(b.strategy.alloc((size_t)std::max(t.N - 1, 1) * g.H));
  CK(b.strategy2.alloc((size_t)std::max(t.N - 1, 1) * g.H));
  CK(b.out.alloc(2));
  b.ready = true;
  return CFRB_OK;
}

static cfrb::BrDev full_tree_dev(cfrb_handle* h) {
  const auto& b = h->br;
  const auto& t = b.t;
  cfrb::BrDev d{};
  d.N = t.N; d.T = t.T; d.levels = t.levels; d.H = h->g.H; d.F = h->g.F;
  d.parent = b.parent.p; d.child_begin = b.child_begin.p; d.nchild = b.nchild.p; d.level_begin = b.level_begin.p;
  d.term_node = b.term_node.p; d.matches = h->d_matches.p; d.strategy = b.strategy.p;
  d.scratch = b.scratch.p; d.scratch_stride = b.scratch_stride; d.out = b.out.p;
  return d;
}

// dense full-tree [n][h][a] -> compact [edge = child - 1][h] on the device
static int upload_compact(cfrb_handle* h, const double* dense, double* dst) {
  const auto& t = h->br.t;
  const auto& g = h->g;
  std::vector<double> compact((size_t)std::max(t.N - 1, 1) * g.H, 0.0);
  for (int n = 0; n < t.N; ++n)
    for (int j = 0; j < t.nchild[n]; ++j)
      for (int hd = 0; hd < g.H; ++hd)
        compact[(size_t)(t.child_begin[n] + j - 1) * g.H + hd] = dense[((size_t)n * g.H + hd) * g.A + t.act_lo[n] + j];
  CK(cudaMemcpyAsync(dst, compact.data(), compact.size() * sizeof(double), cudaMemcpyHostToDevice, h->own_stream));
  CK(cudaStreamSynchronize(h->own_stream));   // `compact` goes out of scope
  return CFRB_OK;
}

int cfrb_exploitability(cfrb_handle* h, const double* full_strategy, double* out2) {
  if (!h || !full_strategy || !out2) return fail(CFRB_EINVAL, "cfrb_exploitability: null argument");
  CK(cudaSetDevice(h->cfg.device));
  int rc = full_tree_setup(h, "cfrb_exploitability");
  if (!rc) rc = upload_compact(h, full_strategy, h->br.strategy.p);
  if (rc) return rc;
  cfrb::br_launch(full_tree_dev(h), h->own_stream);
  ++h->launches;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out2, h->br.out.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, h->own_stream));
  CK(cudaStreamSynchronize(h->own_stream));
  return CFRB_OK;
}

int cfrb_ev2(cfrb_handle* h, const double* s1_dense, const double* s2_dense, double* out2) {
  if (!h || !s1_dense || !s2_dense || !out2) return fail(CFRB_EINVAL, "cfrb_ev2: null argument");
  CK(cudaSetDevice(h->cfg.device));
  int rc = full_tree_setup(h, "cfrb_ev2");
  if (!rc) rc = upload_compact(h, s1_dense, h->br.strategy.p);
  if (!rc) rc = upload_compact(h, s2_dense, h->br.strategy2.p);
  if (rc) return rc;
  cfrb::ev_launch(full_tree_dev(h), h->br.strategy.p, h->br.strategy2.p, h->own_stream);
  ++h->launches;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out2, h->br.out.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, h->own_stream));
  CK(cudaStreamSynchronize(h->own_stream));
  return CFRB_OK;
}

int cfrb_full_tree_nodes(cfrb_handle* h) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  int rc = full_tree_setup(h, "cfrb_full_tree_nodes");
  return rc ? rc : h->br.t.N;
}

int cfrb_regrets_reset(cfrb_handle* h) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  int rc = full_tree_setup(h, "cfrb_regrets_reset");
  if (rc) return rc;
  auto& r = h->rg;
  const auto& t = h->br.t;
  if (!r.ready) {
    CK(r.acc.alloc((size_t)t.N * h->g.H * h->g.A));
    r.ready = true;
  }
  CK(cudaMemsetAsync(r.acc.p, 0, r.acc.n * sizeof(double), h->own_stream));
  CK(cudaStreamSynchronize(h->own_stream));
  r.count = 0;
  return CFRB_OK;
}

// Room for `S` strategies per batch: traverser values [S][2][N][H], reach scratch per (strategy, traverser), fp32 staging.
static int regrets_reserve(cfrb_handle* h, int S) {
  auto& r = h->rg;
  if (S <= r.cap) return CFRB_OK;
  const auto& t = h->br.t;
  const size_t NH = (size_t)t.N * h->g.H;
  CK(r.val.alloc((size_t)S * 2 * NH));
  CK(r.scratch.alloc((size_t)S * 2 * (2 * NH + (size_t)10 * std::max(t.T, 1))));
  CK(r.s32.alloc((size_t)S * std::max(t.N - 1, 1) * h->g.H));
  r.cap = S;
  return CFRB_OK;
}

static int regrets_launch(cfrb_handle* h, const float* s32, const double* s64, int S) {
  auto& r = h->rg;
  const auto& t = h->br.t;
  cfrb::RegretDev d{};
  d.tree = full_tree_dev(h);
  d.tree.scratch = r.scratch.p;
  d.tree.scratch_stride = 2 * (size_t)t.N * h->g.H + (size_t)10 * std::max(t.T, 1);
  d.depth = h->br.depth.p; d.act_lo = h->br.act_lo.p; d.A = h->g.A;
  d.s_stride = (size_t)std::max(t.N - 1, 1) * h->g.H;
  d.val = r.val.p; d.acc = r.acc.p;
  cfrb::regret_launch(d, s32, s64, S, h->own_stream);
  h->launches += 2;
  CK(cudaGetLastError());
  r.count += S;
  return CFRB_OK;
}

static constexpr int kRegretBatch = 64;

int cfrb_regrets_add(cfrb_handle* h, const float* compact, int32_t n) {
  if (!h || n < 0 || (n > 0 && !compact)) return fail(CFRB_EINVAL, "cfrb_regrets_add: bad argument");
  if (!h->rg.ready) return fail(CFRB_ESTATE, "cfrb_regrets_add: cfrb_regrets_reset has not been called");
  CK(cudaSetDevice(h->cfg.device));
  const size_t stride = (size_t)std::max(h->br.t.N - 1, 1) * h->g.H;
  for (int off = 0; off < n; off += kRegretBatch) {
    const int S = std::min(kRegretBatch, n - off);
    int rc = regrets_reserve(h, S);
    if (rc) return rc;
    CK(cudaMemcpyAsync(h->rg.s32.p, compact + (size_t)off * stride, (size_t)S * stride * sizeof(float), cudaMemcpyHostToDevice,
                       h->own_stream));
    if ((rc = regrets_launch(h, h->rg.s32.p, nullptr, S))) return rc;
    CK(cudaStreamSynchronize(h->own_stream));   // the host buffer and the staging area are reused
  }
  return CFRB_OK;
}

int cfrb_regrets_add_current(cfrb_handle* h) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  if (!h->rg.ready) return fail(CFRB_ESTATE, "cfrb_regrets_add_current: cfrb_regrets_reset has not been called");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());   // runs enqueued on other streams have finished before the table is read
  { int rc = sync_mirror(h); if (rc) return rc; }
  const auto& t = h->br.t;
  // subgame 0 must be the whole game: rooted at the initial state, player 0, with the full tree's node order
  if (h->n < 1 || h->h_tmpl[0] != 0 || h->h_player[0] != 0 || h->tmpl[0].N != t.N || h->tmpl[0].L != 0)
    return fail(CFRB_EINVAL, "cfrb_regrets_add_current: subgame 0 of the wave is not the full game tree");
  int rc = regrets_reserve(h, 1);
  if (rc) return rc;
  // the sampling strategy (CFR: last_strategies, FP: average_strategies) is the Sg table in both solvers, read in place
  if (h->f64) rc = regrets_launch(h, nullptr, h->sd.Sg.p, 1);
  else rc = regrets_launch(h, h->sf.Sg.p, nullptr, 1);
  return rc;
}

int cfrb_regrets_fetch(cfrb_handle* h, double* immediate, double* sums, int64_t* count) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  if (!h->rg.ready) return fail(CFRB_ESTATE, "cfrb_regrets_fetch: cfrb_regrets_reset has not been called");
  CK(cudaSetDevice(h->cfg.device));
  const int N = h->br.t.N, H = h->g.H, A = h->g.A;
  std::vector<double> acc((size_t)N * H * A);
  CK(cudaMemcpyAsync(acc.data(), h->rg.acc.p, acc.size() * sizeof(double), cudaMemcpyDeviceToHost, h->own_stream));
  CK(cudaStreamSynchronize(h->own_stream));
  if (sums) std::memcpy(sums, acc.data(), acc.size() * sizeof(double));
  if (count) *count = h->rg.count;
  if (immediate) {
    // max over all A actions (illegal ones stay 0) / number of strategies; 0 at leaves (subgame_solving.cc:1035-1048)
    const double cnt = (double)h->rg.count;
    for (int n = 0; n < N; ++n)
      for (int hd = 0; hd < H; ++hd) {
        const double* r = acc.data() + ((size_t)n * H + hd) * A;
        double m = r[0];
        for (int a = 1; a < A; ++a) if (m < r[a]) m = r[a];
        immediate[(size_t)n * H + hd] = h->br.t.nchild[n] ? m / cnt : 0.0;
      }
  }
  return CFRB_OK;
}

int64_t cfrb_kernel_launches(const cfrb_handle* h) { return h ? h->launches : 0; }
int64_t cfrb_wave_leaf_rows(const cfrb_handle* h) {
  if (!h) return 0;
  if (h->rows_on_device && h->mirror_stale) {   // a wave built on the device: the count lives there
    int wave[2] = {0, 0};
    cudaSetDevice(h->cfg.device);
    cudaDeviceSynchronize();
    if (cudaMemcpy(wave, h->d_wave.p, sizeof(wave), cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); return -1; }
    return wave[1];
  }
  return h->rows;
}

// Timing marks: CUDA events recorded on the launching stream (NULL = the handle's stream); elapsed device time between two.
int cfrb_mark(cfrb_handle* h, int32_t slot, void* cuda_stream) {
  if (!h || slot < 0 || slot >= 8) return fail(CFRB_EINVAL, "cfrb_mark: slot must be in [0, 8)");
  CK(cudaSetDevice(h->cfg.device));
  if (!h->marks[slot]) CK(cudaEventCreate(h->marks[slot].put()));
  CK(cudaEventRecord(h->marks[slot], cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream));
  return CFRB_OK;
}
int cfrb_mark_wait(cfrb_handle* h, int32_t slot) {
  if (!h || slot < 0 || slot >= 8 || !h->marks[slot]) return fail(CFRB_EINVAL, "cfrb_mark_wait: mark not recorded");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->marks[slot]));
  return CFRB_OK;
}
void* cfrb_handle_stream(cfrb_handle* h) { return h ? (void*)h->own_stream.get() : nullptr; }
int cfrb_mark_elapsed_ms(cfrb_handle* h, int32_t a, int32_t b, float* ms) {
  if (!h || !ms || a < 0 || a >= 8 || b < 0 || b >= 8 || !h->marks[a] || !h->marks[b]) return fail(CFRB_EINVAL, "cfrb_mark_elapsed_ms: bad marks");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->marks[b]));
  CK(cudaEventElapsedTime(ms, h->marks[a], h->marks[b]));
  return CFRB_OK;
}
// Evict the L2 cache: overwrite a scratch buffer of `bytes` (> the 50 MB L2 of an H100) on the stream, for benchmarks' timed loops.
int cfrb_l2_flush(cfrb_handle* h, size_t bytes, void* cuda_stream) {
  if (!h || bytes == 0) return fail(CFRB_EINVAL, "cfrb_l2_flush: bad argument");
  CK(cudaSetDevice(h->cfg.device));
  if (h->flush_buf.n < bytes) CK(h->flush_buf.alloc(bytes));
  CK(cudaMemsetAsync(h->flush_buf.p, 1, bytes, cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream));
  return CFRB_OK;
}

int cfrb_last_run_ms(cfrb_handle* h, float* total_ms, float* net_ms) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->ev_b));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, h->ev_a, h->ev_b));
  h->last_total_ms = ms;
  float net = 0.f;
  for (int i = 0; i + 1 < h->net_ev_used; i += 2) {
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, h->net_ev[i], h->net_ev[i + 1]));
    net += t;
  }
  // sampled launches -> estimate for all value-net launches of the run
  if (h->net_ev_used > 0) net = net / (h->net_ev_used / 2) * h->net_launches_run;
  h->last_net_ms = net;
  if (total_ms) *total_ms = ms;
  if (net_ms) *net_ms = net;
  return CFRB_OK;
}

// Starts a wave of n subgames built on the device (its leaf rows and roots exist only there) and runs num_iters on it.  sorted:
// d_sg_order holds the wave's schedule; otherwise the depth-2 kernel takes wave order.  drop_sum: a self-play wave, whose loop
// reads the snapshots and root means only; CFR then leaves the sum table alone (materialise_sum rebuilds it for a reader).  Match,
// LBR and agent waves keep it: they act with the average strategy of the wave they have just solved (act_slot).
static int solve_device_wave(cfrb_handle* h, int n, bool sorted, bool drop_sum, cudaStream_t st) {
  h->n = n; h->rows = 0; h->rows_on_device = true; h->mirror_stale = true; h->iters_done = 0; h->sp.pending = false;
  h->sorted = sorted;
  h->sum_dropped = drop_sum && h->cfg.solver == CFRB_SOLVER_CFR;
  h->sum_uploads = h->weight_uploads;
  const int rc = launch_init(h, st);
  return rc ? rc : cfrb_run(h, h->cfg.num_iters, st);
}

// ============================================================================================ recursive to-leaf exploitability
// Sizes of the device walk from the game alone.  The full tree has 2^A - 1 nodes, 2^(A-1) - 1 of them terminal (liar calls), and
// C(A - 1, d) non-terminal nodes at depth d (d increasing bids out of the A - 1), so level l of the walk holds C(A - 1, l * max_depth)
// subgames.  The largest subgame template, the game root's, has A - 1 nodes at depth 1 and C(A, d) at depth d >= 2.
static int64_t binom(int n, int k) {
  if (k < 0 || k > n) return 0;
  int64_t r = 1;
  for (int i = 1; i <= k; ++i) r = r * (n - k + i) / i;
  return r;
}
struct ToLeafSizes { int64_t tree_bytes = 0, walk_bytes = 0, level_cap = 0; };
static ToLeafSizes to_leaf_sizes(const cfrb::GameShape& g, int max_depth, int K) {
  const int A = g.A;
  const int64_t H = g.H, N = ((int64_t)1 << A) - 1, T = ((int64_t)1 << (A - 1)) - 1, levels = A + 1;
  ToLeafSizes s;
  // full_tree_setup: parent, child_begin, nchild, depth, act_lo [N], level_begin [levels + 1] and term_node [3][T] ints; two
  // strategies [N - 1][H], the best-response scratch 2 x (3 N H + 10 T) and out [2] doubles
  s.tree_bytes = (5 * N + levels + 1 + 3 * T) * 4 + (2 * (N - 1) * H + 2 * (3 * N * H + 10 * T) + 2) * 8;
  int64_t nmax = 1;
  for (int d = 1; d <= std::min(max_depth, A); ++d) nmax += d == 1 ? A - 1 : binom(A, d);
  for (int d = 0; d <= A - 1; d += max_depth) s.level_cap = std::max(s.level_cap, binom(A - 1, d));
  // the template-to-full-tree map [K][nmax], and two levels of roots and fp64 beliefs [2][H]
  s.walk_bytes = (int64_t)K * nmax * 4 + 2 * s.level_cap * (4 + 2 * H * 8);
  return s;
}

int64_t cfrb_to_leaf_bytes(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t max_subgames) {
  if (num_dice < 1 || num_faces < 1 || max_depth < 1 || max_subgames < 1)
    return fail(CFRB_EINVAL, "cfrb_to_leaf_bytes: num_dice, num_faces, max_depth, max_subgames must be >= 1");
  if (2L * num_dice * num_faces + 1 > 26) return fail(CFRB_EINVAL, "cfrb_to_leaf_bytes: full tree too large (2^A - 1 nodes, A > 26)");
  const auto s = to_leaf_sizes(cfrb::GameShape(num_dice, num_faces), max_depth, max_subgames);
  return s.tree_bytes + s.walk_bytes;
}

int cfrb_debug_to_leaf_free_cap(cfrb_handle* h, int64_t bytes) {
  if (!h || bytes < 0) return fail(CFRB_EINVAL, "cfrb_debug_to_leaf_free_cap: bad argument");
  h->to_leaf_free_cap = bytes;
  return CFRB_OK;
}

int cfrb_to_leaf_exploitability(cfrb_handle* h, double* br_out2, int64_t* subgames, int64_t* subgame_iters, double* seconds2) {
  if (!h || !br_out2) return fail(CFRB_EINVAL, "cfrb_to_leaf_exploitability: null argument");
  const auto& g = h->g;
  if (g.A > CFRB_TO_LEAF_MAX_ACTIONS)
    return fail(CFRB_EINVAL, "cfrb_to_leaf_exploitability: games with more than " + std::to_string(CFRB_TO_LEAF_MAX_ACTIONS) +
                                 " actions are not supported (A = " + std::to_string(g.A) + ": the full tree has 2^A - 1 nodes)");
  if (h->in_match) return fail(CFRB_EINVAL, "cfrb_to_leaf_exploitability: the handle plays in a live match or agent");
  if (h->cfg.net_mode != CFRB_NET_ZERO && !h->have_weights && h->Lmax > 0)
    return fail(CFRB_ESTATE, "cfrb_to_leaf_exploitability: value-net weights not set (cfrb_set_weights)");
  CK(cudaSetDevice(h->cfg.device));
  const int K = h->cfg.max_subgames, H = g.H, W = 2 * H;
  const auto sz = to_leaf_sizes(g, h->cfg.max_depth, K);
  // refused before anything is allocated: on a shared device an allocation that fails late may starve other processes
  const int64_t need = (h->br.ready ? 0 : sz.tree_bytes) + sz.walk_bytes;
  size_t free_b = 0, total_b = 0;
  CK(cudaMemGetInfo(&free_b, &total_b));
  int64_t avail = (int64_t)free_b;
  if (h->to_leaf_free_cap > 0) avail = std::min(avail, h->to_leaf_free_cap);
  if (need > avail)
    return fail(CFRB_ENOMEM, "cfrb_to_leaf_exploitability: needs " + std::to_string(need) + " bytes of device memory beyond the "
                             "handle (full tree and best-response scratch " + std::to_string(h->br.ready ? 0 : sz.tree_bytes) +
                             ", walk " + std::to_string(sz.walk_bytes) + "), " + std::to_string(avail) + " free");
  int rc = full_tree_setup(h, "cfrb_to_leaf_exploitability");
  if (rc) return rc;
  cudaStream_t st = h->own_stream;
  DevBuf<int> roots[2], fid, fill;
  DevBuf<double> bel[2];
  for (int i = 0; i < 2; ++i) { CK(roots[i].alloc(sz.level_cap)); CK(bel[i].alloc((size_t)sz.level_cap * W)); }
  CK(fid.alloc((size_t)K * h->Nmax)); CK(fill.alloc(1));
  const auto t0 = std::chrono::steady_clock::now();
  const std::vector<double> uniform(W, 1.0 / H);   // level 0: the game root with uniform beliefs
  const int root = 0;
  CK(cudaMemcpyAsync(roots[0].p, &root, sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(bel[0].p, uniform.data(), W * sizeof(double), cudaMemcpyHostToDevice, st));
  cfrb::ExplDev d{};
  d.H = H;
  d.full_child_begin = h->br.child_begin.p; d.full_depth = h->br.depth.p; d.full_act_lo = h->br.act_lo.p; d.strategy = h->br.strategy.p;
  d.tmpl = h->d_tmpl.p; d.parent = h->d_parent.p; d.child_begin = h->d_child_begin.p; d.nchild = h->d_nchild.p;
  d.level_begin = h->d_level_begin.p; d.pleaf_node = h->d_pleaf_node.p;
  d.sg_tmpl = h->d_sg_tmpl.p; d.sg_player = h->d_sg_player.p; d.sg_act = h->d_sg_act.p; d.sg_row_off = h->d_sg_row_off.p;
  d.wave = h->d_wave.p; d.steps = h->d_steps.p; d.table_stride = h->table_stride;
  d.fill = fill.p; d.cap = (int)sz.level_cap; d.fid = fid.p; d.nmax = h->Nmax;
  cfrb::SpDev scan{};   // sp_scan_kernel's view of the wave
  scan.A = g.A; scan.tmpl = h->d_tmpl.p; scan.wave = h->d_wave.p; scan.sg_tmpl = h->d_sg_tmpl.p; scan.sg_row_off = h->d_sg_row_off.p;
  scan.sg_order = h->d_sg_order.p; scan.tmpl_rank = h->d_tmpl_rank.p;
  int64_t solved = 0;
  int cur = 0, n_level = 1;
  for (int depth = 0; n_level > 0; depth += h->cfg.max_depth) {
    d.roots = roots[cur].p; d.bel = bel[cur].p; d.next_roots = roots[cur ^ 1].p; d.next_bel = bel[cur ^ 1].p;
    CK(cudaMemsetAsync(fill.p, 0, sizeof(int), st));
    for (int off = 0; off < n_level; off += K) {
      const int n = std::min(K, n_level - off);
      d.off = off; scan.K = n;
      with_state(h, [&](auto& s) { cfrb::expl_launch_begin(d, scan, n, s.beliefs.p, st); });
      h->launches += 2;
      CK(cudaGetLastError());
      if ((rc = solve_device_wave(h, n, true, false, st))) return rc;
      with_state(h, [&](auto& s) {
        const auto avg = avg_table(h, s);
        cfrb::expl_launch_expand(d, n, avg.p, avg.normalise ? 1 : 0, st);
      });
      h->launches += 2;
      CK(cudaGetLastError());
    }
    solved += n_level;
    int next = 0;
    CK(cudaMemcpyAsync(&next, fill.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (next != binom(g.A - 1, depth + h->cfg.max_depth))
      return fail(CFRB_ECUDA, "cfrb_to_leaf_exploitability: level at depth " + std::to_string(depth + h->cfg.max_depth) + " has " +
                                  std::to_string(next) + " subgames, the tree " + std::to_string(binom(g.A - 1, depth + h->cfg.max_depth)));
    n_level = next;
    cur ^= 1;
  }
  const auto t1 = std::chrono::steady_clock::now();
  cfrb::br_launch(full_tree_dev(h), st);
  ++h->launches;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(br_out2, h->br.out.p, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const auto t2 = std::chrono::steady_clock::now();
  if (subgames) *subgames = solved;
  if (subgame_iters) *subgame_iters = solved * h->cfg.num_iters;
  if (seconds2) {
    seconds2[0] = std::chrono::duration<double>(t1 - t0).count();
    seconds2[1] = std::chrono::duration<double>(t2 - t1).count();
  }
  return CFRB_OK;
}

int cfrb_to_leaf_strategy(cfrb_handle* h, double* compact) {
  if (!h || !compact) return fail(CFRB_EINVAL, "cfrb_to_leaf_strategy: null argument");
  if (!h->br.ready) return fail(CFRB_ESTATE, "cfrb_to_leaf_strategy: the handle holds no full-tree strategy (run cfrb_to_leaf_exploitability)");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->own_stream));
  CK(cudaMemcpy(compact, h->br.strategy.p, h->br.strategy.n * sizeof(double), cudaMemcpyDeviceToHost));
  return CFRB_OK;
}

// ============================================================================================ device-resident self-play
int cfrb_selfplay_create(cfrb_handle* h, int32_t n_games, const uint32_t* seeds, float random_action_prob, int32_t sample_leaf) {
  if (!h || !seeds) return fail(CFRB_EINVAL, "null argument");
  if (n_games < 1 || n_games > h->cfg.max_subgames) return fail(CFRB_EINVAL, "n_games must be in [1, max_subgames]");
  if (h->g.H > cfrb::kSpMaxH) return fail(CFRB_EINVAL, "device self-play supports num_hands <= 64");
  if (h->cfg.max_depth > cfrb::kSpMaxPath) return fail(CFRB_EINVAL, "device self-play supports max_depth <= 16");
  CK(cudaSetDevice(h->cfg.device));
  auto& sp = h->sp;
  const int K = n_games, H = h->g.H;
  CK(sp.last_bid.alloc(K)); CK(sp.player.alloc(K)); CK(sp.mt_idx.alloc(K)); CK(sp.beliefs.alloc((size_t)K * 2 * H));
  CK(sp.mt.alloc((size_t)624 * K)); CK(sp.seeds.alloc(K));
  cfrb::SpDev& d = sp.dev;
  d.K = K; d.A = h->g.A; d.H = H; d.Q = h->g.Q; d.iters = h->cfg.num_iters; d.sample_leaf = sample_leaf;
  d.random_action_prob = random_action_prob;
  d.g_last_bid = sp.last_bid.p; d.g_player = sp.player.p; d.g_beliefs = sp.beliefs.p; d.mt = sp.mt.p; d.mt_idx = sp.mt_idx.p;
  d.tmpl = h->d_tmpl.p; d.child_begin = h->d_child_begin.p; d.nchild = h->d_nchild.p; d.last_bid = h->d_last_bid.p;
  d.wave = h->d_wave.p; d.sg_tmpl = h->d_sg_tmpl.p; d.sg_player = h->d_sg_player.p; d.sg_row_off = h->d_sg_row_off.p;
  d.sg_act = h->d_sg_act.p; d.table_stride = h->table_stride;
  d.sg_order = h->d_sg_order.p; d.tmpl_rank = h->d_tmpl_rank.p;
  CK(cudaStreamSynchronize(h->own_stream));
  CK(cudaMemcpyAsync(sp.seeds.p, seeds, (size_t)K * sizeof(uint32_t), cudaMemcpyHostToDevice, h->own_stream));
  cfrb::sp_launch_seed(d, sp.seeds.p, h->own_stream);
  ++h->launches;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(h->own_stream));
  if (!sp.ev_examples) CK(cudaEventCreateWithFlags(sp.ev_examples.put(), cudaEventDisableTiming));
  sp.K = K; sp.ready = true; sp.pending = false; sp.waves = 0; sp.ev_recorded = false;
  return CFRB_OK;
}

int cfrb_selfplay_wave(cfrb_handle* h, float* dev_ex_q, float* dev_ex_v, int32_t start_next, void* cuda_stream) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  if (!h->sp.ready) return fail(CFRB_ESTATE, "cfrb_selfplay_create has not been called");
  if ((dev_ex_q == nullptr) != (dev_ex_v == nullptr)) return fail(CFRB_EINVAL, "example buffers: both or none");
  CK(cudaSetDevice(h->cfg.device));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
  int rows_out = 0;
  if (h->sp.pending) {
    if (!h->rows_on_device || h->n != h->sp.K || h->iters_done != h->cfg.num_iters)
      return fail(CFRB_ESTATE, "the pending self-play wave was replaced or not run to num_iters");
    with_state(h, [&](auto& s) { cfrb::sp_launch_finish(h->sp.dev, s.mu.p, s.Snap.p, dev_ex_q, dev_ex_v, st); });
    h->launches += dev_ex_q ? 2 : 1;
    CK(cudaGetLastError());
    h->sp.pending = false;
    rows_out = dev_ex_q ? 2 * h->sp.K : 0;
    CK(cudaEventRecord(h->sp.ev_examples, st));
    h->sp.ev_recorded = true;
  }
  if (start_next) {
    with_state(h, [&](auto& s) { cfrb::sp_launch_begin(h->sp.dev, s.beliefs.p, st); });
    h->launches += 2;
    CK(cudaGetLastError());
    const int rc = solve_device_wave(h, h->sp.K, true, true, st);
    if (rc) return rc;
    h->sp.pending = true;
    ++h->sp.waves;
  }
  return rows_out;
}

int cfrb_selfplay_wait_examples(cfrb_handle* h) {
  if (!h || !h->sp.ready) return fail(CFRB_ESTATE, "no self-play session");
  if (!h->sp.ev_recorded) return CFRB_OK;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaEventSynchronize(h->sp.ev_examples));
  return CFRB_OK;
}

int cfrb_selfplay_state(cfrb_handle* h, int32_t* last_bid, int32_t* player, double* beliefs) {
  if (!h || !h->sp.ready) return fail(CFRB_ESTATE, "no self-play session");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const int K = h->sp.K;
  if (last_bid) CK(cudaMemcpy(last_bid, h->sp.last_bid.p, K * sizeof(int), cudaMemcpyDeviceToHost));
  if (player) CK(cudaMemcpy(player, h->sp.player.p, K * sizeof(int), cudaMemcpyDeviceToHost));
  if (beliefs) CK(cudaMemcpy(beliefs, h->sp.beliefs.p, (size_t)K * 2 * h->g.H * sizeof(double), cudaMemcpyDeviceToHost));
  return K;
}

// Session image of cfrb_selfplay_export / _import: this header, then beliefs f64 [K][2][H], mt u32 [624][K], last_bid i32 [K],
// player i32 [K], mt_idx i32 [K].  Host byte order.
namespace {
constexpr uint32_t kSpMagic = 0x50534643u;   // "CFSP"
constexpr uint32_t kSpVersion = 1;
struct SpImageHeader {
  uint32_t magic, version;
  int32_t num_dice, num_faces, n_games, num_hands, sample_leaf;
  uint32_t random_action_prob_bits;
  int64_t waves;
};
static_assert(sizeof(SpImageHeader) == 40, "session image header layout");

size_t sp_image_bytes(int K, int H) {
  return sizeof(SpImageHeader) + (size_t)K * 2 * H * sizeof(double) + (size_t)624 * K * sizeof(uint32_t) + (size_t)3 * K * sizeof(int32_t);
}
SpImageHeader sp_image_header(const cfrb_handle* h) {
  SpImageHeader hd{kSpMagic, kSpVersion, h->cfg.num_dice, h->cfg.num_faces, h->sp.K, h->g.H, h->sp.dev.sample_leaf, 0, h->sp.waves};
  std::memcpy(&hd.random_action_prob_bits, &h->sp.dev.random_action_prob, sizeof(float));
  return hd;
}
}  // namespace

int64_t cfrb_selfplay_export(cfrb_handle* h, void* out, size_t cap) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  if (!h->sp.ready) return fail(CFRB_ESTATE, "cfrb_selfplay_export: no self-play session (cfrb_selfplay_create)");
  if (h->sp.pending)
    return fail(CFRB_ESTATE, "cfrb_selfplay_export: a wave is pending; drain it first with cfrb_selfplay_wave(..., start_next=0)");
  const int K = h->sp.K, H = h->g.H;
  const size_t bytes = sp_image_bytes(K, H);
  if (!out) return (int64_t)bytes;
  if (cap < bytes) return fail(CFRB_EINVAL, "cfrb_selfplay_export: buffer of " + std::to_string(cap) + " bytes, the session needs " + std::to_string(bytes));
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const SpImageHeader hd = sp_image_header(h);
  char* p = static_cast<char*>(out);
  std::memcpy(p, &hd, sizeof hd); p += sizeof hd;
  CK(cudaMemcpy(p, h->sp.beliefs.p, (size_t)K * 2 * H * sizeof(double), cudaMemcpyDeviceToHost)); p += (size_t)K * 2 * H * sizeof(double);
  CK(cudaMemcpy(p, h->sp.mt.p, (size_t)624 * K * sizeof(uint32_t), cudaMemcpyDeviceToHost)); p += (size_t)624 * K * sizeof(uint32_t);
  CK(cudaMemcpy(p, h->sp.last_bid.p, K * sizeof(int32_t), cudaMemcpyDeviceToHost)); p += K * sizeof(int32_t);
  CK(cudaMemcpy(p, h->sp.player.p, K * sizeof(int32_t), cudaMemcpyDeviceToHost)); p += K * sizeof(int32_t);
  CK(cudaMemcpy(p, h->sp.mt_idx.p, K * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return (int64_t)bytes;
}

int cfrb_selfplay_import(cfrb_handle* h, const void* in, size_t bytes) {
  if (!h || !in) return fail(CFRB_EINVAL, "null argument");
  if (!h->sp.ready) return fail(CFRB_ESTATE, "cfrb_selfplay_import: no self-play session (call cfrb_selfplay_create with the same n_games first)");
  if (h->sp.pending)
    return fail(CFRB_ESTATE, "cfrb_selfplay_import: a wave is pending; drain it first with cfrb_selfplay_wave(..., start_next=0)");
  // Everything is checked on the host before the device is touched: a refused image leaves the session as it was.
  const int K = h->sp.K, H = h->g.H, A = h->g.A;
  if (bytes < sizeof(SpImageHeader)) return fail(CFRB_EINVAL, "cfrb_selfplay_import: " + std::to_string(bytes) + " bytes is shorter than the header");
  SpImageHeader hd;
  std::memcpy(&hd, in, sizeof hd);
  const SpImageHeader want = sp_image_header(h);
  auto field = [](const char* name, int64_t got, int64_t exp) {
    return fail(CFRB_EINVAL, std::string("cfrb_selfplay_import: ") + name + " is " + std::to_string(got) + ", this session has " + std::to_string(exp));
  };
  if (hd.magic != kSpMagic) return fail(CFRB_EINVAL, "cfrb_selfplay_import: not a self-play session image (bad magic)");
  if (hd.version != kSpVersion) return field("format version", hd.version, kSpVersion);
  if (hd.num_dice != want.num_dice) return field("num_dice", hd.num_dice, want.num_dice);
  if (hd.num_faces != want.num_faces) return field("num_faces", hd.num_faces, want.num_faces);
  if (hd.n_games != want.n_games) return field("n_games", hd.n_games, want.n_games);
  if (hd.num_hands != want.num_hands) return field("num_hands", hd.num_hands, want.num_hands);
  if (hd.sample_leaf != want.sample_leaf) return field("sample_leaf", hd.sample_leaf, want.sample_leaf);
  if (hd.random_action_prob_bits != want.random_action_prob_bits) {
    float got, exp;
    std::memcpy(&got, &hd.random_action_prob_bits, 4); std::memcpy(&exp, &want.random_action_prob_bits, 4);
    return fail(CFRB_EINVAL, "cfrb_selfplay_import: random_action_prob is " + std::to_string(got) + ", this session has " + std::to_string(exp));
  }
  if (hd.waves < 0) return field("wave count", hd.waves, 0);
  const size_t need = sp_image_bytes(K, H);
  if (bytes != need) return fail(CFRB_EINVAL, "cfrb_selfplay_import: " + std::to_string(bytes) + " bytes, the image of this session has " + std::to_string(need));
  const char* p = static_cast<const char*>(in) + sizeof hd;
  std::vector<double> bel((size_t)K * 2 * H);
  std::vector<uint32_t> mt((size_t)624 * K);
  std::vector<int32_t> last_bid(K), player(K), mt_idx(K);
  std::memcpy(bel.data(), p, bel.size() * sizeof(double)); p += bel.size() * sizeof(double);
  std::memcpy(mt.data(), p, mt.size() * sizeof(uint32_t)); p += mt.size() * sizeof(uint32_t);
  std::memcpy(last_bid.data(), p, K * sizeof(int32_t)); p += K * sizeof(int32_t);
  std::memcpy(player.data(), p, K * sizeof(int32_t)); p += K * sizeof(int32_t);
  std::memcpy(mt_idx.data(), p, K * sizeof(int32_t));
  for (int g = 0; g < K; ++g) {
    const std::string at = " of game " + std::to_string(g);
    if (mt_idx[g] < 0 || mt_idx[g] > 624) return fail(CFRB_EINVAL, "cfrb_selfplay_import: mt_idx" + at + " is " + std::to_string(mt_idx[g]) + ", outside [0, 624]");
    if (player[g] != 0 && player[g] != 1) return fail(CFRB_EINVAL, "cfrb_selfplay_import: player" + at + " is " + std::to_string(player[g]) + ", not 0 or 1");
    // the walk leaves a game at the initial state (-1, player 0) or after a non-terminal bid; a liar call restarts the game
    if (last_bid[g] < -1 || last_bid[g] > A - 2 || (last_bid[g] == -1 && player[g] != 0))
      return fail(CFRB_EINVAL, "cfrb_selfplay_import: last_bid " + std::to_string(last_bid[g]) + " with player " + std::to_string(player[g]) + at +
                                   " is not a state the walk produces (last_bid in [-1, " + std::to_string(A - 2) + "], player 0 at -1)");
    for (int i = 0; i < 2 * H; ++i) {
      const double b = bel[(size_t)g * 2 * H + i];
      if (!std::isfinite(b) || b < 0) return fail(CFRB_EINVAL, "cfrb_selfplay_import: belief " + std::to_string(i) + at + " is " + std::to_string(b));
    }
  }
  // Device-wide synchronisation on both sides: a finish kernel of the last wave may still be writing the session on a caller's
  // stream, and copies from pageable memory may return before their DMA lands, while the next wave starts on the non-blocking
  // own_stream.
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h->sp.beliefs.p, bel.data(), bel.size() * sizeof(double), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->sp.mt.p, mt.data(), mt.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->sp.last_bid.p, last_bid.data(), K * sizeof(int32_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->sp.player.p, player.data(), K * sizeof(int32_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->sp.mt_idx.p, mt_idx.data(), K * sizeof(int32_t), cudaMemcpyHostToDevice));
  CK(cudaDeviceSynchronize());
  h->sp.waves = hd.waves;
  h->sp.ev_recorded = false;
  // The handle holds no wave, as after cfrb_create: the readers of a solved wave (cfrb_fetch, the sum rebuild, ...) find none.
  h->n = 0; h->rows = 0; h->iters_done = 0; h->rows_on_device = false; h->mirror_stale = false; h->sum_dropped = false;
  return CFRB_OK;
}

// Roots of the current wave (inspection; pulls the descriptors of a device-built wave).  Returns the number of subgames.
int cfrb_wave_roots(cfrb_handle* h, int32_t* last_bid, int32_t* player_id, int32_t cap) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  { int rc = sync_mirror(h); if (rc) return rc; }
  for (int k = 0; k < h->n && k < cap; ++k) {
    if (last_bid) last_bid[k] = h->h_last_bid[k];
    if (player_id) player_id[k] = h->h_player[k];
  }
  return h->n;
}

int cfrb_wave_order(cfrb_handle* h, int32_t* order, int32_t cap) {
  if (!h || !order) return fail(CFRB_EINVAL, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const int n = std::min(h->n, (int)std::max(cap, 0));
  if (h->sorted) CK(cudaMemcpy(order, h->d_sg_order.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  else for (int k = 0; k < n; ++k) order[k] = k;
  return h->n;
}

int cfrb_schedule_order(int32_t num_dice, int32_t num_faces, int32_t max_depth, int32_t n, const int32_t* last_bid, int32_t* order,
                        int64_t* cost) {
  if (num_dice < 1 || num_faces < 1 || max_depth < 1 || n < 0 || (n > 0 && (!last_bid || !order))) return fail(CFRB_EINVAL, "bad argument");
  const cfrb::GameShape g(num_dice, num_faces);
  std::vector<cfrb::TreeTemplate> tmpl;
  for (int rb = -1; rb <= g.A - 2; ++rb) tmpl.push_back(cfrb::build_template(g, rb, max_depth));
  std::vector<int> tm(n);
  for (int k = 0; k < n; ++k) {
    if (last_bid[k] < -1 || last_bid[k] > g.A - 2) return fail(CFRB_EINVAL, "subgame root bid out of range (terminal or invalid)");
    tm[k] = last_bid[k] + 1;
    if (cost) cost[k] = cfrb::schedule_cost(tmpl[tm[k]], g.H);
  }
  cfrb::schedule_order(cfrb::schedule_ranks(tmpl, g.H), tm.data(), n, order);
  return CFRB_OK;
}

// Test aid: a persistent grid of at most max_ctas CTAs makes every warp of the depth-2 kernel solve many subgames per launch.
// Graphs bake the grid in, so they are dropped.
int cfrb_debug_d2_grid(cfrb_handle* h, int32_t max_ctas) {
  if (!h || max_ctas < 0) return fail(CFRB_EINVAL, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  h->graphs.clear(); h->graph_seen.clear();
  h->d2_grid_cap = max_ctas;
  return h->d2_ctas;
}

// Development / test aid: div_by_rcp (reciprocal + two fused-multiply-add corrections, cfr_kernels.cuh; the regret matching of
// cfr_iter_d2_kernel) against IEEE division on `blocks` x 256 x 4096 pseudo-random operand pairs; *mismatches receives the number
// of differing quotients.
int cfrb_debug_div_check(cfrb_handle* h, uint64_t seed, int32_t blocks, uint64_t* mismatches) {
  if (!h || !mismatches || blocks < 1) return fail(CFRB_EINVAL, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  DevBuf<unsigned long long> d;
  CK(d.alloc(1));
  CK(cudaMemset(d.p, 0, sizeof(unsigned long long)));
  cfrb::div_check_launch(seed, blocks, d.p, h->own_stream);
  cudaError_t e = cudaStreamSynchronize(h->own_stream);
  unsigned long long out = 0;
  if (e == cudaSuccess) e = cudaMemcpy(&out, d.p, sizeof(out), cudaMemcpyDeviceToHost);
  CK(e);
  *mismatches = out;
  return CFRB_OK;
}

// Development / test aid: what the packed-half GELU of the value-net epilogue computes, for every fp16 input.  what = 0:
// tanh.approx.f16x2 itself; 1 / 2: gelu_hy_x2 / gelu_hy_t32 with hy = the input (leaf_mlp_tc.cuh).  out[i] = fp16 bits of f(fp16 with bits i).
namespace {
__global__ void gelu_table_kernel(int what, unsigned short* out) {
  const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 65536u) return;
  const __half x = __ushort_as_half((unsigned short)i);
  unsigned short r;
  if (what == 0) {
    const __half2 u = __halves2half2(x, x);
    uint32_t t;
    asm("tanh.approx.f16x2 %0, %1;" : "=r"(t) : "r"(*reinterpret_cast<const uint32_t*>(&u)));
    r = (unsigned short)(t & 0xffffu);
  } else {
    const float f = __half2float(x);
    r = (unsigned short)((what == 1 ? cfrb::tc::gelu_hy_x2(f, f) : cfrb::tc::gelu_hy_t32(f, f)) & 0xffffu);
  }
  out[i] = r;
}
}  // namespace
int cfrb_debug_gelu_table(cfrb_handle* h, int32_t what, uint16_t* out) {
  if (!h || !out || what < 0 || what > 2) return fail(CFRB_EINVAL, "bad argument");
  CK(cudaSetDevice(h->cfg.device));
  DevBuf<unsigned short> d;
  CK(d.alloc(65536));
  gelu_table_kernel<<<256, 256, 0, h->own_stream>>>(what, d.p);
  cudaError_t e = cudaStreamSynchronize(h->own_stream);
  if (e == cudaSuccess) e = cudaMemcpy(out, d.p, 65536 * sizeof(unsigned short), cudaMemcpyDeviceToHost);
  CK(e);
  return CFRB_OK;
}

int cfrb_stream_wait(cfrb_handle* h, void* cuda_stream) {
  if (!h) return fail(CFRB_EINVAL, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream));
  return CFRB_OK;
}

}  // extern "C"

// ============================================================================================ head-to-head matches
struct cfrb_match {
  cfrb_handle* h[2] = {nullptr, nullptr};
  int S = 0, G = 0, T = 0;
  DevBuf<int> game, last_bid, player, hands, ply, round, widx, act, mt_idx, running, left, plies, rounds;
  DevBuf<int> tr_ply, tr_plies, tr_act, tr_rounds;
  DevBuf<double> bel, tr_prob, tr_bel;
  DevBuf<float> payoff;
  DevBuf<uint32_t> mt;
  cfrb::MatchDev dev{};
  Pinned<int> pin_left;               // slots with a game left, copied behind the last round of every cfrb_match_run
  Event ev_left;
  bool ev_recorded = false;
  // local best response (cfrb_match_create_lbr): h[1] is null, agent 1 is LBR
  bool lbr = false;
  cfrb::LbrDev ldev{};
  DevBuf<int> nsg, pend, rr, solves_g, whatif_g;
  DevBuf<double> sigx, tr_val, tr_beta;
  DevBuf<unsigned long long> deferred;
};

// Agent slot k of the tables a match, LBR or agent kernel reads: the handle's wave beliefs and the table it acts with, the
// sampled snapshot or its average strategy (avg_table).
template <typename real>
static void act_slot(cfrb::MatchTabs<real>& t, int k, const cfrb_handle* h, WaveState<real>& s, bool sampled) {
  const auto avg = avg_table(h, s);
  t.wave_beliefs[k] = s.beliefs.p;
  t.table[k] = sampled ? s.Snap.p : avg.p;
  t.normalise[k] = !sampled && avg.normalise;
}

// The kernels of a round around the agents' solves: the scan that packs the round's subgames (begin), or the walk that plays it.
static int match_kernels(cfrb_match* m, bool begin, cudaStream_t st) {
  cfrb_handle* a = m->h[0];
  with_state(a, m->lbr ? a : m->h[1], [&](auto& sa, auto& sb) {
    cfrb::MatchTabs<typename std::decay_t<decltype(sa)>::real> t{};
    if (m->lbr) {   // LBR reads the agent's table as in an AVERAGE match
      act_slot(t, 0, a, sa, false);
      if (begin) cfrb::lbr_launch_begin(m->ldev, t, st);
      else cfrb::lbr_launch_advance(m->ldev, t, st);
    } else {
      act_slot(t, 0, a, sa, m->dev.sampled);
      act_slot(t, 1, m->h[1], sb, m->dev.sampled);
      if (begin) cfrb::match_launch_begin(m->dev, t, st);
      else cfrb::match_launch_advance(m->dev, t, st);
    }
  });
  CK(cudaGetLastError());
  return CFRB_OK;
}

// Everything enqueued has finished: each handle's current wave becomes the match's last wave (its size lives on the device).
static int match_settle(cfrb_match* m) {
  CK(cudaSetDevice(m->h[0]->cfg.device));
  CK(cudaDeviceSynchronize());
  for (cfrb_handle* h : m->h) {
    if (!h) continue;
    int wave[2] = {0, 0};
    CK(cudaMemcpy(wave, h->d_wave.p, sizeof(wave), cudaMemcpyDeviceToHost));
    h->n = wave[0];
    h->mirror_stale = true;
  }
  return CFRB_OK;
}

extern "C" {

int cfrb_match_destroy(cfrb_match* m) {
  if (!m) return CFRB_OK;
  int rc = CFRB_OK;
  if (m->h[0]) {
    rc = match_settle(m);
    for (cfrb_handle* h : m->h)
      if (h) h->in_match = false;
  }
  delete m;
  return rc;
}

static int match_alloc(cfrb_match* m, cfrb_handle* a, int32_t n_slots, int32_t n_games, uint64_t seed);

static int match_create_impl(cfrb_match* m, cfrb_handle* a, cfrb_handle* b, int32_t n_slots, int32_t n_games, uint64_t seed,
                             int32_t policy) {
  if (!a || !b) return fail(CFRB_EINVAL, "cfrb_match_create: null handle");
  if (a == b) return fail(CFRB_EINVAL, "cfrb_match_create: the two agents need two handles (create a second one with the same config)");
  if (policy != CFRB_MATCH_AVERAGE && policy != CFRB_MATCH_SAMPLED) return fail(CFRB_EINVAL, "cfrb_match_create: bad policy");
  if (n_slots < 1) return fail(CFRB_EINVAL, "cfrb_match_create: n_slots must be >= 1");
  if (n_games < 2 || n_games % 2) return fail(CFRB_EINVAL, "cfrb_match_create: n_games must be even and >= 2 (seat-swapped pairs)");
  const auto &ca = a->cfg, &cb = b->cfg;
  if (ca.num_dice != cb.num_dice || ca.num_faces != cb.num_faces)
    return fail(CFRB_EINVAL, "cfrb_match_create: the agents play different games (" + std::to_string(ca.num_dice) + "x" +
                                 std::to_string(ca.num_faces) + "f vs " + std::to_string(cb.num_dice) + "x" + std::to_string(cb.num_faces) + "f)");
  if (ca.max_depth != cb.max_depth)
    return fail(CFRB_EINVAL, "cfrb_match_create: the agents have different max_depth (" + std::to_string(ca.max_depth) + " vs " +
                                 std::to_string(cb.max_depth) + ")");
  if (ca.device != cb.device) return fail(CFRB_EINVAL, "cfrb_match_create: the agents are on different devices");
  if (ca.state_dtype != cb.state_dtype) return fail(CFRB_EINVAL, "cfrb_match_create: the agents have different state dtypes");
  for (cfrb_handle* h : {a, b}) {
    if (h->cfg.max_subgames < n_slots)
      return fail(CFRB_EINVAL, "cfrb_match_create: a handle's capacity (max_subgames " + std::to_string(h->cfg.max_subgames) +
                                   ") is smaller than n_slots " + std::to_string(n_slots));
    if (h->sp.ready) return fail(CFRB_EINVAL, "cfrb_match_create: a handle has a live self-play session");
    if (h->in_match) return fail(CFRB_EINVAL, "cfrb_match_create: a handle already plays in a live match");
  }
  int rc = match_alloc(m, a, n_slots, n_games, seed);
  if (rc) return rc;
  cfrb::MatchDev& d = m->dev;
  d.sampled = policy == CFRB_MATCH_SAMPLED;
  d.iters[0] = ca.num_iters; d.iters[1] = cb.num_iters;
  cfrb_handle* hs[2] = {a, b};
  for (int k = 0; k < 2; ++k) {
    cfrb_handle* h = hs[k];
    d.wave[k] = h->d_wave.p; d.sg_tmpl[k] = h->d_sg_tmpl.p; d.sg_player[k] = h->d_sg_player.p; d.sg_row_off[k] = h->d_sg_row_off.p;
    d.sg_act[k] = h->d_sg_act.p; d.steps[k] = h->d_steps.p;
  }
  cfrb::match_launch_deal(d, a->own_stream);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(a->own_stream));
  m->h[0] = a; m->h[1] = b;
  a->in_match = b->in_match = true;
  return CFRB_OK;
}

// Slots, games, streams and trace buffers of a match played with agent a's game (the part shared by both kinds of match).
static int match_alloc(cfrb_match* m, cfrb_handle* a, int32_t n_slots, int32_t n_games, uint64_t seed) {
  const auto& ca = a->cfg;
  CK(cudaSetDevice(ca.device));
  CK(cudaDeviceSynchronize());
  const int S = n_slots, G = n_games, H = a->g.H, A = a->g.A, T = std::min(G, (int)CFRB_MATCH_TRACE_GAMES);
  m->S = S; m->G = G; m->T = T;
  for (auto* p : {&m->game, &m->last_bid, &m->player, &m->ply, &m->round, &m->widx, &m->mt_idx}) CK(p->alloc(S));
  CK(m->hands.alloc((size_t)2 * S)); CK(m->act.alloc((size_t)2 * S));
  CK(m->running.alloc(1)); CK(m->left.alloc(1));
  CK(m->bel.alloc((size_t)S * 4 * H)); CK(m->mt.alloc((size_t)624 * S));
  CK(m->payoff.alloc(G)); CK(m->plies.alloc(G)); CK(m->rounds.alloc(G));
  CK(cudaMemset(m->payoff.p, 0, (size_t)G * sizeof(float)));
  CK(cudaMemset(m->plies.p, 0, (size_t)G * sizeof(int)));
  CK(cudaMemset(m->rounds.p, 0, (size_t)G * sizeof(int)));
  CK(m->tr_ply.alloc((size_t)T * A * 6)); CK(m->tr_prob.alloc((size_t)T * A)); CK(m->tr_plies.alloc(T));
  CK(m->tr_act.alloc((size_t)T * A * 2)); CK(m->tr_bel.alloc((size_t)T * A * 4 * H)); CK(m->tr_rounds.alloc(T));
  CK(cudaMemset(m->tr_plies.p, 0, (size_t)T * sizeof(int)));
  CK(cudaMemset(m->tr_rounds.p, 0, (size_t)T * sizeof(int)));
  CK(cudaMallocHost((void**)m->pin_left.put(), sizeof(int)));
  CK(cudaEventCreateWithFlags(m->ev_left.put(), cudaEventDisableTiming));
  cfrb::MatchDev& d = m->dev;
  d.S = S; d.G = G; d.A = A; d.H = H; d.F = a->g.F; d.max_depth = ca.max_depth; d.seed = seed;
  d.game = m->game.p; d.last_bid = m->last_bid.p; d.player = m->player.p; d.hands = m->hands.p; d.ply = m->ply.p; d.round = m->round.p;
  d.widx = m->widx.p; d.act = m->act.p; d.bel = m->bel.p; d.mt = m->mt.p; d.mt_idx = m->mt_idx.p; d.running = m->running.p;
  d.left = m->left.p;
  d.payoff = m->payoff.p; d.plies = m->plies.p; d.rounds = m->rounds.p;
  d.trace_games = T; d.tr_ply = m->tr_ply.p; d.tr_prob = m->tr_prob.p; d.tr_plies = m->tr_plies.p; d.tr_act = m->tr_act.p;
  d.tr_bel = m->tr_bel.p; d.tr_rounds = m->tr_rounds.p;
  d.tmpl = a->d_tmpl.p; d.child_begin = a->d_child_begin.p; d.nchild = a->d_nchild.p; d.matches = a->d_matches.p;
  d.table_stride = a->table_stride;
  return CFRB_OK;
}

int cfrb_match_create(cfrb_handle* a, cfrb_handle* b, int32_t n_slots, int32_t n_games, uint64_t seed, int32_t policy, cfrb_match** out) {
  if (!out) return fail(CFRB_EINVAL, "cfrb_match_create: null argument");
  *out = nullptr;
  auto m = std::make_unique<cfrb_match>();
  const int rc = match_create_impl(m.get(), a, b, n_slots, n_games, seed, policy);
  if (rc != CFRB_OK) return rc;
  *out = m.release();
  return CFRB_OK;
}

static int lbr_create_impl(cfrb_match* m, cfrb_handle* a, int32_t n_slots, int32_t n_games, uint64_t seed) {
  if (!a) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: null handle");
  if (n_slots < 1) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: n_slots must be >= 1");
  if (n_games < 2 || n_games % 2) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: n_games must be even and >= 2 (seat-swapped pairs)");
  if (a->sp.ready) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: the handle has a live self-play session");
  if (a->in_match) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: the handle already plays in a live match");
  const int A = a->g.A;
  if (a->cfg.max_subgames < A - 1)
    return fail(CFRB_EINVAL, "cfrb_match_create_lbr: the handle's capacity (max_subgames " + std::to_string(a->cfg.max_subgames) +
                                 ") must hold the A - 1 = " + std::to_string(A - 1) + " what-if subgames of one LBR decision");
  int rc = match_alloc(m, a, n_slots, n_games, seed);
  if (rc) return rc;
  const int S = n_slots, G = n_games, H = a->g.H, T = m->T;
  cfrb::MatchDev& d = m->dev;
  d.sampled = 0;
  d.iters[0] = a->cfg.num_iters;
  d.wave[0] = a->d_wave.p; d.sg_tmpl[0] = a->d_sg_tmpl.p; d.sg_player[0] = a->d_sg_player.p; d.sg_row_off[0] = a->d_sg_row_off.p;
  d.sg_act[0] = a->d_sg_act.p; d.steps[0] = a->d_steps.p;
  CK(m->nsg.alloc(S)); CK(m->pend.alloc(S)); CK(m->rr.alloc(1)); CK(m->deferred.alloc(1));
  CK(m->solves_g.alloc(G)); CK(m->whatif_g.alloc(G));
  CK(m->sigx.alloc((size_t)S * A * H));
  CK(m->tr_val.alloc((size_t)T * A * A)); CK(m->tr_beta.alloc((size_t)T * A * H));
  CK(cudaMemset(m->pend.p, 0, (size_t)S * sizeof(int)));
  CK(cudaMemset(m->nsg.p, 0, (size_t)S * sizeof(int)));
  CK(cudaMemset(m->rr.p, 0, sizeof(int)));
  CK(cudaMemset(m->deferred.p, 0, sizeof(unsigned long long)));
  CK(cudaMemset(m->solves_g.p, 0, (size_t)G * sizeof(int)));
  CK(cudaMemset(m->whatif_g.p, 0, (size_t)G * sizeof(int)));
  CK(cudaMemset(m->tr_bel.p, 0, (size_t)T * A * 4 * H * sizeof(double)));   // LBR's root beliefs stay zero
  CK(cudaMemset(m->tr_beta.p, 0, (size_t)T * A * H * sizeof(double)));
  const std::vector<double> nan((size_t)T * A * A, std::numeric_limits<double>::quiet_NaN());
  CK(cudaMemcpy(m->tr_val.p, nan.data(), nan.size() * sizeof(double), cudaMemcpyHostToDevice));
  cfrb::LbrDev& l = m->ldev;
  l.K = a->cfg.max_subgames;
  l.nsg = m->nsg.p; l.pend = m->pend.p; l.sigx = m->sigx.p; l.rr = m->rr.p; l.deferred = m->deferred.p;
  l.solves = m->solves_g.p; l.whatif = m->whatif_g.p; l.tr_val = m->tr_val.p; l.tr_beta = m->tr_beta.p;
  cfrb::match_launch_deal(d, a->own_stream);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(a->own_stream));
  l.m = d;
  m->lbr = true;
  m->h[0] = a;
  a->in_match = true;
  return CFRB_OK;
}

int cfrb_match_create_lbr(cfrb_handle* agent, int32_t n_slots, int32_t n_games, uint64_t seed, cfrb_match** out) {
  if (!out) return fail(CFRB_EINVAL, "cfrb_match_create_lbr: null argument");
  *out = nullptr;
  auto m = std::make_unique<cfrb_match>();
  const int rc = lbr_create_impl(m.get(), agent, n_slots, n_games, seed);
  if (rc != CFRB_OK) return rc;
  *out = m.release();
  return CFRB_OK;
}

int cfrb_match_lbr_trace(cfrb_match* m, int32_t game, double* values, double* beliefs) {
  if (!m || !m->lbr) return fail(CFRB_EINVAL, "cfrb_match_lbr_trace: not an LBR match");
  if (game < 0 || game >= m->T) return fail(CFRB_EINVAL, "cfrb_match_lbr_trace: only games < min(n_games, CFRB_MATCH_TRACE_GAMES) are traced");
  int rc = match_settle(m);
  if (rc) return rc;
  const size_t A = m->dev.A, H = m->dev.H;
  int np = 0;
  CK(cudaMemcpy(&np, m->tr_plies.p + game, sizeof(int), cudaMemcpyDeviceToHost));
  if (values) CK(cudaMemcpy(values, m->tr_val.p + game * A * A, A * A * sizeof(double), cudaMemcpyDeviceToHost));
  if (beliefs) CK(cudaMemcpy(beliefs, m->tr_beta.p + game * A * H, A * H * sizeof(double), cudaMemcpyDeviceToHost));
  return np;
}

int cfrb_match_lbr_counts(cfrb_match* m, int64_t* whatif_solves, int64_t* deferred_slot_rounds) {
  if (!m || !m->lbr) return fail(CFRB_EINVAL, "cfrb_match_lbr_counts: not an LBR match");
  int rc = match_settle(m);
  if (rc) return rc;
  std::vector<int> w(m->G);
  CK(cudaMemcpy(w.data(), m->whatif_g.p, (size_t)m->G * sizeof(int), cudaMemcpyDeviceToHost));
  unsigned long long dr = 0;
  CK(cudaMemcpy(&dr, m->deferred.p, sizeof(dr), cudaMemcpyDeviceToHost));
  if (whatif_solves) {
    int64_t s = 0;
    for (int x : w) s += x;
    *whatif_solves = s;
  }
  if (deferred_slot_rounds) *deferred_slot_rounds = (int64_t)dr;
  return CFRB_OK;
}

int cfrb_match_run(cfrb_match* m, int32_t max_rounds, void* cuda_stream) {
  if (!m || max_rounds < 1) return fail(CFRB_EINVAL, "cfrb_match_run: bad argument");
  CK(cudaSetDevice(m->h[0]->cfg.device));
  if (m->ev_recorded) {
    CK(cudaEventSynchronize(m->ev_left));
    if (*m->pin_left == 0) return 0;
  }
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : m->h[0]->own_stream;
  for (int r = 0; r < max_rounds; ++r) {
    int rc = match_kernels(m, true, st);
    if (rc) return rc;
    // one wave per agent; LBR: one wave of at most max_subgames subgames of the agent
    for (cfrb_handle* h : m->h)
      if (h && (rc = solve_device_wave(h, m->lbr ? h->cfg.max_subgames : m->S, false, false, st))) return rc;
    CK(cudaMemsetAsync(m->left.p, 0, sizeof(int), st));
    if ((rc = match_kernels(m, false, st))) return rc;
    m->h[0]->launches += 3;
  }
  CK(cudaMemcpyAsync(m->pin_left, m->left.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaEventRecord(m->ev_left, st));
  m->ev_recorded = true;
  return max_rounds;
}

int cfrb_match_results(cfrb_match* m, float* payoff_a, int32_t* plies, int64_t* solves, int64_t* subgame_iters) {
  if (!m) return fail(CFRB_EINVAL, "cfrb_match_results: null match");
  int rc = match_settle(m);
  if (rc) return rc;
  const int G = m->G;
  std::vector<int> rounds(G);
  CK(cudaMemcpy(rounds.data(), m->lbr ? m->solves_g.p : m->rounds.p, (size_t)G * sizeof(int), cudaMemcpyDeviceToHost));
  if (payoff_a) CK(cudaMemcpy(payoff_a, m->payoff.p, (size_t)G * sizeof(float), cudaMemcpyDeviceToHost));
  if (plies) CK(cudaMemcpy(plies, m->plies.p, (size_t)G * sizeof(int), cudaMemcpyDeviceToHost));
  int64_t r = 0;
  for (int x : rounds) r += x;
  if (m->lbr) {                       // every subgame the agent solved, the what-if ones included
    if (solves) *solves = r;
    if (subgame_iters) *subgame_iters = r * (int64_t)m->dev.iters[0];
    return CFRB_OK;
  }
  if (solves) *solves = 2 * r;
  if (subgame_iters) *subgame_iters = r * ((int64_t)m->dev.iters[0] + m->dev.iters[1]);
  return CFRB_OK;
}

int cfrb_match_trace(cfrb_match* m, int32_t game, int32_t* ply_records, double* probs, int32_t* act_iterations, double* root_beliefs,
                     int32_t* n_rounds) {
  if (!m) return fail(CFRB_EINVAL, "cfrb_match_trace: null match");
  if (game < 0 || game >= m->T) return fail(CFRB_EINVAL, "cfrb_match_trace: only games < min(n_games, CFRB_MATCH_TRACE_GAMES) are traced");
  int rc = match_settle(m);
  if (rc) return rc;
  const size_t A = m->dev.A, H = m->dev.H;
  int np = 0, nr = 0;
  CK(cudaMemcpy(&np, m->tr_plies.p + game, sizeof(int), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&nr, m->tr_rounds.p + game, sizeof(int), cudaMemcpyDeviceToHost));
  if (ply_records) CK(cudaMemcpy(ply_records, m->tr_ply.p + game * A * 6, A * 6 * sizeof(int), cudaMemcpyDeviceToHost));
  if (probs) CK(cudaMemcpy(probs, m->tr_prob.p + game * A, A * sizeof(double), cudaMemcpyDeviceToHost));
  if (act_iterations) CK(cudaMemcpy(act_iterations, m->tr_act.p + game * A * 2, A * 2 * sizeof(int), cudaMemcpyDeviceToHost));
  if (root_beliefs) CK(cudaMemcpy(root_beliefs, m->tr_bel.p + game * A * 4 * H, A * 4 * H * sizeof(double), cudaMemcpyDeviceToHost));
  if (n_rounds) *n_rounds = nr;
  return np;
}

// ============================================================================================ device-resident example rows
struct cfrb_rows {
  int device = 0, q_dim = 0, v_dim = 0;
  int64_t cap = 0;
  DevBuf<float> q, v;
  // id staging for gathers (a small ring: a gather on the consumer's stream is not waited for, its staging slot is reused only
  // after its completion event) and the staging area for batches that leave the device
  struct IdSlot { DevBuf<int> dev; Pinned<int> pin; int cap = 0; Event done; bool used = false; };
  IdSlot ids[4];
  int next_id = 0;
  DevBuf<float> stage_q, stage_v; int64_t stage_rows = 0;
  Stream st;
};

int cfrb_rows_destroy(cfrb_rows* r) {
  if (!r) return CFRB_OK;
  cudaSetDevice(r->device);
  cudaDeviceSynchronize();
  delete r;
  return CFRB_OK;
}

int cfrb_rows_create(int32_t device, int64_t capacity_rows, int32_t q_dim, int32_t v_dim, cfrb_rows** out) {
  if (!out || capacity_rows < 1 || q_dim < 1 || v_dim < 1) return fail(CFRB_EINVAL, "bad argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return fail(CFRB_ENODEV, "no CUDA device"); }
  if (device < 0 || device >= ndev) return fail(CFRB_EINVAL, "device ordinal out of range");
  CK(cudaSetDevice(device));
  auto r = std::make_unique<cfrb_rows>();
  r->device = device; r->q_dim = q_dim; r->v_dim = v_dim; r->cap = capacity_rows;
  cudaError_t e = r->q.alloc((size_t)capacity_rows * q_dim);
  if (e == cudaSuccess) e = r->v.alloc((size_t)capacity_rows * v_dim);
  // Highest stream priority: the store's gathers and copies run next to a generator that keeps every SM busy with back-to-back
  // (programmatically chained) kernels; at equal priority their blocks waited tens of milliseconds for a slot (measured: 47 ms for a
  // 32 768-row sample, whatever its size), at high priority they take the next slot a retiring CTA frees.
  int prio_least = 0, prio_greatest = 0;
  if (e == cudaSuccess) e = cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(r->st.put(), cudaStreamNonBlocking, prio_greatest);
  // gather scratch (row-id slots, staging rows of host-bound batches) for batches of up to min(capacity, 262 144) rows, allocated
  // HERE: an allocation later, next to a generator that keeps the GPU busy with whole waves, waits for the end of a wave (measured:
  // 47 ms per sample while the four slots were being created one call at a time)
  const int64_t scratch_rows = std::min<int64_t>(capacity_rows, 1 << 18);
  for (auto& s : r->ids) {
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(s.done.put(), cudaEventDisableTiming);
    if (e == cudaSuccess) e = s.dev.alloc(scratch_rows);
    if (e == cudaSuccess) e = cudaMallocHost((void**)s.pin.put(), (size_t)scratch_rows * sizeof(int));
    if (e == cudaSuccess) s.cap = (int)scratch_rows;
  }
  if (e == cudaSuccess) e = r->stage_q.alloc((size_t)scratch_rows * q_dim);
  if (e == cudaSuccess) e = r->stage_v.alloc((size_t)scratch_rows * v_dim);
  if (e == cudaSuccess) r->stage_rows = (int)scratch_rows;
  if (e != cudaSuccess) return fail(CFRB_ENOMEM, std::string("cfrb_rows_create: ") + cudaGetErrorString(e));
  *out = r.release();
  return CFRB_OK;
}

int cfrb_rows_device(const cfrb_rows* r) { return r ? r->device : -1; }

// kind: 0 = host source, 1 = device source on `src_device` (peer copy when that is another GPU).  Ring wrap-around handled
// here.  Ordered after every gather still in flight on a consumer's stream (it may read the slots being replaced); blocks until
// the rows are in place (the caller publishes them right after).
int cfrb_rows_write(cfrb_rows* r, int64_t slot, int32_t n, const float* q, const float* v, int32_t kind, int32_t src_device) {
  if (!r || !q || !v || n < 0 || slot < 0 || slot >= r->cap || n > r->cap) return fail(CFRB_EINVAL, "cfrb_rows_write: bad argument");
  CK(cudaSetDevice(r->device));
  for (auto& s : r->ids)
    if (s.used) CK(cudaStreamWaitEvent(r->st, s.done, 0));
  auto put = [&](float* dst_base, const float* src, int dim) -> cudaError_t {
    const int64_t first = std::min<int64_t>(n, r->cap - slot);
    for (int part = 0; part < 2; ++part) {
      const int64_t cnt = part == 0 ? first : n - first;
      if (cnt <= 0) continue;
      float* dst = dst_base + (size_t)(part == 0 ? slot : 0) * dim;
      const float* s2 = src + (size_t)(part == 0 ? 0 : first) * dim;
      const size_t bytes = (size_t)cnt * dim * sizeof(float);
      cudaError_t e;
      if (kind == 0) e = cudaMemcpyAsync(dst, s2, bytes, cudaMemcpyHostToDevice, r->st);
      else if (src_device == r->device) e = cudaMemcpyAsync(dst, s2, bytes, cudaMemcpyDeviceToDevice, r->st);
      else e = cudaMemcpyPeerAsync(dst, r->device, s2, src_device, bytes, r->st);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  };
  CK(put(r->q.p, q, r->q_dim));
  CK(put(r->v.p, v, r->v_dim));
  CK(cudaStreamSynchronize(r->st));
  return CFRB_OK;
}

int cfrb_rows_read(cfrb_rows* r, int64_t slot, int32_t n, float* q, float* v) {
  if (!r || !q || !v || n < 0 || slot < 0 || slot >= r->cap || n > r->cap) return fail(CFRB_EINVAL, "cfrb_rows_read: bad argument");
  CK(cudaSetDevice(r->device));
  const int64_t first = std::min<int64_t>(n, r->cap - slot);
  CK(cudaMemcpy(q, r->q.p + (size_t)slot * r->q_dim, (size_t)first * r->q_dim * sizeof(float), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(v, r->v.p + (size_t)slot * r->v_dim, (size_t)first * r->v_dim * sizeof(float), cudaMemcpyDeviceToHost));
  if (n > first) {
    CK(cudaMemcpy(q + (size_t)first * r->q_dim, r->q.p, (size_t)(n - first) * r->q_dim * sizeof(float), cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(v + (size_t)first * r->v_dim, r->v.p, (size_t)(n - first) * r->v_dim * sizeof(float), cudaMemcpyDeviceToHost));
  }
  return CFRB_OK;
}

// Rows ids[0..n) -> out_q [n][q_dim], out_v [n][v_dim].  out_device: -1 = host memory, otherwise the CUDA ordinal the output
// buffers live on.  When the output is on the ring's device and a stream is given, the id upload and the two gather kernels are
// enqueued on THAT stream (the consumer's: the batch is ordered like any other work of the trainer) and the call returns
// without waiting; otherwise the batch is staged on the ring's device, copied out and the call waits for it.
int cfrb_rows_gather(cfrb_rows* r, const int32_t* ids, int32_t n, float* out_q, float* out_v, int32_t out_device, void* cuda_stream) {
  if (!r || !ids || !out_q || !out_v || n < 0) return fail(CFRB_EINVAL, "cfrb_rows_gather: bad argument");
  if (n == 0) return CFRB_OK;
  CK(cudaSetDevice(r->device));
  if (n > r->ids[0].cap) {
    // grow ALL id slots at once (cfrb_rows_create sized them for min(capacity, 262 144) rows, so this is rare): allocations
    // synchronise with the device, and next to a generator that keeps the GPU busy with whole waves each one waits for the end of a wave
    const int cap = 2 * n;
    for (auto& s : r->ids) {
      if (s.used) CK(cudaEventSynchronize(s.done));
      s.cap = 0; s.used = false;
      CK(s.dev.alloc(cap));
      CK(cudaMallocHost((void**)s.pin.put(), (size_t)cap * sizeof(int)));
      s.cap = cap;
    }
  }
  auto& sl = r->ids[r->next_id];
  r->next_id = (r->next_id + 1) % 4;
  if (sl.used) CK(cudaEventSynchronize(sl.done));
  for (int i = 0; i < n; ++i) {
    if (ids[i] < 0 || ids[i] >= r->cap) return fail(CFRB_EINVAL, "cfrb_rows_gather: row id out of range");
    sl.pin[i] = ids[i];
  }
  const bool same = out_device == r->device;
  const bool direct = same && cuda_stream != nullptr;
  cudaStream_t st = direct ? (cudaStream_t)cuda_stream : r->st;
  CK(cudaMemcpyAsync(sl.dev.p, sl.pin, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  float* tq = out_q; float* tv = out_v;
  if (!same) {
    if (n > r->stage_rows) {
      CK(cudaStreamSynchronize(r->st));
      r->stage_rows = 0;
      const int rows = 2 * n;
      CK(r->stage_q.alloc((size_t)rows * r->q_dim));
      CK(r->stage_v.alloc((size_t)rows * r->v_dim));
      r->stage_rows = rows;
    }
    tq = r->stage_q.p; tv = r->stage_v.p;
  }
  cfrb::rows_launch_gather(r->q.p, r->q_dim, sl.dev.p, n, tq, st);
  cfrb::rows_launch_gather(r->v.p, r->v_dim, sl.dev.p, n, tv, st);
  CK(cudaGetLastError());
  if (!same) {
    const size_t bq = (size_t)n * r->q_dim * sizeof(float), bv = (size_t)n * r->v_dim * sizeof(float);
    if (out_device < 0) {
      CK(cudaMemcpyAsync(out_q, tq, bq, cudaMemcpyDeviceToHost, st));
      CK(cudaMemcpyAsync(out_v, tv, bv, cudaMemcpyDeviceToHost, st));
    } else {
      CK(cudaMemcpyPeerAsync(out_q, out_device, tq, r->device, bq, st));
      CK(cudaMemcpyPeerAsync(out_v, out_device, tv, r->device, bv, st));
    }
  }
  CK(cudaEventRecord(sl.done, st));
  sl.used = true;
  if (!direct) CK(cudaStreamSynchronize(st));
  return CFRB_OK;
}

// Scratch device buffers for hand-over between a generator handle and a row store (examples of one wave).
int cfrb_dev_alloc(int32_t device, size_t bytes, void** out) {
  if (!out) return fail(CFRB_EINVAL, "null argument");
  CK(cudaSetDevice(device));
  CK(cudaMalloc(out, std::max<size_t>(bytes, 1)));
  return CFRB_OK;
}
int cfrb_dev_free(int32_t device, void* p) {
  if (!p) return CFRB_OK;
  CK(cudaSetDevice(device));
  CK(cudaFree(p));
  return CFRB_OK;
}
int cfrb_dev_to_host(int32_t device, void* dst, const void* src, size_t bytes) {
  CK(cudaSetDevice(device));
  CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return CFRB_OK;
}

}  // extern "C"

// ============================================================================================ NCCL (one process per GPU)
// The reference is a single process: generator threads share the trainer's model replicas and its host-memory replay.  With
// one process per GPU the two hand-overs become collectives over NVLink, issued from THIS library on device buffers:
//   ModelLocker::updateModel (rela/model_locker.h:69-79)      -> ncclBroadcast of the flat weight buffer from the trainer's rank
//   PrioritizedReplay::add   (rela/prioritized_replay.h:247-261) -> grouped ncclSend / ncclRecv of every rank's example rows
//                                                                   into the trainer rank's device-resident replay rows
//   recursive_eval's accumulation (recursive_eval.cc:343-363) -> ncclReduce(sum) of the float32 accumulators
#include <nccl.h>

struct cfrb_comm {
  Owner<ncclComm_t, ncclCommDestroy> comm;           // destroyed last
  int rank = 0, world = 1, device = 0;
  Stream st;
  DevBuf<float> scratch;
  Pinned<float> pin; size_t pin_floats = 0;          // pinned staging of the stream-ordered weight broadcast
  DevBuf<int> vote;                                  // [4] device ints of the vote
  Pinned<int> pin_vote; int* pin_vote_out = nullptr; // pinned [4] each: contributions / result
};

#define NCK(call)                                                                                                       \
  do {                                                                                                                  \
    ncclResult_t r__ = (call);                                                                                          \
    if (r__ != ncclSuccess) return fail(CFRB_ECUDA, std::string(#call) + ": " + ncclGetErrorString(r__));              \
  } while (0)

extern "C" {

int cfrb_comm_unique_id(uint8_t* out128) {
  if (!out128) return fail(CFRB_EINVAL, "null argument");
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  ncclUniqueId id;
  NCK(ncclGetUniqueId(&id));
  std::memcpy(out128, &id, 128);
  return CFRB_OK;
}

int cfrb_comm_create(const uint8_t* id128, int32_t rank, int32_t world, int32_t device, cfrb_comm** out) {
  if (!id128 || !out || world < 1 || rank < 0 || rank >= world) return fail(CFRB_EINVAL, "cfrb_comm_create: bad argument");
  CK(cudaSetDevice(device));
  auto c = std::make_unique<cfrb_comm>();
  c->rank = rank; c->world = world; c->device = device;
  ncclUniqueId id;
  std::memcpy(&id, id128, 128);
  ncclComm_t comm = nullptr;
  ncclResult_t r = ncclCommInitRank(&comm, world, id, rank);
  if (r != ncclSuccess) return fail(CFRB_ECUDA, std::string("ncclCommInitRank: ") + ncclGetErrorString(r));
  c->comm = decltype(c->comm)(comm);
  cudaError_t e = cudaStreamCreateWithFlags(c->st.put(), cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMallocHost((void**)c->pin_vote.put(), 8 * sizeof(int));
  if (e != cudaSuccess) return fail(CFRB_ECUDA, cudaGetErrorString(e));
  c->pin_vote_out = c->pin_vote + 4;
  *out = c.release();
  return CFRB_OK;
}

int cfrb_comm_destroy(cfrb_comm* c) {
  if (!c) return CFRB_OK;
  cudaSetDevice(c->device);
  if (c->st) cudaStreamSynchronize(c->st);
  delete c;
  return CFRB_OK;
}

int cfrb_comm_rank(const cfrb_comm* c) { return c ? c->rank : -1; }
int cfrb_comm_world(const cfrb_comm* c) { return c ? c->world : 0; }

static int comm_scratch(cfrb_comm* c, size_t floats) {
  if (c->scratch.n < floats) CK(c->scratch.alloc(floats));
  return CFRB_OK;
}

int cfrb_comm_broadcast_weights(cfrb_comm* c, float* flat_host, size_t n, int32_t root, void* cuda_stream) {
  if (!c || n == 0 || (!flat_host && (!cuda_stream || c->rank == root))) return fail(CFRB_EINVAL, "cfrb_comm_broadcast_weights: bad argument");
  CK(cudaSetDevice(c->device));
  int rc = comm_scratch(c, n);
  if (rc) return rc;
  if (!cuda_stream) {
    if (c->rank == root) CK(cudaMemcpyAsync(c->scratch.p, flat_host, n * sizeof(float), cudaMemcpyHostToDevice, c->st));
    NCK(ncclBroadcast(c->scratch.p, c->scratch.p, n, ncclFloat, root, c->comm, c->st));
    if (c->rank != root) CK(cudaMemcpyAsync(flat_host, c->scratch.p, n * sizeof(float), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
    return CFRB_OK;
  }
  // stream-ordered: staged through pinned memory owned by the communicator; nothing is waited for here.  The root's buffer is
  // copied now (the caller may reuse it); the other ranks read theirs with cfrb_comm_broadcast_fetch once the stream got there.
  cudaStream_t st = (cudaStream_t)cuda_stream;
  if (c->pin_floats < n) {
    c->pin_floats = 0;
    CK(cudaMallocHost((void**)c->pin.put(), n * sizeof(float)));
    c->pin_floats = n;
  }
  if (c->rank == root) {
    std::memcpy(c->pin, flat_host, n * sizeof(float));
    CK(cudaMemcpyAsync(c->scratch.p, c->pin, n * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  NCK(ncclBroadcast(c->scratch.p, c->scratch.p, n, ncclFloat, root, c->comm, st));
  if (c->rank != root) CK(cudaMemcpyAsync(c->pin, c->scratch.p, n * sizeof(float), cudaMemcpyDeviceToHost, st));
  return CFRB_OK;
}
int cfrb_comm_broadcast_fetch(cfrb_comm* c, float* out_host, size_t n) {
  if (!c || !out_host || !c->pin || n > c->pin_floats) return fail(CFRB_EINVAL, "cfrb_comm_broadcast_fetch: no stream-ordered broadcast of that size");
  std::memcpy(out_host, c->pin, n * sizeof(float));
  return CFRB_OK;
}

int cfrb_comm_gather_rows(cfrb_comm* c, const float* dev_q, const float* dev_v, int32_t n, int32_t q_dim, int32_t v_dim, float* recv_q,
                          float* recv_v, int32_t root, void* cuda_stream) {
  if (!c || !dev_q || !dev_v || n < 0 || q_dim < 1 || v_dim < 1) return fail(CFRB_EINVAL, "cfrb_comm_gather_rows: bad argument");
  if (c->rank == root && (!recv_q || !recv_v)) return fail(CFRB_EINVAL, "cfrb_comm_gather_rows: the root needs receive buffers");
  CK(cudaSetDevice(c->device));
  const size_t nq = (size_t)n * q_dim, nv = (size_t)n * v_dim;
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->st;
  NCK(ncclGroupStart());
  if (c->rank == root) {
    for (int r = 0; r < c->world; ++r) {
      if (r == root) continue;
      NCK(ncclRecv(recv_q + (size_t)r * nq, nq, ncclFloat, r, c->comm, st));
      NCK(ncclRecv(recv_v + (size_t)r * nv, nv, ncclFloat, r, c->comm, st));
    }
  } else {
    NCK(ncclSend(dev_q, nq, ncclFloat, root, c->comm, st));
    NCK(ncclSend(dev_v, nv, ncclFloat, root, c->comm, st));
  }
  NCK(ncclGroupEnd());
  if (c->rank == root) {     // the root's own block: a device-to-device copy into its slot
    CK(cudaMemcpyAsync(recv_q + (size_t)root * nq, dev_q, nq * sizeof(float), cudaMemcpyDeviceToDevice, st));
    CK(cudaMemcpyAsync(recv_v + (size_t)root * nv, dev_v, nv * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  if (!cuda_stream) CK(cudaStreamSynchronize(st));     // on the caller's stream the collective is just enqueued (stream-ordered)
  return CFRB_OK;
}

// Agreement between the ranks' generator loops (they must issue the same number of collectives): every rank contributes a flag,
// all ranks get the maximum.  Enqueued on `cuda_stream` (NULL: the communicator's stream); cfrb_comm_vote_result reads it once the
// stream has passed that point (the caller synchronises, e.g. with cfrb_mark_wait).
int cfrb_comm_vote(cfrb_comm* c, const int32_t* values, int32_t n, void* cuda_stream) {
  if (!c || !values || n < 1 || n > 4) return fail(CFRB_EINVAL, "cfrb_comm_vote: 1..4 values");
  CK(cudaSetDevice(c->device));
  if (!c->vote.p) CK(c->vote.alloc(4));
  cudaStream_t st = cuda_stream ? (cudaStream_t)cuda_stream : c->st;
  int* pin_i = c->pin_vote;      // contributions from pinned words owned by the communicator (the previous vote has been read)
  for (int i = 0; i < n; ++i) pin_i[i] = values[i];
  CK(cudaMemcpyAsync(c->vote.p, pin_i, n * sizeof(int), cudaMemcpyHostToDevice, st));
  NCK(ncclAllReduce(c->vote.p, c->vote.p, n, ncclInt32, ncclMax, c->comm, st));
  CK(cudaMemcpyAsync(c->pin_vote_out, c->vote.p, n * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (!cuda_stream) CK(cudaStreamSynchronize(st));
  return CFRB_OK;
}
int cfrb_comm_vote_result(cfrb_comm* c, int32_t* out, int32_t n) {
  if (!c || !out || !c->vote.p || n < 1 || n > 4) return fail(CFRB_EINVAL, "cfrb_comm_vote_result: no vote");
  for (int i = 0; i < n; ++i) out[i] = c->pin_vote_out[i];
  return CFRB_OK;
}

int cfrb_comm_reduce_sum(cfrb_comm* c, float* dev_buf, size_t n, int32_t root) {
  if (!c || !dev_buf) return fail(CFRB_EINVAL, "cfrb_comm_reduce_sum: bad argument");
  CK(cudaSetDevice(c->device));
  NCK(ncclReduce(dev_buf, dev_buf, n, ncclFloat, ncclSum, root, c->comm, c->st));
  CK(cudaStreamSynchronize(c->st));
  return CFRB_OK;
}

}  // extern "C"

// ============================================================================================ an agent against external players
struct cfrb_agent {
  cfrb_handle* h = nullptr;
  int T = 0, sampled = 0;
  uint64_t games_started = 0;
  DevBuf<int> seat, hand, last_bid, player, ply, root_lb, root_player, node, depth, act, status, subgames, mt_idx;
  DevBuf<int> ids, io, hands, widx, flags;
  DevBuf<uint64_t> keys;
  DevBuf<double> root_bel, bel, cache, probs, pol;
  DevBuf<uint32_t> mt;
  cfrb::AgentDev dev{};
  // host mirror of each table's public state, updated from every call's outputs (all calls synchronise)
  std::vector<char> running, need_solve;
  std::vector<int> h_seat, h_last_bid, h_player;
  std::vector<int64_t> stamp;         // call number that last listed the table (repeated ids)
  int64_t calls = 0, solves = 0;
  double solve_ms = 0;
  Event ev[2];
};

static std::string agent_table(const char* who, int id) { return std::string(who) + ": table " + std::to_string(id) + ": "; }

// Ids in range, distinct, and (running) holding a game.
static int agent_check_ids(cfrb_agent* a, const char* who, int n, const int32_t* ids, bool running) {
  ++a->calls;
  for (int i = 0; i < n; ++i) {
    const int t = ids[i];
    if (t < 0 || t >= a->T) return fail(CFRB_EINVAL, agent_table(who, t) + "id out of range [0, " + std::to_string(a->T) + ")");
    if (a->stamp[t] == a->calls) return fail(CFRB_EINVAL, agent_table(who, t) + "listed twice");
    a->stamp[t] = a->calls;
    if (running && !a->running[t]) return fail(CFRB_EINVAL, agent_table(who, t) + "no running game");
  }
  return CFRB_OK;
}

// Copies the call's ids to the device and returns the per-call view of the state.
static int agent_call(cfrb_agent* a, int n, const int32_t* ids, cfrb::AgentDev* d) {
  CK(cudaSetDevice(a->h->cfg.device));
  CK(cudaMemcpyAsync(a->ids.p, ids, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, a->h->own_stream));
  *d = a->dev;
  d->n = n;
  return CFRB_OK;
}

// One wave: every listed table at an unsolved root, packed in list order, solved and captured into the cache.
static int agent_solve(cfrb_agent* a, const cfrb::AgentDev& d, int n, const int32_t* ids) {
  int n_solve = 0;
  for (int i = 0; i < n; ++i) n_solve += a->need_solve[ids[i]];
  if (n_solve == 0) return CFRB_OK;
  cfrb_handle* h = a->h;
  cudaStream_t st = h->own_stream;
  auto launch = [&](bool begin) -> int {
    with_state(h, [&](auto& s) {
      cfrb::MatchTabs<typename std::decay_t<decltype(s)>::real> t{};
      act_slot(t, 0, h, s, a->sampled);
      if (begin) cfrb::agent_launch_begin(d, t, st);
      else cfrb::agent_launch_capture(d, t, st);
    });
    CK(cudaGetLastError());
    return CFRB_OK;
  };
  int rc = launch(true);
  if (rc) return rc;
  CK(cudaEventRecord(a->ev[0], st));
  if ((rc = solve_device_wave(h, n_solve, false, false, st))) return rc;
  CK(cudaEventRecord(a->ev[1], st));
  if ((rc = launch(false))) return rc;
  h->launches += 3;
  CK(cudaEventSynchronize(a->ev[1]));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, a->ev[0], a->ev[1]));
  a->solve_ms += ms;
  a->solves += n_solve;
  for (int i = 0; i < n; ++i) a->need_solve[ids[i]] = 0;
  return CFRB_OK;
}

static int agent_create_impl(cfrb_agent* a, cfrb_handle* h, int32_t n_tables, uint64_t seed, int32_t policy) {
  if (!h) return fail(CFRB_EINVAL, "cfrb_agent_create: null handle");
  if (policy != CFRB_MATCH_AVERAGE && policy != CFRB_MATCH_SAMPLED) return fail(CFRB_EINVAL, "cfrb_agent_create: bad policy");
  if (n_tables < 1) return fail(CFRB_EINVAL, "cfrb_agent_create: n_tables must be >= 1");
  if (h->cfg.max_subgames < n_tables)
    return fail(CFRB_EINVAL, "cfrb_agent_create: the handle's capacity (max_subgames " + std::to_string(h->cfg.max_subgames) +
                                 ") is smaller than n_tables " + std::to_string(n_tables) + " (one wave solves every listed table)");
  if (h->sp.ready) return fail(CFRB_EINVAL, "cfrb_agent_create: the handle has a live self-play session");
  if (h->in_match) return fail(CFRB_EINVAL, "cfrb_agent_create: the handle already plays in a live match or agent");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaDeviceSynchronize());
  const int T = n_tables, H = h->g.H, A = h->g.A;
  a->T = T;
  a->sampled = policy == CFRB_MATCH_SAMPLED;
  for (auto* b : {&a->seat, &a->hand, &a->last_bid, &a->player, &a->ply, &a->root_lb, &a->root_player, &a->node, &a->depth, &a->act,
                  &a->status, &a->subgames, &a->mt_idx, &a->ids, &a->io, &a->hands, &a->widx, &a->flags}) {
    CK(b->alloc(T));
    CK(cudaMemset(b->p, 0, (size_t)T * sizeof(int)));
  }
  CK(a->keys.alloc(T));
  CK(a->root_bel.alloc((size_t)T * 2 * H)); CK(a->bel.alloc((size_t)T * 2 * H));
  CK(cudaMemset(a->root_bel.p, 0, (size_t)T * 2 * H * sizeof(double)));
  CK(a->cache.alloc((size_t)T * h->table_stride)); CK(a->probs.alloc((size_t)T * A)); CK(a->pol.alloc((size_t)T * H * A));
  CK(a->mt.alloc((size_t)624 * T));
  CK(cudaEventCreate(a->ev[0].put())); CK(cudaEventCreate(a->ev[1].put()));
  a->running.assign(T, 0); a->need_solve.assign(T, 0);
  a->h_seat.assign(T, 0); a->h_last_bid.assign(T, -1); a->h_player.assign(T, 0);
  a->stamp.assign(T, 0);
  cfrb::AgentDev& d = a->dev;
  d.T = T; d.A = A; d.H = H; d.max_depth = h->cfg.max_depth; d.sampled = a->sampled; d.iters = h->cfg.num_iters; d.seed = seed;
  d.seat = a->seat.p; d.hand = a->hand.p; d.last_bid = a->last_bid.p; d.player = a->player.p; d.ply = a->ply.p;
  d.root_lb = a->root_lb.p; d.root_player = a->root_player.p; d.node = a->node.p; d.depth = a->depth.p;
  d.act = a->act.p; d.status = a->status.p; d.subgames = a->subgames.p;
  d.root_bel = a->root_bel.p; d.bel = a->bel.p; d.mt = a->mt.p; d.mt_idx = a->mt_idx.p;
  d.cache = a->cache.p; d.stride = h->table_stride;
  d.ids = a->ids.p; d.io = a->io.p; d.hands = a->hands.p; d.keys = a->keys.p; d.widx = a->widx.p; d.probs = a->probs.p;
  d.flags = a->flags.p; d.pol = a->pol.p;
  d.tmpl = h->d_tmpl.p; d.child_begin = h->d_child_begin.p; d.nchild = h->d_nchild.p; d.level_begin = h->d_level_begin.p;
  d.table_stride = h->table_stride;
  d.wave = h->d_wave.p; d.sg_tmpl = h->d_sg_tmpl.p; d.sg_player = h->d_sg_player.p; d.sg_row_off = h->d_sg_row_off.p;
  d.sg_act = h->d_sg_act.p; d.steps = h->d_steps.p;
  a->h = h;
  h->in_match = true;
  return CFRB_OK;
}

extern "C" {

int cfrb_agent_create(cfrb_handle* h, int32_t n_tables, uint64_t seed, int32_t policy, cfrb_agent** out) {
  if (!out) return fail(CFRB_EINVAL, "cfrb_agent_create: null argument");
  *out = nullptr;
  auto a = std::make_unique<cfrb_agent>();
  const int rc = agent_create_impl(a.get(), h, n_tables, seed, policy);
  if (rc != CFRB_OK) return rc;
  *out = a.release();
  return CFRB_OK;
}

int cfrb_agent_destroy(cfrb_agent* a) {
  if (!a) return CFRB_OK;
  int rc = CFRB_OK;
  if (cudaSetDevice(a->h->cfg.device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
    rc = fail(CFRB_ECUDA, std::string("cfrb_agent_destroy: ") + cudaGetErrorString(cudaGetLastError()));
  a->h->in_match = false;
  delete a;
  return rc;
}

int cfrb_agent_new_games(cfrb_agent* a, int32_t n, const int32_t* ids, const int32_t* seats, const int32_t* hands, const uint64_t* keys) {
  static const char* who = "cfrb_agent_new_games";
  if (!a || n < 0 || n > (a ? a->T : 0)) return fail(CFRB_EINVAL, std::string(who) + ": bad argument");
  if (n == 0) return CFRB_OK;
  if (!ids || !seats || !hands) return fail(CFRB_EINVAL, std::string(who) + ": null argument");
  int rc = agent_check_ids(a, who, n, ids, false);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    if (seats[i] != 0 && seats[i] != 1) return fail(CFRB_EINVAL, agent_table(who, ids[i]) + "seat must be 0 or 1");
    if (hands[i] < 0 || hands[i] >= a->dev.H)
      return fail(CFRB_EINVAL, agent_table(who, ids[i]) + "hand " + std::to_string(hands[i]) + " outside [0, " + std::to_string(a->dev.H) + ")");
  }
  std::vector<uint64_t> k(n);
  for (int i = 0; i < n; ++i) k[i] = keys ? keys[i] : a->games_started + (uint64_t)i;
  cfrb::AgentDev d;
  if ((rc = agent_call(a, n, ids, &d))) return rc;
  cudaStream_t st = a->h->own_stream;
  CK(cudaMemcpyAsync(a->io.p, seats, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(a->hands.p, hands, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(a->keys.p, k.data(), (size_t)n * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
  cfrb::agent_launch_new(d, st);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  a->games_started += n;
  for (int i = 0; i < n; ++i) {
    const int t = ids[i];
    a->running[t] = 1; a->need_solve[t] = 1; a->h_seat[t] = seats[i]; a->h_last_bid[t] = -1; a->h_player[t] = 0;
  }
  return CFRB_OK;
}

int cfrb_agent_step(cfrb_agent* a, int32_t n, const int32_t* ids, int32_t* actions, double* probs, int32_t* done) {
  static const char* who = "cfrb_agent_step";
  if (!a || n < 0 || n > (a ? a->T : 0)) return fail(CFRB_EINVAL, std::string(who) + ": bad argument");
  if (n == 0) return CFRB_OK;
  if (!ids || !actions || !done) return fail(CFRB_EINVAL, std::string(who) + ": null argument");
  int rc = agent_check_ids(a, who, n, ids, true);
  if (rc) return rc;
  const int A = a->dev.A;
  for (int i = 0; i < n; ++i) {
    const int t = ids[i], x = actions[i], lb = a->h_last_bid[t];
    if (x == -1) {
      if (a->h_player[t] != a->h_seat[t]) return fail(CFRB_EINVAL, agent_table(who, t) + "-1 (the agent plays) on the opponent's turn");
    } else if (x < 0 || x >= A) {
      return fail(CFRB_EINVAL, agent_table(who, t) + "action " + std::to_string(x) + " outside [-1, " + std::to_string(A) + ")");
    } else if (x <= lb) {
      return fail(CFRB_EINVAL, agent_table(who, t) + "illegal action " + std::to_string(x) + ": not above the last bid " + std::to_string(lb));
    } else if (x == A - 1 && lb < 0) {
      return fail(CFRB_EINVAL, agent_table(who, t) + "illegal action: liar call before any bid");
    }
  }
  cfrb::AgentDev d;
  if ((rc = agent_call(a, n, ids, &d))) return rc;
  cudaStream_t st = a->h->own_stream;
  CK(cudaMemcpyAsync(a->io.p, actions, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
  if ((rc = agent_solve(a, d, n, ids))) return rc;
  if (!probs) d.probs = nullptr;
  cfrb::agent_launch_step(d, st);
  CK(cudaGetLastError());
  a->h->launches += 1;
  std::vector<int> flags(n);
  CK(cudaMemcpyAsync(actions, a->io.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(flags.data(), a->flags.p, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
  if (probs) CK(cudaMemcpyAsync(probs, a->probs.p, (size_t)n * A * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  for (int i = 0; i < n; ++i) {
    const int t = ids[i];
    done[i] = flags[i] & 1;
    a->running[t] = !done[i];
    a->need_solve[t] = (flags[i] >> 1) & 1;
    a->h_last_bid[t] = actions[i];
    a->h_player[t] ^= 1;
  }
  return CFRB_OK;
}

int cfrb_agent_policy(cfrb_agent* a, int32_t n, const int32_t* ids, double* out) {
  static const char* who = "cfrb_agent_policy";
  if (!a || n < 0 || n > (a ? a->T : 0)) return fail(CFRB_EINVAL, std::string(who) + ": bad argument");
  if (n == 0) return CFRB_OK;
  if (!ids || !out) return fail(CFRB_EINVAL, std::string(who) + ": null argument");
  int rc = agent_check_ids(a, who, n, ids, true);
  if (rc) return rc;
  cfrb::AgentDev d;
  if ((rc = agent_call(a, n, ids, &d))) return rc;
  cudaStream_t st = a->h->own_stream;
  if ((rc = agent_solve(a, d, n, ids))) return rc;
  cfrb::agent_launch_policy(d, st);
  CK(cudaGetLastError());
  a->h->launches += 1;
  CK(cudaMemcpyAsync(out, a->pol.p, (size_t)n * d.H * d.A * sizeof(double), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return CFRB_OK;
}

int cfrb_agent_state(cfrb_agent* a, int32_t n, const int32_t* ids, int32_t* last_bid, int32_t* player, int32_t* ply, int32_t* subgames,
                     int32_t* act_iteration, double* root_beliefs) {
  static const char* who = "cfrb_agent_state";
  if (!a || n < 0 || n > (a ? a->T : 0)) return fail(CFRB_EINVAL, std::string(who) + ": bad argument");
  if (n == 0) return CFRB_OK;
  if (!ids) return fail(CFRB_EINVAL, std::string(who) + ": null argument");
  int rc = agent_check_ids(a, who, n, ids, false);
  if (rc) return rc;
  CK(cudaSetDevice(a->h->cfg.device));
  CK(cudaStreamSynchronize(a->h->own_stream));
  const int T = a->T, H2 = 2 * a->dev.H;
  auto gather = [&](const DevBuf<int>& src, int32_t* dst) -> int {
    if (!dst) return CFRB_OK;
    std::vector<int> all(T);
    CK(cudaMemcpy(all.data(), src.p, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) dst[i] = all[ids[i]];
    return CFRB_OK;
  };
  if ((rc = gather(a->last_bid, last_bid)) || (rc = gather(a->player, player)) || (rc = gather(a->ply, ply)) ||
      (rc = gather(a->subgames, subgames)) || (rc = gather(a->act, act_iteration)))
    return rc;
  if (root_beliefs) {
    std::vector<double> all((size_t)T * H2);
    CK(cudaMemcpy(all.data(), a->root_bel.p, all.size() * sizeof(double), cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; ++i) std::copy_n(all.data() + (size_t)ids[i] * H2, H2, root_beliefs + (size_t)i * H2);
  }
  return CFRB_OK;
}

int cfrb_agent_counts(cfrb_agent* a, int64_t* solves, int64_t* subgame_iters) {
  if (!a) return fail(CFRB_EINVAL, "cfrb_agent_counts: null agent");
  if (solves) *solves = a->solves;
  if (subgame_iters) *subgame_iters = a->solves * (int64_t)a->dev.iters;
  return CFRB_OK;
}

int cfrb_agent_solve_ms(cfrb_agent* a, double* ms) {
  if (!a || !ms) return fail(CFRB_EINVAL, "cfrb_agent_solve_ms: null argument");
  *ms = a->solve_ms;
  return CFRB_OK;
}

// ============================================================================================ value-net trainer
struct cfrb_trainer {
  int device = 0, B = 0, Q = 0, H = 0;
  cfrb::train::Layout L;
  DevBuf<float> params, grads, m, v;
  DevBuf<long long> step;
  DevBuf<float> sq_norms, last;   // sq_norms [kParams]; last = {loss, pre-clip grad norm}
  // activations and their gradients, [B][256] unless noted
  DevBuf<float> z1, xh1, rs1, a1, z2, xh2, rs2, a2, pred, dpred, row_loss;   // rs* [B], pred / dpred [B][H], row_loss [B]
  DevBuf<float> da2, dy2, dz2, da1, dy1, dz1;
};

int cfrb_trainer_create(int32_t device, int32_t num_dice, int32_t num_faces, int32_t max_batch, cfrb_trainer** out) {
  static const char* who = "cfrb_trainer_create: ";
  if (!out) return fail(CFRB_EINVAL, std::string(who) + "null argument");
  if (num_dice < 1 || num_faces < 1) return fail(CFRB_EINVAL, std::string(who) + "num_dice and num_faces must be >= 1");
  if (max_batch < 1) return fail(CFRB_EINVAL, std::string(who) + "max_batch must be >= 1");
  const cfrb::GameShape g(num_dice, num_faces);
  if (g.A > 1024 || g.H > 4096) return fail(CFRB_EINVAL, std::string(who) + "game too large");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(CFRB_ENODEV, "no CUDA device visible: libcfrb200 has no CPU fallback");
  }
  if (device < 0 || device >= ndev) return fail(CFRB_EINVAL, std::string(who) + "device ordinal out of range");
  CK(cudaSetDevice(device));
  auto t = std::make_unique<cfrb_trainer>();
  t->device = device; t->B = max_batch; t->Q = g.Q; t->H = g.H;
  t->L = cfrb::train::Layout(g.Q, g.H);
  const size_t P = (size_t)t->L.total(), BH = (size_t)max_batch * cfrb::train::kHid, BO = (size_t)max_batch * g.H;
  cudaError_t e = cudaSuccess;
  for (auto* b : {&t->params, &t->grads, &t->m, &t->v})
    if (e == cudaSuccess) e = b->alloc(P);
  for (auto* b : {&t->z1, &t->xh1, &t->a1, &t->z2, &t->xh2, &t->a2, &t->da2, &t->dy2, &t->dz2, &t->da1, &t->dy1, &t->dz1})
    if (e == cudaSuccess) e = b->alloc(BH);
  for (auto* b : {&t->rs1, &t->rs2, &t->row_loss})
    if (e == cudaSuccess) e = b->alloc(max_batch);
  for (auto* b : {&t->pred, &t->dpred})
    if (e == cudaSuccess) e = b->alloc(BO);
  if (e == cudaSuccess) e = t->sq_norms.alloc(cfrb::train::kParams);
  if (e == cudaSuccess) e = t->last.alloc(2);
  if (e == cudaSuccess) e = t->step.alloc(1);
  for (auto* b : {&t->params, &t->grads, &t->m, &t->v})
    if (e == cudaSuccess) e = cudaMemset(b->p, 0, P * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(t->last.p, 0, 2 * sizeof(float));
  if (e == cudaSuccess) e = cudaMemset(t->step.p, 0, sizeof(long long));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) return fail(CFRB_ENOMEM, std::string(who) + cudaGetErrorString(e));
  *out = t.release();
  return CFRB_OK;
}

int cfrb_trainer_destroy(cfrb_trainer* t) {
  if (!t) return CFRB_OK;
  cudaSetDevice(t->device);
  cudaDeviceSynchronize();
  delete t;
  return CFRB_OK;
}

int64_t cfrb_trainer_num_params(const cfrb_trainer* t) { return t ? t->L.total() : 0; }

int cfrb_trainer_set_state(cfrb_trainer* t, const float* params, const float* m, const float* v, int64_t step) {
  if (!t || !params) return fail(CFRB_EINVAL, "cfrb_trainer_set_state: null argument");
  if (step < 0) return fail(CFRB_EINVAL, "cfrb_trainer_set_state: step must be >= 0");
  const size_t bytes = (size_t)t->L.total() * sizeof(float);
  const long long s = step;
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(t->params.p, params, bytes, cudaMemcpyHostToDevice));
  if (m) CK(cudaMemcpy(t->m.p, m, bytes, cudaMemcpyHostToDevice));
  else CK(cudaMemset(t->m.p, 0, bytes));
  if (v) CK(cudaMemcpy(t->v.p, v, bytes, cudaMemcpyHostToDevice));
  else CK(cudaMemset(t->v.p, 0, bytes));
  CK(cudaMemcpy(t->step.p, &s, sizeof(s), cudaMemcpyHostToDevice));
  CK(cudaDeviceSynchronize());
  return CFRB_OK;
}

int cfrb_trainer_get_state(cfrb_trainer* t, float* params, float* m, float* v, int64_t* step) {
  if (!t) return fail(CFRB_EINVAL, "cfrb_trainer_get_state: null trainer");
  const size_t bytes = (size_t)t->L.total() * sizeof(float);
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  if (params) CK(cudaMemcpy(params, t->params.p, bytes, cudaMemcpyDeviceToHost));
  if (m) CK(cudaMemcpy(m, t->m.p, bytes, cudaMemcpyDeviceToHost));
  if (v) CK(cudaMemcpy(v, t->v.p, bytes, cudaMemcpyDeviceToHost));
  if (step) {
    long long s = 0;
    CK(cudaMemcpy(&s, t->step.p, sizeof(s), cudaMemcpyDeviceToHost));
    *step = s;
  }
  return CFRB_OK;
}

int cfrb_trainer_debug_grads(cfrb_trainer* t, float* out) {
  if (!t || !out) return fail(CFRB_EINVAL, "cfrb_trainer_debug_grads: null argument");
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(out, t->grads.p, (size_t)t->L.total() * sizeof(float), cudaMemcpyDeviceToHost));
  return CFRB_OK;
}

int cfrb_trainer_last(cfrb_trainer* t, float* loss, float* grad_norm) {
  if (!t) return fail(CFRB_EINVAL, "cfrb_trainer_last: null trainer");
  float h[2];
  CK(cudaSetDevice(t->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(h, t->last.p, sizeof(h), cudaMemcpyDeviceToHost));
  if (loss) *loss = h[0];
  if (grad_norm) *grad_norm = h[1];
  return CFRB_OK;
}

// A pointer the caller says is memory of the trainer's device.
static int trainer_check_ptr(const cfrb_trainer* t, const void* p, const std::string& what) {
  if (!p) return fail(CFRB_EINVAL, what + " is NULL");
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return fail(CFRB_EINVAL, what + " is not CUDA memory");
  }
  if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != t->device)
    return fail(CFRB_EINVAL, what + " must be device memory of cuda:" + std::to_string(t->device) +
                                 (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged
                                      ? " (it is on cuda:" + std::to_string(a.device) + ")" : " (it is host memory)"));
  return CFRB_OK;
}

static int trainer_check_batch(const cfrb_trainer* t, const char* who, const float* q, const float* v, int32_t n, int32_t loss_kind,
                               const float* out) {
  if (!t) return fail(CFRB_EINVAL, std::string(who) + "null trainer");
  if (n < 1 || n > t->B)
    return fail(CFRB_EINVAL, std::string(who) + "batch of " + std::to_string(n) + " rows, must be 1 .. max_batch = " + std::to_string(t->B));
  if (loss_kind != cfrb::train::LOSS_HUBER && loss_kind != cfrb::train::LOSS_MSE)
    return fail(CFRB_EINVAL, std::string(who) + "loss_kind must be CFRB_LOSS_HUBER or CFRB_LOSS_MSE");
  int rc;
  if ((rc = trainer_check_ptr(t, q, std::string(who) + "queries")) || (rc = trainer_check_ptr(t, v, std::string(who) + "values")))
    return rc;
  if (out && (rc = trainer_check_ptr(t, out, std::string(who) + "out"))) return rc;
  return CFRB_OK;
}

// Forward pass and loss of n rows: pred, row_loss and dpred in the trainer's scratch.
static int trainer_forward(cfrb_trainer* t, const float* q, const float* vals, int n, int loss_kind, cudaStream_t st) {
  using namespace cfrb::train;
  const auto& L = t->L;
  const float* P = t->params.p;
  const int Q = t->Q, H = t->H, rb = (n + kRowsPerBlock - 1) / kRowsPerBlock;
  Gemm f1{q, Q, 1, P + L.off[W1], 1, Q, t->z1.p, kHid, P + L.off[B1], n, kHid, Q};
  CK(launch_gemm(&f1, 1, st));
  ln_gelu_fwd<<<rb, 256, 0, st>>>(t->z1.p, P + L.off[G1], P + L.off[BE1], t->xh1.p, t->rs1.p, t->a1.p, n);
  Gemm f2{t->a1.p, kHid, 1, P + L.off[W2], 1, kHid, t->z2.p, kHid, P + L.off[B2], n, kHid, kHid};
  CK(launch_gemm(&f2, 1, st));
  ln_gelu_fwd<<<rb, 256, 0, st>>>(t->z2.p, P + L.off[G2], P + L.off[BE2], t->xh2.p, t->rs2.p, t->a2.p, n);
  Gemm f3{t->a2.p, kHid, 1, P + L.off[W3], 1, kHid, t->pred.p, H, P + L.off[B3], n, H, kHid};
  CK(launch_gemm(&f3, 1, st));
  loss_rows<<<rb, 256, 0, st>>>(t->pred.p, vals, n, H, loss_kind, t->row_loss.p, t->dpred.p);
  CK(cudaGetLastError());
  return CFRB_OK;
}

int cfrb_trainer_step(cfrb_trainer* t, const float* dev_q, const float* dev_v, int32_t n, double lr, double max_norm, int32_t loss_kind,
                      void* cuda_stream, float* dev_out) {
  using namespace cfrb::train;
  static const char* who = "cfrb_trainer_step: ";
  int rc = trainer_check_batch(t, who, dev_q, dev_v, n, loss_kind, dev_out);
  if (rc) return rc;
  if (!std::isfinite(lr) || lr < 0) return fail(CFRB_EINVAL, std::string(who) + "lr must be finite and >= 0");
  if (std::isnan(max_norm)) return fail(CFRB_EINVAL, std::string(who) + "max_norm is NaN");
  CK(cudaSetDevice(t->device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  if ((rc = trainer_forward(t, dev_q, dev_v, n, loss_kind, st))) return rc;
  const auto& L = t->L;
  float* P = t->params.p;
  float* G = t->grads.p;
  const int Q = t->Q, H = t->H, rb = (n + kRowsPerBlock - 1) / kRowsPerBlock;
  // output layer: dW3 = dpred^T a2, da2 = dpred W3
  const Gemm b3[2] = {{t->dpred.p, 1, H, t->a2.p, kHid, 1, G + L.off[W3], kHid, nullptr, H, kHid, n},
                      {t->dpred.p, H, 1, P + L.off[W3], kHid, 1, t->da2.p, kHid, nullptr, n, kHid, H}};
  CK(launch_gemm(b3, 2, st));
  ln_gelu_bwd<<<rb, 256, 0, st>>>(t->da2.p, t->xh2.p, t->rs2.p, P + L.off[G2], P + L.off[BE2], t->dy2.p, t->dz2.p, n);
  const ColJob c2[4] = {{t->dpred.p, nullptr, G + L.off[B3], H}, {t->dy2.p, t->xh2.p, G + L.off[G2], kHid},
                        {t->dy2.p, nullptr, G + L.off[BE2], kHid}, {t->dz2.p, nullptr, G + L.off[B2], kHid}};
  CK(launch_colsum(c2, 4, n, st));
  // hidden layer 2: dW2 = dz2^T a1, da1 = dz2 W2
  const Gemm b2[2] = {{t->dz2.p, 1, kHid, t->a1.p, kHid, 1, G + L.off[W2], kHid, nullptr, kHid, kHid, n},
                      {t->dz2.p, kHid, 1, P + L.off[W2], kHid, 1, t->da1.p, kHid, nullptr, n, kHid, kHid}};
  CK(launch_gemm(b2, 2, st));
  ln_gelu_bwd<<<rb, 256, 0, st>>>(t->da1.p, t->xh1.p, t->rs1.p, P + L.off[G1], P + L.off[BE1], t->dy1.p, t->dz1.p, n);
  const ColJob c1[3] = {{t->dy1.p, t->xh1.p, G + L.off[G1], kHid}, {t->dy1.p, nullptr, G + L.off[BE1], kHid},
                        {t->dz1.p, nullptr, G + L.off[B1], kHid}};
  CK(launch_colsum(c1, 3, n, st));
  // hidden layer 1: dW1 = dz1^T q
  const Gemm b1{t->dz1.p, 1, kHid, dev_q, Q, 1, G + L.off[W1], Q, nullptr, kHid, Q, n};
  CK(launch_gemm(&b1, 1, st));
  FinishArgs fa{G, L, t->sq_norms.p, t->step.p, t->row_loss.p, n, t->last.p, dev_out};
  finish_kernel<<<kParams + 1, 256, 0, st>>>(fa);
  CK(cudaGetLastError());
  AdamArgs aa{P, G, t->m.p, t->v.p, L.total(), t->sq_norms.p, t->step.p, lr, (float)max_norm, t->last.p, dev_out};
  const int blocks = (int)std::min<int64_t>((L.total() + 255) / 256, 1024);
  adam_kernel<<<blocks, 256, 0, st>>>(aa);
  CK(cudaGetLastError());
  return CFRB_OK;
}

int cfrb_trainer_loss(cfrb_trainer* t, const float* dev_q, const float* dev_v, int32_t n, int32_t loss_kind, void* cuda_stream,
                      float* dev_out) {
  using namespace cfrb::train;
  int rc = trainer_check_batch(t, "cfrb_trainer_loss: ", dev_q, dev_v, n, loss_kind, dev_out);
  if (rc) return rc;
  if (!dev_out) return fail(CFRB_EINVAL, "cfrb_trainer_loss: out is NULL");
  CK(cudaSetDevice(t->device));
  cudaStream_t st = (cudaStream_t)cuda_stream;
  if ((rc = trainer_forward(t, dev_q, dev_v, n, loss_kind, st))) return rc;
  // the loss block alone; cfrb_trainer_last keeps reporting the most recent training step
  FinishArgs fa{t->grads.p, t->L, t->sq_norms.p, t->step.p, t->row_loss.p, n, nullptr, dev_out};
  finish_kernel<<<1, 256, 0, st>>>(fa);
  CK(cudaGetLastError());
  return CFRB_OK;
}

}  // extern "C"
