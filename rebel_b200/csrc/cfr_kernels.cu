// CFR wave kernels, compiled as their own translation unit with -fmad=false: without fused multiply-adds every fp64
// operation is an individually rounded IEEE operation in the same order as the reference's scalar C++ (built without
// contraction), which makes the CFRB_STATE_F64 path reproduce the reference bit for bit between value-net calls.
#include <algorithm>
#include <type_traits>

#include "cfr_kernels.cuh"
#include "br_kernel.cuh"
#include "ev_regret_kernels.cuh"
#include "selfplay_kernels.cuh"
#include "match_kernels.cuh"
#include "lbr_kernels.cuh"
#include "agent_kernels.cuh"
#include "ply_kernels.cuh"
#include "expl_kernels.cuh"
#include "full_game_kernels.cuh"
#include "regret_grid_kernels.cuh"
#include "fp_forest_kernels.cuh"

namespace cfrb {

// Hand counts with a compile-time specialisation (1x4f, 1x5f, 1x6f, 2x3f, 2x4f); anything else takes the generic path.
#define CFRB_DISPATCH_H(H, CALL)          \
  switch (H) {                            \
    case 4: { CALL(4); break; }           \
    case 5: { CALL(5); break; }           \
    case 6: { CALL(6); break; }           \
    case 9: { CALL(9); break; }           \
    case 16: { CALL(16); break; }         \
    default: { CALL(0); break; }          \
  }

// The dynamic shared-memory limit is an attribute of the kernel, shared by every handle of the process: each handle raises it to
// the device's opt-in maximum, so that a handle created later with a smaller need (another game or tree depth, e.g. an
// exploitability evaluation beside running generator loops) cannot lower it under the launches of an earlier one.
static int smem_limit(int smem_bytes) {
  int dev = 0, optin = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return smem_bytes;
  return std::max(smem_bytes, optin);
}

template <typename real>
cudaError_t cfr_configure(int group, int smem_bytes) {
  if (group != 32) return cudaSuccess;
  cudaError_t e = cudaSuccess;
  const int limit = smem_limit(smem_bytes);
#define CFRB_CFG(HC)                                                                                                      \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(cfr_iter_kernel<real, 32, HC>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit);
  CFRB_CFG(0) CFRB_CFG(4) CFRB_CFG(5) CFRB_CFG(6) CFRB_CFG(9) CFRB_CFG(16)
#undef CFRB_CFG
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(cfr_init_kernel<real, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit);
}

template <typename real>
void cfr_launch_init(const CfrDev<real>& p, int group, int blocks, int threads, size_t smem, cudaStream_t st, int scratch_per_group) {
  if (group == 32) cfr_init_kernel<real, 32><<<blocks, threads, smem, st>>>(p, scratch_per_group);
  else cfr_init_kernel<real, 256><<<blocks, 256, 0, st>>>(p, scratch_per_group);
}

template <typename real>
void cfr_launch_iter(const CfrDev<real>& p, int group, int blocks, int threads, size_t smem, cudaStream_t st, int iter, int do_b,
                     int do_f, int scratch_per_group) {
  if (group == 32) {
#define CFRB_CALL(HC) cfr_iter_kernel<real, 32, HC><<<blocks, threads, smem, st>>>(p, iter, do_b, do_f, scratch_per_group)
    CFRB_DISPATCH_H(p.H, CFRB_CALL)
#undef CFRB_CALL
  } else {
    cfr_iter_kernel<real, 256, 0><<<blocks, 256, 0, st>>>(p, iter, do_b, do_f, scratch_per_group);
  }
}

void br_launch(const BrDev& p, cudaStream_t st) { br_kernel<<<2, 1024, 0, st>>>(p); }

void ev_launch(const BrDev& p, const double* s1, const double* s2, cudaStream_t st) { ev_kernel<<<2, 1024, 0, st>>>(p, s1, s2); }

void regret_launch(const RegretDev& r, const float* s32, const double* s64, int S, cudaStream_t st) {
  if (S <= 0) return;
  if (s32) regret_values_kernel<float><<<2 * S, 1024, 0, st>>>(r, s32);
  else regret_values_kernel<double><<<2 * S, 1024, 0, st>>>(r, s64);
  const size_t nh = (size_t)r.tree.N * r.tree.H;
  const int blocks = (int)std::min<size_t>((nh + 255) / 256, 132 * 8);
  regret_accumulate_kernel<<<blocks, 256, 0, st>>>(r, S);
}

template <typename real>
cudaError_t cfr_configure_d2(int H, int threads, int smem_bytes, int* ctas_per_sm) {
  cudaError_t e = cudaSuccess;
  const int limit = smem_limit(smem_bytes);
#define CFRB_CFG1(HC, KEEP, WIDE)                                                                                                      \
  if (e == cudaSuccess) e = cudaFuncSetAttribute(cfr_iter_d2_kernel<real, HC, KEEP, WIDE>, cudaFuncAttributeMaxDynamicSharedMemorySize, limit);
#define CFRB_CFG(HC) CFRB_CFG1(HC, true, true) CFRB_CFG1(HC, false, true) CFRB_CFG1(HC, true, false) CFRB_CFG1(HC, false, false)
  CFRB_CFG(0) CFRB_CFG(4) CFRB_CFG(5) CFRB_CFG(6) CFRB_CFG(9) CFRB_CFG(16)
#undef CFRB_CFG
#undef CFRB_CFG1
  if (e != cudaSuccess) return e;
  // the persistent grid of every variant (with and without the sum table, with and without wide tickets): the smallest residency
  int occ[4] = {0, 0, 0, 0};
#define CFRB_OCC(HC)                                                                                                              \
  e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], cfr_iter_d2_kernel<real, HC, true, true>, threads, smem_bytes);         \
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], cfr_iter_d2_kernel<real, HC, false, true>, threads, smem_bytes);  \
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[2], cfr_iter_d2_kernel<real, HC, true, false>, threads, smem_bytes);  \
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[3], cfr_iter_d2_kernel<real, HC, false, false>, threads, smem_bytes);
  CFRB_DISPATCH_H(H, CFRB_OCC)
#undef CFRB_OCC
  *ctas_per_sm = std::min(std::min(occ[0], occ[1]), std::min(occ[2], occ[3]));
  return e;
}

// Launch with programmatic stream serialization (PDL): the grid may start before its predecessor in the stream has finished;
// the kernel orders itself with griddepcontrol.wait.  Captured into CUDA graphs as a programmatic dependency edge.
template <typename... KArgs, typename... Args>
static void launch_pdl(void (*kernel)(KArgs...), int blocks, int threads, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, args...);
}

template <typename real>
void cfr_launch_iter_d2(const CfrDev<real>& p, int blocks, int threads, size_t smem, cudaStream_t st, int iter, int do_b, int do_f,
                        int scratch_per_group) {
#define CFRB_KEEP(HC) launch_pdl(cfr_iter_d2_kernel<real, HC, true, W>, blocks, threads, smem, st, p, iter, do_b, do_f, scratch_per_group)
#define CFRB_DROP(HC) launch_pdl(cfr_iter_d2_kernel<real, HC, false, W>, blocks, threads, smem, st, p, iter, do_b, do_f, scratch_per_group)
  auto launch = [&](auto wide) {
    constexpr bool W = decltype(wide)::value;
    if (p.keep_sum || p.fp) {
      CFRB_DISPATCH_H(p.H, CFRB_KEEP)
    } else {
      CFRB_DISPATCH_H(p.H, CFRB_DROP)
    }
  };
  // waves that can take wide tickets get the kernel with them; the others keep the narrow loop's registers
  if (p.wide != nullptr) launch(std::true_type{});
  else launch(std::false_type{});
#undef CFRB_KEEP
#undef CFRB_DROP
}

void sp_launch_seed(const SpDev& p, const uint32_t* dev_seeds, cudaStream_t st) {
  sp_seed_kernel<<<(p.K + 127) / 128, 128, 0, st>>>(p, dev_seeds);
}
template <typename real>
void sp_launch_begin(const SpDev& p, real* wave_beliefs, cudaStream_t st) {
  sp_begin_kernel<real><<<(p.K + 127) / 128, 128, 0, st>>>(p, wave_beliefs);
  sp_scan_kernel<<<1, 1024, 0, st>>>(p);
}
template <typename real>
void sp_launch_finish(const SpDev& p, const real* mu, const real* snap, float* ex_q, float* ex_v, cudaStream_t st) {
  if (ex_q) sp_examples_kernel<real><<<(2 * p.K + 127) / 128, 128, 0, st>>>(p, mu, ex_q, ex_v);
  sp_advance_kernel<real><<<(p.K + 127) / 128, 128, 0, st>>>(p, snap);
}
template <typename real>
void sp_launch_share(const SpDev& p, const CfrDev<real>& d, cudaStream_t st) {
  sp_share_kernel<real><<<p.K, 128, 0, st>>>(p, d);
}
void match_launch_deal(const MatchDev& p, cudaStream_t st) { match_deal_kernel<match_start><<<(p.S + 127) / 128, 128, 0, st>>>(p); }
template <typename real>
void match_launch_begin(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  match_scan_kernel<<<1, 1024, 0, st>>>(p);
  match_begin_kernel<real><<<(p.S + 127) / 128, 128, 0, st>>>(p, t);
}
template <typename real>
void match_launch_advance(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  match_advance_kernel<real><<<(p.S + 127) / 128, 128, 0, st>>>(p, t);
}
void ply_launch_deal(const MatchDev& p, cudaStream_t st) { match_deal_kernel<ply_start><<<(p.S + 127) / 128, 128, 0, st>>>(p); }
template <typename real>
void ply_launch_begin(const MatchDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  ply_scan_kernel<<<1, 1024, 0, st>>>(p);
  ply_begin_kernel<real><<<(p.S + 127) / 128, 128, 0, st>>>(p, t);
}
template <typename real>
void ply_launch_advance(const MatchDev& p, const MatchTabs<real>& t, bool capture, cudaStream_t st) {
  if (capture) ply_capture_kernel<real><<<(2 * p.S + 3) / 4, 128, 0, st>>>(p, t);
  ply_advance_kernel<real><<<(p.S + 127) / 128, 128, 0, st>>>(p, t);
}
template <typename real>
void lbr_launch_begin(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  lbr_scan_kernel<<<1, 1024, 0, st>>>(p);
  lbr_begin_kernel<real><<<(p.m.S + 127) / 128, 128, 0, st>>>(p, t);
}
template <typename real>
void lbr_launch_advance(const LbrDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  lbr_advance_kernel<real><<<(p.m.S + 127) / 128, 128, 0, st>>>(p, t);
}
void lbr_launch_blueprint(const LbrDev& p, cudaStream_t st) { lbr_blueprint_kernel<<<(p.m.S + 127) / 128, 128, 0, st>>>(p); }
void agent_launch_new(const AgentDev& p, cudaStream_t st) { agent_new_kernel<<<(p.n + 127) / 128, 128, 0, st>>>(p); }
template <typename real>
void agent_launch_begin(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  agent_scan_kernel<<<1, 1024, 0, st>>>(p);
  agent_begin_kernel<real><<<(p.n + 127) / 128, 128, 0, st>>>(p, t);
}
template <typename real>
void agent_launch_capture(const AgentDev& p, const MatchTabs<real>& t, cudaStream_t st) {
  agent_capture_kernel<real><<<(p.n + 3) / 4, 128, 0, st>>>(p, t);
}
void agent_launch_step(const AgentDev& p, cudaStream_t st) { agent_step_kernel<<<(p.n + 127) / 128, 128, 0, st>>>(p); }
void agent_launch_policy(const AgentDev& p, cudaStream_t st) {
  agent_policy_kernel<<<(p.n * p.H + 127) / 128, 128, 0, st>>>(p);
}
template <typename real>
void expl_launch_begin(const ExplDev& p, const SpDev& scan, int n, real* wave_beliefs, cudaStream_t st) {
  expl_begin_kernel<real><<<(n + 127) / 128, 128, 0, st>>>(p, n, wave_beliefs);
  sp_scan_kernel<<<1, 1024, 0, st>>>(scan);
}
template <typename real>
void expl_launch_expand(const ExplDev& p, int n, const real* table, int normalise, cudaStream_t st) {
  expl_expand_kernel<real><<<n, 128, 0, st>>>(p, table, normalise);
  expl_fill_kernel<<<1, 1, 0, st>>>(p);
}
template <typename real>
void rec_launch_expand(const ExplDev& p, int n, const real* table, int normalise, cudaStream_t st) {
  rec_expand_kernel<real><<<(n + 3) / 4, 128, 0, st>>>(p, n, table, normalise);   // a warp per subgame
}
template <typename real>
void expl_sampled_launch_expand(const ExplDev& p, int n, const real* snap, cudaStream_t st) {
  expl_sampled_expand_kernel<real><<<n / p.b, 128, 0, st>>>(p, snap);
  expl_fill_kernel<<<1, 1, 0, st>>>(p);
}
void expl_sampled_launch_finalize(const ExplDev& p, cudaStream_t st) {
  const size_t total = (size_t)(p.full_nodes - 1) * p.H;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 8);
  expl_sampled_finalize_kernel<<<std::max(blocks, 1), 256, 0, st>>>(p);
}
// Full-game solver: level_begin is the host copy of the full tree's [levels + 1] level starts; grids are sized per level.
static int fg_blocks(long long items, int max_blocks) {
  return (int)std::max<long long>(1, std::min<long long>((items + 255) / 256, max_blocks));
}
void full_game_launch_init(const FullGameDev& p, const int* level_begin, int levels, int max_blocks, cudaStream_t st) {
  for (int d = 1; d < levels; ++d) {
    const int nb = level_begin[d], ne = level_begin[d + 1];
    fg_init_kernel<<<fg_blocks((long long)(ne - nb) * p.H, max_blocks), 256, 0, st>>>(p, nb, ne, d);
  }
}
void full_game_launch_iter(const FullGameDev& p, const int* level_begin, int levels, int max_blocks, cudaStream_t st) {
  auto blocks = [&](int d) { return fg_blocks((long long)(level_begin[d + 1] - level_begin[d]) * p.H, max_blocks); };
  if (p.fp)
    for (int d = 1; d < levels; ++d) fg_reach_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  fg_terminal_kernel<<<fg_blocks(p.T, max_blocks), 256, 0, st>>>(p);
  for (int d = levels - 2; d >= 0; --d) fg_up_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  for (int d = 0; d + 1 < levels; ++d) fg_down_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  fg_advance_kernel<<<1, 1, 0, st>>>(p.iter);
}
// FP subtree forest from level d0 (fp_forest_kernels.cuh): the full-game solver's launches on levels d0 .. levels - 1.
void fp_forest_launch_init(const FullGameDev& p, const double* bel, double* mu, const int* level_begin, int levels, int d0, int max_blocks,
                           cudaStream_t st) {
  const int nb = level_begin[d0], ne = level_begin[d0 + 1];
  ff_root_init_kernel<<<fg_blocks((long long)(ne - nb) * p.H, max_blocks), 256, 0, st>>>(p, bel, mu, nb, ne);
  for (int d = d0 + 1; d < levels; ++d)
    fg_init_kernel<<<fg_blocks((long long)(level_begin[d + 1] - level_begin[d]) * p.H, max_blocks), 256, 0, st>>>(p, level_begin[d],
                                                                                                               level_begin[d + 1], d);
}
void fp_forest_launch_iter(const FullGameDev& p, const double* bel, double* mu, const int* level_begin, int levels, int d0, int max_blocks,
                           cudaStream_t st) {
  auto blocks = [&](int d) { return fg_blocks((long long)(level_begin[d + 1] - level_begin[d]) * p.H, max_blocks); };
  const int nb = level_begin[d0], ne = level_begin[d0 + 1];
  ff_root_reach_kernel<<<blocks(d0), 256, 0, st>>>(p, bel, nb, ne);
  for (int d = d0 + 1; d < levels; ++d) fg_reach_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  fg_terminal_kernel<<<fg_blocks(p.T, max_blocks), 256, 0, st>>>(p);
  for (int d = levels - 2; d >= d0; --d) fg_up_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  ff_root_mean_kernel<<<blocks(d0), 256, 0, st>>>(p, bel, mu, nb, ne);
  for (int d = d0; d + 1 < levels; ++d) fg_down_kernel<<<blocks(d), 256, 0, st>>>(p, level_begin[d], level_begin[d + 1], d);
  fg_advance_kernel<<<1, 1, 0, st>>>(p.iter);
}
void fp_forest_launch_reach(const RegretGridDev& p, const double* strategy, const int* nodes, int n, double* node_reach, double* rows,
                            const int* level_begin, int levels, int max_blocks, cudaStream_t st) {
  auto blocks = [&](int d) { return fg_blocks((long long)(level_begin[d + 1] - level_begin[d]) * p.H, max_blocks); };
  for (int d = 1; d < levels; ++d) rg_reach_kernel<double><<<blocks(d), 256, 0, st>>>(p, strategy, level_begin[d], level_begin[d + 1], d);
  ff_gather_kernel<<<fg_blocks(n, max_blocks), 256, 0, st>>>(p, nodes, n, node_reach, rows);
}
// Grid-wide immediate regrets: the same level-by-level grid sizes as the full-game solver.
template <typename S>
static void regret_grid_launch_t(const RegretGridDev& p, const S* s, const int* level_begin, int levels, int max_blocks, cudaStream_t st) {
  auto blocks = [&](int d) { return fg_blocks((long long)(level_begin[d + 1] - level_begin[d]) * p.H, max_blocks); };
  for (int d = 1; d < levels; ++d) rg_reach_kernel<S><<<blocks(d), 256, 0, st>>>(p, s, level_begin[d], level_begin[d + 1], d);
  rg_terminal_kernel<<<fg_blocks(p.T, max_blocks), 256, 0, st>>>(p);
  for (int d = levels - 2; d >= 0; --d) rg_value_kernel<S><<<blocks(d), 256, 0, st>>>(p, s, level_begin[d], level_begin[d + 1], d);
}
void regret_grid_launch(const RegretGridDev& p, const float* s32, const double* s64, const int* level_begin, int levels, int max_blocks,
                        cudaStream_t st) {
  if (s32) regret_grid_launch_t(p, s32, level_begin, levels, max_blocks, st);
  else regret_grid_launch_t(p, s64, level_begin, levels, max_blocks, st);
}
void regret_grid_launch_readout(const RegretGridDev& p, double count, double* immediate, double* node_sums, int max_blocks,
                                cudaStream_t st) {
  rg_readout_kernel<<<fg_blocks((long long)p.N * 32, max_blocks), 256, 0, st>>>(p, count, immediate, node_sums);
}
void full_game_launch_average(const FullGameDev& p, const int* depth, int untouched0, int untouched1, int max_blocks, cudaStream_t st) {
  fg_average_kernel<<<fg_blocks((long long)p.N * p.H, max_blocks), 256, 0, st>>>(p, depth, untouched0, untouched1);
}

__global__ void rows_gather_kernel(const float* __restrict__ src, int width, const int* __restrict__ ids, int n, float* __restrict__ out) {
  const size_t total = (size_t)n * width;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int r = (int)(i / width), c = (int)(i % width);
    out[i] = src[(size_t)ids[r] * width + c];
  }
}
void rows_launch_gather(const float* src, int width, const int* ids, int n, float* out, cudaStream_t st) {
  if (n <= 0) return;
  const size_t total = (size_t)n * width;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, 132 * 8);   // grid-stride: 8 CTAs per SM of an H100
  rows_gather_kernel<<<blocks, 256, 0, st>>>(src, width, ids, n, out);
}

// div_by_rcp against IEEE division on pseudo-random operands: quotient mantissas spread over [1, 2), including operands whose
// quotient lies within a few ulp of a power of two and denominators with all-ones / all-zeros low mantissa bits.
__global__ void div_check_kernel(unsigned long long seed, unsigned long long* mismatches) {
  unsigned long long s = seed + (unsigned long long)(blockIdx.x * blockDim.x + threadIdx.x) * 0x9E3779B97F4A7C15ull;
  auto next = [&]() { s ^= s << 13; s ^= s >> 7; s ^= s << 17; return s; };
  unsigned long long bad = 0;
  for (int i = 0; i < 4096; ++i) {
    const unsigned long long a = next(), c = next(), m = next();
    double b = __longlong_as_double((long long)(0x3FF0000000000000ull | (c >> 12)));           // [1, 2)
    double x = __longlong_as_double((long long)(0x3FF0000000000000ull | (a >> 12)));
    const int kind = (int)(m & 7);
    if (kind == 1) b = __longlong_as_double((long long)(0x3FFFFFFFFFFFFF00ull | (c & 0xFF)));     // denominator just below 2
    if (kind == 2) b = __longlong_as_double((long long)(0x3FF0000000000000ull | (c & 0xFF)));     // just above 1
    if (kind == 3) x = b * (1.0 + (double)((long long)(a & 0xF) - 8) * 2.220446049250313e-16);      // quotient within a few ulp of 1
    if (kind == 4) x = x * 1e-80;                                                                   // the smoothing epsilon's scale
    if (kind == 5) b = b * (double)(1 + (c & 15));                                                  // sums of up to a dozen regrets
    const double y = 1.0 / b;
    const double q = div_by_rcp(x, b, y);
    if (__double_as_longlong(q) != __double_as_longlong(x / b)) ++bad;
  }
  if (bad) atomicAdd(mismatches, bad);
}
void div_check_launch(unsigned long long seed, int blocks, unsigned long long* mismatches, cudaStream_t st) {
  div_check_kernel<<<blocks, 256, 0, st>>>(seed, mismatches);
}

#define CFRB_INSTANTIATE(real)                                                                                             \
  template cudaError_t cfr_configure<real>(int, int);                                                                      \
  template void cfr_launch_init<real>(const CfrDev<real>&, int, int, int, size_t, cudaStream_t, int);                      \
  template void cfr_launch_iter<real>(const CfrDev<real>&, int, int, int, size_t, cudaStream_t, int, int, int, int);             \
  template cudaError_t cfr_configure_d2<real>(int, int, int, int*);                                                        \
  template void cfr_launch_iter_d2<real>(const CfrDev<real>&, int, int, size_t, cudaStream_t, int, int, int, int);                \
  template void sp_launch_begin<real>(const SpDev&, real*, cudaStream_t);                                                  \
  template void sp_launch_finish<real>(const SpDev&, const real*, const real*, float*, float*, cudaStream_t);              \
  template void sp_launch_share<real>(const SpDev&, const CfrDev<real>&, cudaStream_t);                                    \
  template void match_launch_begin<real>(const MatchDev&, const MatchTabs<real>&, cudaStream_t);                           \
  template void match_launch_advance<real>(const MatchDev&, const MatchTabs<real>&, cudaStream_t);                         \
  template void ply_launch_begin<real>(const MatchDev&, const MatchTabs<real>&, cudaStream_t);                             \
  template void ply_launch_advance<real>(const MatchDev&, const MatchTabs<real>&, bool, cudaStream_t);                     \
  template void lbr_launch_begin<real>(const LbrDev&, const MatchTabs<real>&, cudaStream_t);                               \
  template void lbr_launch_advance<real>(const LbrDev&, const MatchTabs<real>&, cudaStream_t);                             \
  template void agent_launch_begin<real>(const AgentDev&, const MatchTabs<real>&, cudaStream_t);                           \
  template void agent_launch_capture<real>(const AgentDev&, const MatchTabs<real>&, cudaStream_t);                         \
  template void expl_launch_begin<real>(const ExplDev&, const SpDev&, int, real*, cudaStream_t);                           \
  template void expl_launch_expand<real>(const ExplDev&, int, const real*, int, cudaStream_t);                              \
  template void rec_launch_expand<real>(const ExplDev&, int, const real*, int, cudaStream_t);                               \
  template void expl_sampled_launch_expand<real>(const ExplDev&, int, const real*, cudaStream_t);
CFRB_INSTANTIATE(float)
CFRB_INSTANTIATE(double)

}  // namespace cfrb
