// Expected value against a second strategy (compute_ev / compute_ev2, subgame_solving.cc:931-982) and the immediate regrets of
// a list of strategies (compute_immediate_regrets, :984-1050) on the full tree of BrDev.  Same phases as br_kernel.cuh: top-down
// reach (:54-78), terminal payoffs by match-count histogram (:80-98, :765-789) and a bottom-up pass.  Compiled in the
// -fmad=false translation unit and written in the reference's operation order, so every result is bit-identical to the CPU code.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"

namespace cfrb {

namespace evr {
constexpr int kMaxBins = 9;

// reach_out[c] = reach_out[parent] * strategy(parent -> c) at `player`'s nodes, a copy elsewhere (compute_reach_probabilities)
template <typename S>
__device__ void reach_pass(const BrDev& p, const S* strategy, int player, double* reach) {
  const int H = p.H, tid = threadIdx.x, nt = blockDim.x;
  for (int h = tid; h < H; h += nt) reach[h] = 1. / H;   // get_initial_beliefs (subgame_solving.h:112-117)
  __syncthreads();
  for (int d = 1; d < p.levels; ++d) {
    const int nb = p.level_begin[d], ne = p.level_begin[d + 1];
    const bool acts = ((d - 1) & 1) == player;      // the root is player 0's node
    for (int it = tid; it < (ne - nb) * H; it += nt) {
      const int c = nb + it / H, h = it % H;
      const double a = reach[p.parent[c] * H + h];
      reach[c * H + h] = acts ? a * (double)strategy[(size_t)(c - 1) * H + h] : a;
    }
    __syncthreads();
  }
}

// compute_expected_terminal_values(inverse = player(z) != traverser) from the opponent's reach
__device__ void terminal_pass(const BrDev& p, const double* ropp, int traverser, double* hist, double* val) {
  const int H = p.H, tid = threadIdx.x, nt = blockDim.x;
  for (int z = tid; z < p.T; z += nt) {
    const int n = p.term_node[z];
    const int face = p.term_node[p.T + z] % p.F;
    const double* ro = ropp + (size_t)n * H;
    double cnt[kMaxBins];
#pragma unroll
    for (int m = 0; m < kMaxBins; ++m) cnt[m] = 0;
    double tot = 0;
    for (int g = 0; g < H; ++g) {
      const double r = ro[g];
      const int mg = (int)p.matches[g * p.F + face];
      tot += r;
#pragma unroll
      for (int m = 0; m < kMaxBins; ++m) cnt[m] += (m == mg) ? r : 0.0;
    }
#pragma unroll
    for (int m = kMaxBins - 2; m >= 0; --m) cnt[m] += cnt[m + 1];
#pragma unroll
    for (int m = 0; m < kMaxBins; ++m) hist[(size_t)z * (kMaxBins + 1) + m] = cnt[m];
    hist[(size_t)z * (kMaxBins + 1) + kMaxBins] = tot;
  }
  __syncthreads();
  for (int it = tid; it < p.T * H; it += nt) {
    const int z = it / H, h = it % H;
    const int n = p.term_node[z], pbid = p.term_node[p.T + z], ndepth = p.term_node[2 * p.T + z];
    const int quantity = 1 + pbid / p.F, face = pbid % p.F;
    int left = quantity - (int)p.matches[h * p.F + face];
    left = left < 0 ? 0 : (left > kMaxBins - 1 ? kMaxBins - 1 : left);
    const double win = hist[(size_t)z * (kMaxBins + 1) + left], tot = hist[(size_t)z * (kMaxBins + 1) + kMaxBins];
    const double v = (double)(float)win * 2 - tot;
    val[(size_t)n * H + h] = ((ndepth & 1) != traverser) ? -v : v;
  }
  __syncthreads();
}

// Bottom-up values of `traverser`: sum_a child * strategy at its own nodes, the plain sum over the children elsewhere.
template <typename S>
__device__ void value_pass(const BrDev& p, const S* strategy, int traverser, double* val) {
  const int H = p.H, tid = threadIdx.x, nt = blockDim.x;
  for (int d = p.levels - 2; d >= 0; --d) {
    const int nb = p.level_begin[d], ne = p.level_begin[d + 1];
    const bool mine = (d & 1) == traverser;
    for (int it = tid; it < (ne - nb) * H; it += nt) {
      const int n = nb + it / H, h = it % H;
      const int nc = p.nchild[n];
      if (!nc) continue;
      const int c0 = p.child_begin[n];
      double v = 0;
      if (mine) {
        for (int j = 0; j < nc; ++j) v += val[(size_t)(c0 + j) * H + h] * (double)strategy[(size_t)(c0 + j - 1) * H + h];
      } else {
        for (int j = 0; j < nc; ++j) v += val[(size_t)(c0 + j) * H + h];
      }
      val[(size_t)n * H + h] = v;
    }
    __syncthreads();
  }
}
}  // namespace evr

// compute_ev2: CTA 0 = compute_ev(s1, s2), CTA 1 = compute_ev(s2, s1); player 0's values under its own strategy (first
// argument) against player 1's reach under the second.  out = {sum / H, -sum' / H}.
__global__ void __launch_bounds__(1024) ev_kernel(BrDev p, const double* s1, const double* s2) {
  const int c = blockIdx.x;
  const double* own = c == 0 ? s1 : s2;
  const double* opp = c == 0 ? s2 : s1;
  double* reach1 = p.scratch + (size_t)c * p.scratch_stride;
  double* val = reach1 + (size_t)p.N * p.H;
  double* hist = val + (size_t)p.N * p.H;
  evr::reach_pass(p, opp, 1, reach1);
  evr::terminal_pass(p, reach1, 0, hist, val);
  evr::value_pass(p, own, 0, val);
  if (threadIdx.x == 0) {
    double s = 0;
    for (int h = 0; h < p.H; ++h) s += val[h];
    p.out[c] = c == 0 ? s / p.H : -s / p.H;
  }
}

// Per-strategy pass of compute_immediate_regrets: CTA (s, t) writes the traverser-t values of strategy s to
// val[(s * 2 + t) * N * H ...].  The strategies are compact [S][(N - 1) * H], either fp32 (s32) or fp64 (s64).
template <typename S>
__global__ void __launch_bounds__(1024) regret_values_kernel(RegretDev r, const S* strategies) {
  const BrDev& p = r.tree;
  const int s = blockIdx.x >> 1, t = blockIdx.x & 1;
  const S* sig = strategies + (size_t)s * r.s_stride;
  double* reach0 = p.scratch + (size_t)blockIdx.x * p.scratch_stride;
  double* reach1 = reach0 + (size_t)p.N * p.H;
  double* hist = reach1 + (size_t)p.N * p.H;
  double* val = r.val + (size_t)blockIdx.x * p.N * p.H;
  evr::reach_pass(p, sig, 0, reach0);
  evr::reach_pass(p, sig, 1, reach1);
  evr::terminal_pass(p, t == 0 ? reach1 : reach0, t, hist, val);
  evr::value_pass(p, sig, t, val);
}

// Ordered accumulation: one thread per (inner node, hand), strategies in list order, and per strategy the reference's sequence
// regrets[a] += value(child_a) for every legal action, then regrets[a] -= value(node) for every legal action.
__global__ void regret_accumulate_kernel(RegretDev r, int S) {
  const BrDev& p = r.tree;
  const int H = p.H, A = r.A;
  const size_t NH = (size_t)p.N * H;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < NH; i += (size_t)gridDim.x * blockDim.x) {
    const int n = (int)(i / H), h = (int)(i % H);
    const int nc = p.nchild[n];
    if (!nc) continue;
    const int c0 = p.child_begin[n], t = r.depth[n] & 1, lo = r.act_lo[n];
    double* acc = r.acc + i * A + lo;
    for (int s = 0; s < S; ++s) {
      const double* v = r.val + (size_t)(2 * s + t) * NH;
      for (int j = 0; j < nc; ++j) acc[j] += v[(size_t)(c0 + j) * H + h];
      const double vn = v[i];
      for (int j = 0; j < nc; ++j) acc[j] -= vn;
    }
  }
}

}  // namespace cfrb
