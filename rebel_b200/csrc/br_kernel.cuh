// Best response against a fixed full-tree strategy: BRSolver::compute_br + compute_exploitability2
// (subgame_solving.cc:316-358, 802-816) for both traversers in one launch (CTA t = traverser t).  Same phases as the CFR
// kernels — top-down reach (:54-78), terminal payoffs by match-count histogram (:80-98, :765-789), bottom-up values — with
// max over the children at the traverser's nodes (first child wins ties, :336-337) and sums elsewhere.  Compiled in the
// -fmad=false translation unit and written in the reference's operation order: the result is bit-identical to the CPU code.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"

namespace cfrb {

__global__ void __launch_bounds__(1024) br_kernel(BrDev p) {
  const int trav = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
  const int H = p.H, N = p.N;
  double* reach0 = p.scratch + (size_t)trav * p.scratch_stride;
  double* reach1 = reach0 + (size_t)N * H;
  double* val = reach1 + (size_t)N * H;
  double* hist = val + (size_t)N * H;
  constexpr int kMaxBins = 9;            // match counts 0 .. 8; bin 8 stays empty for num_dice <= kMaxDice = 7 (cfr_types.h)
  static_assert(kMaxBins >= kMaxDice + 2, "a clamped `left` must land on an empty bin");
  for (int h = tid; h < H; h += nt) { reach0[h] = 1. / H; reach1[h] = 1. / H; }   // uniform beliefs (:806-809)
  __syncthreads();
  for (int d = 1; d < p.levels; ++d) {
    const int nb = p.level_begin[d], ne = p.level_begin[d + 1];
    const int actor = (d - 1) & 1;                     // the root is player 0's node
    for (int it = tid; it < (ne - nb) * H; it += nt) {
      const int c = nb + it / H, h = it % H;
      const int par = p.parent[c];
      const double s = p.strategy[(size_t)(c - 1) * H + h];
      const double a0 = reach0[par * H + h], a1 = reach1[par * H + h];
      reach0[c * H + h] = actor == 0 ? a0 * s : a0;
      reach1[c * H + h] = actor == 1 ? a1 * s : a1;
    }
    __syncthreads();
  }
  const double* ropp = trav == 0 ? reach1 : reach0;
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
    val[(size_t)n * H + h] = ((ndepth & 1) != trav) ? -v : v;
  }
  __syncthreads();
  for (int d = p.levels - 2; d >= 0; --d) {
    const int nb = p.level_begin[d], ne = p.level_begin[d + 1];
    const bool mine = (d & 1) == trav;
    for (int it = tid; it < (ne - nb) * H; it += nt) {
      const int n = nb + it / H, h = it % H;
      const int nc = p.nchild[n];
      if (!nc) continue;
      const int c0 = p.child_begin[n];
      double v = 0;
      if (mine) {
        for (int j = 0; j < nc; ++j) {
          const double nv = val[(size_t)(c0 + j) * H + h];
          if (j == 0 || nv > v) v = nv;
        }
      } else {
        for (int j = 0; j < nc; ++j) v += val[(size_t)(c0 + j) * H + h];
      }
      val[(size_t)n * H + h] = v;
    }
    __syncthreads();
  }
  if (tid == 0) {
    double s = 0;
    for (int h = 0; h < H; ++h) s += val[h];
    p.out[trav] = s / H;
  }
}

}  // namespace cfrb
