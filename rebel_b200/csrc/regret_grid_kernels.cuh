// Immediate regrets of full-tree strategies on the whole GPU (compute_immediate_regrets, subgame_solving.cc:984-1050), in the
// level-synchronous style of the full-game solver (full_game_kernels.cuh): one launch per depth level over all (node, hand)
// entries of the level, spread over every SM, instead of regret_values_kernel's one CTA per (strategy, traverser).  The sums are
// compact fp64 [edge = child - 1][H] instead of regret_accumulate_kernel's dense [N][H][A].
//
// Per strategy: top-down reach of both players (evr::reach_pass), terminal payoffs of both traversers from one 9-bin histogram
// each of the opponent's reach (evr::terminal_pass), bottom-up values of both traversers (evr::value_pass).  The value pass of
// a node whose acting player is t also adds traverser t's values into the sums of its edges: acc[j] += value(child j) for every
// child in action order, then acc[j] -= value(node) for every child, regret_accumulate_kernel's sequence.  Compiled in the
// -fmad=false unit, every value and every sum takes the rounded operations of the dense path in its order, so the sums and the
// immediate regrets are bit-identical to cfrb_regrets_*.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"
#include "ev_regret_kernels.cuh"

namespace cfrb {

__device__ __forceinline__ int rg_threads() { return gridDim.x * blockDim.x; }

// Level d's children [nb, ne) of both players' reach: reach_p(c) = reach_p(parent) x strategy(c) where p acts, a copy elsewhere.
template <typename S>
__global__ void rg_reach_kernel(RegretGridDev p, const S* __restrict__ strategy, int nb, int ne, int d) {
  const int H = p.H, actor = (d - 1) & 1;   // the root is player 0's node
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += rg_threads()) {
    const int c = nb + (int)(it / H), h = (int)(it % H);
    const size_t pi = (size_t)p.parent[c] * H + h, ci = (size_t)c * H + h;
    const double a0 = d == 1 ? 1. / H : p.reach0[pi], a1 = d == 1 ? 1. / H : p.reach1[pi];   // get_initial_beliefs at the root
    const double s = (double)strategy[(size_t)(c - 1) * H + h];
    p.reach0[ci] = actor == 0 ? a0 * s : a0;
    p.reach1[ci] = actor == 1 ? a1 * s : a1;
  }
}

// One thread per terminal: the match-count histograms of reach1 (traverser 0's opponent) and reach0 (traverser 1's), each summed
// in hand order, then both traversers' payoffs of every hand.
__global__ void rg_terminal_kernel(RegretGridDev p) {
  constexpr int kMaxBins = evr::kMaxBins;   // evr::terminal_pass's histogram, whose operations this kernel repeats
  const int H = p.H, T = p.T;
  for (int z = blockIdx.x * blockDim.x + threadIdx.x; z < T; z += rg_threads()) {
    const int n = p.term_node[z], pbid = p.term_node[T + z], ndepth = p.term_node[2 * T + z];
    const int face = pbid % p.F;
    const double* r1 = p.reach1 + (size_t)n * H;
    const double* r0 = p.reach0 + (size_t)n * H;
    double c1[kMaxBins], c0[kMaxBins];
#pragma unroll
    for (int m = 0; m < kMaxBins; ++m) c1[m] = c0[m] = 0;
    double t1 = 0, t0 = 0;
    for (int g = 0; g < H; ++g) {
      const double x1 = r1[g], x0 = r0[g];
      const int mg = (int)p.matches[g * p.F + face];
      t1 += x1;
      t0 += x0;
#pragma unroll
      for (int m = 0; m < kMaxBins; ++m) {
        c1[m] += (m == mg) ? x1 : 0.0;
        c0[m] += (m == mg) ? x0 : 0.0;
      }
    }
#pragma unroll
    for (int m = kMaxBins - 2; m >= 0; --m) {
      c1[m] += c1[m + 1];
      c0[m] += c0[m + 1];
    }
    const int quantity = 1 + pbid / p.F;
    double* v0 = p.val0 + (size_t)n * H;
    double* v1 = p.val1 + (size_t)n * H;
    for (int h = 0; h < H; ++h) {
      int left = quantity - (int)p.matches[h * p.F + face];
      left = left < 0 ? 0 : (left > kMaxBins - 1 ? kMaxBins - 1 : left);
      const double w0 = (double)(float)c1[left] * 2 - t1;   // traverser 0 against reach1
      const double w1 = (double)(float)c0[left] * 2 - t0;   // traverser 1 against reach0
      v0[h] = (ndepth & 1) != 0 ? -w0 : w0;                  // the bidder (player ndepth & 1) wins
      v1[h] = (ndepth & 1) != 1 ? -w1 : w1;
    }
  }
}

// Level d's nodes [nb, ne): both traversers' values from their children (the strategy-weighted sum at the traverser's own nodes,
// the plain sum elsewhere), then the acting player's (d & 1) regret sums of the node's edges.
template <typename S>
__global__ void rg_value_kernel(RegretGridDev p, const S* __restrict__ strategy, int nb, int ne, int d) {
  const int H = p.H, actor = d & 1;
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += rg_threads()) {
    const int n = nb + (int)(it / H), h = (int)(it % H);
    const int nc = p.nchild[n];
    if (!nc) continue;
    const int c0 = p.child_begin[n];
    const double* w0 = p.val0 + (size_t)c0 * H + h;   // child j at w0[j * H]
    const double* w1 = p.val1 + (size_t)c0 * H + h;
    const S* sg = strategy + (size_t)(c0 - 1) * H + h;
    double v0 = 0, v1 = 0;
    if (actor == 0) {
      for (int j = 0; j < nc; ++j) v0 += w0[(size_t)j * H] * (double)sg[(size_t)j * H];
      for (int j = 0; j < nc; ++j) v1 += w1[(size_t)j * H];
    } else {
      for (int j = 0; j < nc; ++j) v0 += w0[(size_t)j * H];
      for (int j = 0; j < nc; ++j) v1 += w1[(size_t)j * H] * (double)sg[(size_t)j * H];
    }
    p.val0[(size_t)n * H + h] = v0;
    p.val1[(size_t)n * H + h] = v1;
    const double* w = actor == 0 ? w0 : w1;
    const double vn = actor == 0 ? v0 : v1;
    double* acc = p.acc + (size_t)(c0 - 1) * H + h;
    for (int j = 0; j < nc; ++j) acc[(size_t)j * H] += w[(size_t)j * H];
    for (int j = 0; j < nc; ++j) acc[(size_t)j * H] -= vn;
  }
}

// Read-out, one warp per node: immediate[n][h] = the largest of the A action slots (legal ones from the sums, 0.0 for illegal
// ones; the first maximum wins, as cfrb_regrets_fetch takes it) / count, 0 at leaves; then node_sums[n] = sum over hands in hand
// order (report_regrets' inner loop, recursive_eval.cc:41-52).
__global__ void rg_readout_kernel(RegretGridDev p, double count, double* __restrict__ immediate, double* __restrict__ node_sums) {
  const int H = p.H, A = p.A, lane = threadIdx.x & 31;
  const int warps = rg_threads() >> 5, first = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  for (int n = first; n < p.N; n += warps) {
    const int nc = p.nchild[n];
    const int lo = p.act_lo[n], c0 = p.child_begin[n];
    for (int h = lane; h < H; h += 32) {
      double m = 0.0;
      if (nc) {
        const double* r = p.acc + (size_t)(c0 - 1) * H + h;   // legal slot a = lo + j at r[j * H]
        m = lo == 0 ? r[0] : 0.0;
        for (int a = 1; a < A; ++a) {
          const double x = (a >= lo && a < lo + nc) ? r[(size_t)(a - lo) * H] : 0.0;
          if (m < x) m = x;
        }
        m = m / count;
      }
      immediate[(size_t)n * H + h] = m;
    }
    __syncwarp();
    if (lane == 0) {
      double s = 0;
      for (int h = 0; h < H; ++h) s += immediate[(size_t)n * H + h];
      node_sums[n] = s;
    }
  }
}

}  // namespace cfrb
