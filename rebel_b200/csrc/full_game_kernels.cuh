// Full-game solver on the whole GPU (cfrb_full_game_*): CFR and fictitious play over the full tree of a game, one level of
// (node, hand) entries per launch, the entries of a level spread over every SM.  The one-CTA solver (cfr_iter_kernel with a
// CTA per subgame) walks the same tree level by level inside one CTA; here each of its level loops is a launch of its own.
//
// Layout (fp64): per edge [edge = child - 1][H] the regrets R (CFR), the current strategy Sg (FP: the average strategy) and the
// sum strategy S; per node [N][H] the reach of one player and the values.  The full tree's index arrays are the handle's
// (full_tree_setup), root player 0.
//
// Bit-identical to cfr_iter_kernel: every (node, hand) entry runs that kernel's fp64 operations in its order (children summed in
// action order, the same products and quotients), compiled in the -fmad=false translation unit.  Only independent entries run in
// parallel; no sum is split.  Two fusions change no value: a parent's entry computes the value x sigma products of its children
// inline instead of reading them back from a scratch buffer (the same rounded products), and its new regrets and strategies in
// the same thread.  The reach table holds the reach of ONE player: after a CFR iteration's top-down pass it is the traverser's
// reach under the new strategy, which is exactly what the next iteration's terminal payoffs need (the opponent's reach, the
// `have` shortcut of cfr_forward).  FP rebuilds it each iteration (its average strategy changes after the reach is taken), and
// keeps the best-response flags of the bottom-up pass in it, where cfr_iter_kernel keeps them in its second scratch buffer.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"
#include "selfplay_kernels.cuh"

namespace cfrb {

__device__ __forceinline__ int fg_threads() { return gridDim.x * blockDim.x; }

// CFR constructor (cfr_init_kernel) on level d's nodes [nb, ne): uniform strategy, zero regrets, sum = uniform x the actor's reach
// under the uniform strategy.  val carries player 0's reach, reach player 1's (the opponent of iteration 0's traverser).
__global__ void fg_init_kernel(FullGameDev p, int nb, int ne, int d) {
  const int H = p.H, actor = (d - 1) & 1;
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int c = nb + (int)(it / H), h = (int)(it % H);
    const int par = p.parent[c];
    const size_t e = (size_t)(c - 1) * H + h;
    const double u = 1.0 / p.nchild[par];
    const double a0 = d == 1 ? p.b0 : p.val[(size_t)par * H + h], a1 = d == 1 ? p.b0 : p.reach[(size_t)par * H + h];
    p.Sg[e] = u;
    if (p.R) p.R[e] = 0.0;
    p.S[e] = u * (actor == 0 ? a0 : a1);
    p.val[(size_t)c * H + h] = actor == 0 ? a0 * u : a0;
    p.reach[(size_t)c * H + h] = actor == 1 ? a1 * u : a1;
  }
}

// FP forward: the opponent's reach under the average strategy, level d's nodes [nb, ne) from their parents (cfr_forward).
__global__ void fg_reach_kernel(FullGameDev p, int nb, int ne, int d) {
  const int H = p.H, actor = (d - 1) & 1, opp = 1 - (*p.iter & 1);
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int c = nb + (int)(it / H), h = (int)(it % H);
    const double a = d == 1 ? p.b0 : p.reach[(size_t)p.parent[c] * H + h];
    p.reach[(size_t)c * H + h] = actor == opp ? a * p.Sg[(size_t)(c - 1) * H + h] : a;
  }
}

// Terminal payoffs of the traverser (cfr_forward's two passes fused: one thread per terminal builds the 9-bin match-count
// histogram of the opponent's reach in hand order, its suffix sums and the belief sum, then the payoff of every hand).
__global__ void fg_terminal_kernel(FullGameDev p) {
  constexpr int kMaxBins = 9;            // match counts 0 .. 8; bin 8 stays empty for num_dice <= kMaxDice = 7 (cfr_types.h)
  static_assert(kMaxBins >= kMaxDice + 2, "a clamped `left` must land on an empty bin");
  const int H = p.H, T = p.T, trav = *p.iter & 1;
  for (int z = blockIdx.x * blockDim.x + threadIdx.x; z < T; z += fg_threads()) {
    const int n = p.term_node[z], pbid = p.term_node[T + z], ndepth = p.term_node[2 * T + z];
    const int face = pbid % p.F;
    const double* ro = p.reach + (size_t)n * H;
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
    const int quantity = 1 + pbid / p.F;
    double* out = p.val + (size_t)n * H;
    for (int h = 0; h < H; ++h) {
      int left = quantity - (int)p.matches[h * p.F + face];
      left = left < 0 ? 0 : (left > kMaxBins - 1 ? kMaxBins - 1 : left);
      const double win = cnt[left];
      const double v = (double)(float)win * 2 - tot;
      out[h] = ((ndepth & 1) != trav) ? -v : v;   // the bidder (player ndepth & 1) wins v
    }
  }
}

// Bottom-up values of level d's nodes [nb, ne) from their children (cfr_backward / fp_backward).  CFR: at the traverser's nodes
// the value is sum_j value(child j) x sigma(j), and the children's slots take the new regrets R + value(child) - value(node).  FP:
// at the traverser's nodes the best child (first wins ties), flagged 1 / 0 in the reach table.  Elsewhere the plain sum.
__global__ void fg_up_kernel(FullGameDev p, int nb, int ne, int d) {
  const int H = p.H;
  const bool mine = (d & 1) == (*p.iter & 1);
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int n = nb + (int)(it / H), h = (int)(it % H);
    const int nc = p.nchild[n];
    if (!nc) continue;
    const int c0 = p.child_begin[n];
    double* __restrict__ vc = p.val + (size_t)c0 * H + h;     // child j at vc[j * H]
    double v = 0;
    if (!mine) {
      for (int j = 0; j < nc; ++j) v += vc[(size_t)j * H];
    } else if (p.fp) {
      int best = 0;
      v = vc[0];
      for (int j = 1; j < nc; ++j) {
        const double nv = vc[(size_t)j * H];
        if (nv > v) { v = nv; best = j; }
      }
      double* fl = p.reach + (size_t)c0 * H + h;
      for (int j = 0; j < nc; ++j) fl[(size_t)j * H] = (j == best) ? 1.0 : 0.0;
    } else {
      const double* sg = p.Sg + (size_t)(c0 - 1) * H + h;
      for (int j = 0; j < nc; ++j) v += vc[(size_t)j * H] * sg[(size_t)j * H];
      const double* r = p.R + (size_t)(c0 - 1) * H + h;
      for (int j = 0; j < nc; ++j) vc[(size_t)j * H] = (r[(size_t)j * H] + vc[(size_t)j * H]) - v;
    }
    p.val[(size_t)n * H + h] = v;
  }
}

// Top-down pass over level d's nodes [nb, ne) and their children.  CFR (cfr_backward): regret matching at the traverser's nodes,
// discounted regrets, the sum-strategy update and the traverser's reach under the new strategy.  FP (fp_backward): beliefs x best
// response into the sums, the linear discount and the new average strategy; val carries the traverser's beliefs.
__global__ void fg_down_kernel(FullGameDev p, int nb, int ne, int d) {
  const int H = p.H, iter = *p.iter, trav = iter & 1, s = iter >> 1;   // s: the traverser's earlier updates (steps[trav])
  const bool mine = (d & 1) == trav;
  constexpr double eps = 1e-80;
  double pos = 1, neg = 1, strat = 1;
  {
    const double ns = (double)(s + 1);
    if (p.linear) {
      pos = neg = strat = ns / (ns + 1);
    } else if (p.dcfr) {
      pos = p.dcfr_alpha >= 5 ? 1.0 : pow(ns, p.dcfr_alpha) / (pow(ns, p.dcfr_alpha) + 1);
      neg = p.dcfr_beta <= -5 ? 0.0 : pow(ns, p.dcfr_beta) / (pow(ns, p.dcfr_beta) + 1);
      strat = pow(ns / (ns + 1), p.dcfr_gamma);
    }
  }
  const double disc = (double)(s + 2) / (s + 3);
  double* __restrict__ row = p.fp ? p.val : p.reach;     // CFR: the traverser's reach; FP: its beliefs
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int n = nb + (int)(it / H), h = (int)(it % H);
    const int nc = p.nchild[n];
    if (!nc) continue;
    const int c0 = p.child_begin[n];
    const double rn = d == 0 ? p.b0 : row[(size_t)n * H + h];
    double* __restrict__ rc = row + (size_t)c0 * H + h;          // child j at rc[j * H]
    const size_t e0 = (size_t)(c0 - 1) * H + h;
    if (!mine) {
      for (int j = 0; j < nc; ++j) rc[(size_t)j * H] = rn;
    } else if (!p.fp) {
      const double* vc = p.val + (size_t)c0 * H + h;               // the new regrets of fg_up_kernel
      double sum = 0;
      for (int j = 0; j < nc; ++j) {
        const double r = vc[(size_t)j * H];
        sum += r > eps ? r : eps;
      }
      for (int j = 0; j < nc; ++j) {
        const size_t e = e0 + (size_t)j * H;
        const double r = vc[(size_t)j * H];
        const double sg = (r > eps ? r : eps) / sum;
        p.Sg[e] = sg;
        p.R[e] = r * (r > 0 ? pos : neg);
        p.S[e] = p.S[e] * strat + rn * sg;
        rc[(size_t)j * H] = rn * sg;
      }
    } else {
      const double* fl = p.reach + (size_t)c0 * H + h;             // best-response flags of fg_up_kernel
      double tot = 0, tl = 0;
      for (int j = 0; j < nc; ++j) {
        const size_t e = e0 + (size_t)j * H;
        const double x = rn * fl[(size_t)j * H];
        double sn = p.S[e] + x;
        if (p.linear) sn = sn * disc;
        p.S[e] = sn;
        rc[(size_t)j * H] = x;
        tot += sn;
        tl += x;
      }
      if (p.optimistic) tot = tot + tl;
      for (int j = 0; j < nc; ++j) {
        const size_t e = e0 + (size_t)j * H;
        p.Sg[e] = (p.optimistic ? p.S[e] + rc[(size_t)j * H] : p.S[e]) / tot;
      }
    }
  }
}

__global__ void fg_advance_kernel(int* iter) { ++*iter; }

// The average strategy (ISubgameSolver::get_strategy) into avg: CFR's normalised sum (avg_row).  FP's is Sg itself (copied by the
// host).
__global__ void fg_average_kernel(FullGameDev p, const int* depth, int untouched0, int untouched1) {
  const int H = p.H;
  const long long items = (long long)p.N * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int n = (int)(it / H), h = (int)(it % H);
    const int nc = p.nchild[n];
    if (!nc) continue;
    const bool untouched = (depth[n] & 1) ? untouched1 : untouched0;
    const size_t e0 = (size_t)(p.child_begin[n] - 1) * H + h;
    avg_row(p.avg + e0, p.S + e0, 0, 0, H, nc, true, untouched);
  }
}

}  // namespace cfrb
