// FP subtree forest (cfrb_fp_forest_*): linear fictitious play, without a value net, on every full-tree subtree rooted at the
// nodes of one depth d0, each root with its own beliefs [2][H] -- eval_net's full-depth solves (stats.cc:118-124) of one depth at
// once.  The subtrees below the nodes of one level are disjoint, so this is the full-game solver's level-synchronous FP
// (full_game_kernels.cuh) started at level d0 instead of level 0: fg_reach / fg_terminal / fg_up / fg_down run unchanged on levels
// d0 .. A, and the three kernels here stand in for the root of a one-subgame wave (cfr_init_kernel's root rows, cfr_forward's
// root reach, fp_backward's root value running mean and root beliefs).  Every node of level d0 is a root; the host gives the nodes
// it was not asked about uniform beliefs, so their subtrees stay finite and, being disjoint, feed nothing into the others.
//
// Bit-identical to a wave subgame rooted at the same node (FP, linear, max_depth 10000): the acting player of an absolute depth d
// is d & 1, which is the wave's root player ^ (subgame depth & 1); traversers alternate from iteration 0 in both; every (node,
// hand) entry runs the wave's fp64 operations in its order, compiled in the -fmad=false unit.
//
// The root beliefs bel and the running means mu are [level node - nb][2][H].  Tables as FullGameDev: FP keeps player 0's reach in
// val and player 1's in reach during the constructor, the opponent's reach in reach during the forward pass, the best-response
// flags in reach and the traverser's beliefs in val during the top-down pass.
//
// Reach statistics of a compact strategy (cfrb_fp_forest_reach): rg_reach_kernel (regret_grid_kernels.cuh) forms both players'
// reach from the root's 1 / H, and ff_gather_kernel reads the listed nodes' node_reach and rows out of it, as strategy_reach does.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"
#include "full_game_kernels.cuh"

namespace cfrb {

// FP constructor rows of level d0's nodes [nb, ne) (cfr_init_kernel: reach0 = b[0], reach1 = b[1] at the root), zero means; fg_init
// then builds levels d0 + 1 .. A from them.
__global__ void ff_root_init_kernel(FullGameDev p, const double* __restrict__ bel, double* __restrict__ mu, int nb, int ne) {
  const int H = p.H;
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int r = (int)(it / H), h = (int)(it % H);
    const size_t n = (size_t)(nb + r) * H + h, b = (size_t)r * 2 * H + h;
    p.val[n] = bel[b];
    p.reach[n] = bel[b + H];
    mu[b] = 0;
    mu[b + H] = 0;
  }
}

// Forward half: the opponent's reach at the roots is its belief (cfr_forward, reach_opp[root] = b[opp]).
__global__ void ff_root_reach_kernel(FullGameDev p, const double* __restrict__ bel, int nb, int ne) {
  const int H = p.H, opp = 1 - (*p.iter & 1);
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int r = (int)(it / H), h = (int)(it % H);
    p.reach[(size_t)(nb + r) * H + h] = bel[((size_t)r * 2 + opp) * H + h];
  }
}

// Between the bottom-up and the top-down pass (fp_backward): the root value running mean with num_update = steps[trav] + 1, then
// the traverser's beliefs into the root's value slot, where fg_down_kernel reads the beliefs of level d0.
__global__ void ff_root_mean_kernel(FullGameDev p, const double* __restrict__ bel, double* __restrict__ mu, int nb, int ne) {
  const int H = p.H, iter = *p.iter, trav = iter & 1, s = iter >> 1;
  const double alpha = p.linear ? (double)2 / (s + 2) : (double)1 / (s + 1);
  const long long items = (long long)(ne - nb) * H;
  for (long long it = blockIdx.x * (long long)blockDim.x + threadIdx.x; it < items; it += fg_threads()) {
    const int r = (int)(it / H), h = (int)(it % H);
    const size_t n = (size_t)(nb + r) * H + h, b = ((size_t)r * 2 + trav) * H + h;
    mu[b] += (p.val[n] - mu[b]) * alpha;
    p.val[n] = bel[b];
  }
}

// node_reach[i] = (sum_h reach0) * (sum_h reach1) of node nodes[i], each sum in hand order, and its rows [i][2][H]; the root's rows
// are 1 / H (rg_reach_kernel does not store them).
__global__ void ff_gather_kernel(RegretGridDev p, const int* __restrict__ nodes, int n, double* __restrict__ node_reach,
                                 double* __restrict__ rows) {
  const int H = p.H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int v = nodes[i];
    double s0 = 0, s1 = 0;
    for (int h = 0; h < H; ++h) {
      const double r0 = v == 0 ? 1. / H : p.reach0[(size_t)v * H + h], r1 = v == 0 ? 1. / H : p.reach1[(size_t)v * H + h];
      s0 += r0;
      s1 += r1;
      rows[(size_t)i * 2 * H + h] = r0;
      rows[(size_t)i * 2 * H + H + h] = r1;
    }
    node_reach[i] = s0 * s1;
  }
}

}  // namespace cfrb
