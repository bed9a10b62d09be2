// Recursive to-leaf walk on the device (cfrb_to_leaf_exploitability): compute_strategy_recursive_to_leaf with the average strategy
// (recursive_solving.cc:76-134, as RecursiveEvaluator::strategyToLeaf runs it on the host) for games whose full tree is too large
// for a dense [N][H][A] strategy.  Level l holds the subgames rooted at the non-terminal full-tree nodes of depth l * max_depth, in
// full-tree node order; each wave of a level is solved by the handle's CFR / FP solver, then
//
//   expl_begin    per subgame: template, player and (real) root beliefs of the wave, from the level's roots and fp64 beliefs
//   sp_scan       packed value-net row offsets, wave size, largest-first schedule (selfplay_kernels.cuh)
//   expl_expand   per subgame: the average strategy of its inner nodes (get_strategy; CFR's sum normalised as cfrb_fetch_compact
//                 kind 4 does it) written straight into the compact full-tree strategy, and the beliefs of its non-terminal
//                 pseudo-leaves -- propagated unnormalised with the acting player's strategy, then eps-normalised row by row
//                 (normalize_beliefs_inplace) -- appended to the next level at fill + row offset + leaf slot
//   expl_fill     fill += the wave's pseudo-leaf rows
//
// The row offsets are an exclusive prefix sum over the wave in level order and a template lists its pseudo-leaves in BFS order, so
// the next level comes out in full-tree node order without atomics.  Every fp64 operation is the host walk's, in its order (this
// header is compiled into the -fmad=false translation unit): the strategy and the beliefs are bit-identical to the host's.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"
#include "selfplay_kernels.cuh"

namespace cfrb {

template <typename real>
__global__ void __launch_bounds__(128) expl_begin_kernel(ExplDev p, int n, real* __restrict__ wave_beliefs) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int node = p.roots[p.off + k];
  p.sg_tmpl[k] = p.full_act_lo[node];          // = last_bid + 1 (0 at the game root)
  p.sg_player[k] = p.full_depth[node] & 1;     // the game root is player 0's node
  p.sg_act[k] = -1;
  const double* b = p.bel + (size_t)(p.off + k) * 2 * p.H;
  for (int i = 0; i < 2 * p.H; ++i) wave_beliefs[(size_t)k * 2 * p.H + i] = (real)b[i];
}

// One CTA per subgame of the wave.  table: the solver's average-strategy table (CFR: the sum S, normalised here; FP: Sg).
template <typename real>
__global__ void __launch_bounds__(128) expl_expand_kernel(ExplDev p, const real* __restrict__ table, int normalise) {
  const int k = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, H = p.H;
  const TemplateDev t = p.tmpl[p.sg_tmpl[k]];
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  const int* __restrict__ level_begin = p.level_begin + t.level_off;
  int* fid = p.fid + (size_t)k * p.nmax;
  // full-tree node of every template node: child j of n is child j of n's full-tree node (same bid range, same order)
  if (tid == 0) fid[0] = p.roots[p.off + k];
  __syncthreads();
  for (int d = 1; d < t.levels; ++d) {
    for (int c = level_begin[d] + tid; c < level_begin[d + 1]; c += nt) {
      const int q = parent[c];
      fid[c] = p.full_child_begin[fid[q]] + (c - child_begin[q]);
    }
    __syncthreads();
  }
  // the average strategy of the inner nodes (normalise_avg in cfrb_api.cu: uniform until the acting player's first update)
  const real* tk = table + (size_t)k * p.table_stride;
  for (int it = tid; it < t.N * H; it += nt) {
    const int nn = it / H, hd = it % H;
    const int nc = nchild[nn];
    if (!nc) continue;
    const int cb = child_begin[nn], f = fid[nn];
    double* out = p.strategy + (size_t)(p.full_child_begin[f] - 1) * H + hd;
    if (normalise) {
      const bool untouched = p.steps[2 * k + (p.full_depth[f] & 1)] == 0;
      double sum = 0;
      for (int j = 0; j < nc; ++j) sum += (double)tk[(size_t)(cb + j - 1) * H + hd];
      for (int j = 0; j < nc; ++j) {
        const double v = (double)tk[(size_t)(cb + j - 1) * H + hd];
        out[(size_t)j * H] = (sum > 0 && !untouched) ? v / sum : 1.0 / nc;
      }
    } else {
      for (int j = 0; j < nc; ++j) out[(size_t)j * H] = (double)tk[(size_t)(cb + j - 1) * H + hd];
    }
  }
  __syncthreads();
  // beliefs of the pseudo-leaves, one thread per (leaf, player row): the root row times the strategy of every edge on the path
  // that the row's player acts on, from the root down, then eps-normalised
  const int base = *p.fill + p.sg_row_off[k];
  const double* rb = p.bel + (size_t)(p.off + k) * 2 * H;
  const int D = t.levels - 1;                  // pseudo-leaves sit at the template's last level
  for (int it = tid; it < 2 * t.L; it += nt) {
    const int r = it >> 1, pl = it & 1;
    const int leaf = p.pleaf_node[t.pleaf_off + r];
    const int slot = base + r;
    if (slot >= p.cap) continue;               // cannot happen for a level sized by the host; the host checks the count
    if (pl == 0) p.next_roots[slot] = fid[leaf];
    double* ob = p.next_bel + (size_t)slot * 2 * H + (size_t)pl * H;
    for (int h = 0; h < H; ++h) ob[h] = rb[pl * H + h];
    for (int d = 1; d <= D; ++d) {
      int c = leaf;                            // the leaf's ancestor at depth d, and its parent
      for (int up = D; up > d; --up) c = parent[c];
      const int q = parent[c];
      if ((p.full_depth[fid[q]] & 1) != pl) continue;
      const double* s = p.strategy + (size_t)(fid[c] - 1) * H;
      for (int h = 0; h < H; ++h) ob[h] *= s[h];
    }
    double sum = 0;
    for (int h = 0; h < H; ++h) sum += ob[h] + 1e-80;
    for (int h = 0; h < H; ++h) ob[h] = (ob[h] + 1e-80) / sum;
  }
}

__global__ void expl_fill_kernel(ExplDev p) { *p.fill += p.wave[1]; }

}  // namespace cfrb
