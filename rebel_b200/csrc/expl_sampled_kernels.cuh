// Sampled recursive to-leaf walk on the device (cfrb_to_leaf_sampled): recursive_eval's --num_repeats evaluation
// (recursive_eval.cc:331-369: compute_sampled_strategy_recursive_to_leaf, recursive_solving.cc:301-327 with :76-134, and the
// float32 reach-weighted sums of :138-148, 349-355, as RecursiveEvaluator::run does it on the host) for games whose full tree is
// too large for dense [N][H][A] sums.  A batch of b repeats is walked level by level like expl_kernels.cuh walks the average
// policy; a level holds, for each subgame root in full-tree node order, its b repeats next to each other in repeat order.  Each
// wave (whole root groups) is solved by the handle's CFR / FP solver up to the largest act_iteration of the wave, then
//
//   expl_sampled_begin    per subgame: template, player, act_iteration (the repeat's mt19937 draw for that root) and root beliefs
//   sp_scan               packed value-net row offsets, wave size, largest-first schedule (selfplay_kernels.cuh)
//   expl_sampled_expand   one CTA per root group, its repeats in order: summed_reach[node] += float(reach[player(node)]) at every
//                         node of the subgame but its non-terminal pseudo-leaves, summed_strategy[edge] += float(s) * float(reach)
//                         at every inner edge, s the repeat's snapshot strategy (the sampling strategy at act_iteration); then the
//                         fp64 beliefs (unnormalised down the subgame, eps-normalised at the leaf) and reach (never normalised) of
//                         its non-terminal pseudo-leaves, appended to the next level at fill + group row offset + leaf * b + repeat
//   expl_fill             fill += the wave's pseudo-leaf rows
//
// Every (node, hand) entry of the accumulators gets one contribution per repeat, and a root's repeats are added by one CTA in
// repeat order, batches in order: the float32 sums are the host's bit for bit.  Every fp64 operation is the host walk's, in its
// order (this header is compiled into the -fmad=false translation unit).  At a checkpoint expl_sampled_finalize divides the sums
// in float32 (recursive_eval.cc:362-363) and widens the result into the compact strategy the best response (br_kernel) reads.
#pragma once
#include <cuda_runtime.h>

#include "cfr_types.h"
#include "selfplay_kernels.cuh"

namespace cfrb {

template <typename real>
__global__ void __launch_bounds__(128) expl_sampled_begin_kernel(ExplSampledDev p, int n, real* __restrict__ wave_beliefs) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int pos = p.off + k;
  const int node = p.roots[pos];
  p.sg_tmpl[k] = p.full_act_lo[node];          // = last_bid + 1 (0 at the game root)
  p.sg_player[k] = p.full_depth[node] & 1;     // the game root is player 0's node
  p.sg_act[k] = p.draws[(long long)(pos % p.b) * p.draws_stride + p.level_base + pos / p.b];
  const double* b = p.bel + (size_t)pos * 2 * p.H;
  for (int i = 0; i < 2 * p.H; ++i) wave_beliefs[(size_t)k * 2 * p.H + i] = (real)b[i];
}

// v and w times the snapshot strategy of every edge on the path from the root to template node nn whose parent player pl acts
// on, from the root down (the host's copy-then-multiply per child, recursive_eval.h expand)
template <typename real>
__device__ __forceinline__ void sampled_path(const ExplSampledDev& p, const int* __restrict__ parent, const int* __restrict__ fid,
                                             const real* __restrict__ tk, int nn, int h, int pl, double& v, double& w) {
  int dep = 0;
  for (int c = nn; parent[c] >= 0; c = parent[c]) ++dep;
  for (int d = 1; d <= dep; ++d) {
    int c = nn;                                // nn's ancestor at depth d, and its parent
    for (int up = dep; up > d; --up) c = parent[c];
    const int q = parent[c];
    if ((p.full_depth[fid[q]] & 1) == pl) {
      const double s = (double)tk[(size_t)(c - 1) * p.H + h];
      v *= s;
      w *= s;
    }
  }
}

// One CTA per root group of the wave: subgames g * b .. g * b + b - 1, the b repeats of one root.  snap: the solver's snapshot
// table (the sampling strategy at each subgame's act_iteration).
template <typename real>
__global__ void __launch_bounds__(128) expl_sampled_expand_kernel(ExplSampledDev p, const real* __restrict__ snap) {
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, H = p.H, k0 = g * p.b;
  const TemplateDev t = p.tmpl[p.sg_tmpl[k0]];
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  const int* __restrict__ level_begin = p.level_begin + t.level_off;
  int* fid = p.fid + (size_t)g * p.nmax;
  // full-tree node of every template node: child j of n is child j of n's full-tree node (same bid range, same order)
  if (tid == 0) fid[0] = p.roots[p.off + k0];
  __syncthreads();
  for (int d = 1; d < t.levels; ++d) {
    for (int c = level_begin[d] + tid; c < level_begin[d + 1]; c += nt) {
      const int q = parent[c];
      fid[c] = p.full_child_begin[fid[q]] + (c - child_begin[q]);
    }
    __syncthreads();
  }
  const int base = *p.fill + p.sg_row_off[k0];
  for (int j = 0; j < p.b; ++j) {
    const int k = k0 + j;
    const real* tk = snap + (size_t)k * p.table_stride;
    const double* rb = p.bel + (size_t)(p.off + k) * 2 * H;
    const double* rr = p.rch + (size_t)(p.off + k) * 2 * H;
    // the weights of the infosets (node, hand) (recursive_eval.cc:143-148) and the weighted sampled strategy (:349-355)
    for (int it = tid; it < t.N * H; it += nt) {
      const int nn = it / H, hd = it % H;
      const int f = fid[nn], nc = nchild[nn];
      if (nc == 0 && p.full_act_lo[f] < p.A) continue;   // non-terminal pseudo-leaf: the next level's subgame root
      const int pid = p.full_depth[f] & 1;
      double r = rr[pid * H + hd], unused = 0;
      sampled_path(p, parent, fid, tk, nn, hd, pid, r, unused);
      p.sum_r[(size_t)f * H + hd] += (float)r;
      const int cb = child_begin[nn], fcb = p.full_child_begin[f];
      for (int jj = 0; jj < nc; ++jj) {
        const double s = (double)tk[(size_t)(cb + jj - 1) * H + hd];
        const size_t e = (size_t)(fcb + jj - 1) * H + hd;
        p.sum_s[e] += (float)s * (float)r;
        if (j == p.last_j) p.last[e] = s;
        if (p.rep_s) p.rep_s[(size_t)j * p.rep_stride + e] = (float)s;   // the repeat's strategy as recursive_eval's float32 tensor
      }
    }
    // beliefs and reach of the pseudo-leaves, one thread per (leaf, player row)
    for (int it = tid; it < 2 * t.L; it += nt) {
      const int r = it >> 1, pl = it & 1;
      const int leaf = p.pleaf_node[t.pleaf_off + r];
      const long long slot = (long long)base + (long long)r * p.b + j;
      if (slot >= p.cap) continue;             // cannot happen for a level sized by the host; the host checks the count
      if (pl == 0) p.next_roots[slot] = fid[leaf];
      double* ob = p.next_bel + (size_t)slot * 2 * H + (size_t)pl * H;
      double* orch = p.next_rch + (size_t)slot * 2 * H + (size_t)pl * H;
      for (int h = 0; h < H; ++h) {
        double vb = rb[pl * H + h], vr = rr[pl * H + h];
        sampled_path(p, parent, fid, tk, leaf, h, pl, vb, vr);
        ob[h] = vb;
        orch[h] = vr;
      }
      double sum = 0;
      for (int h = 0; h < H; ++h) sum += ob[h] + 1e-80;
      for (int h = 0; h < H; ++h) ob[h] = (ob[h] + 1e-80) / sum;
    }
    __syncthreads();                           // repeat j + 1 adds to the entries repeat j has just added to
  }
}

__global__ void expl_sampled_fill_kernel(ExplSampledDev p) { *p.fill += p.wave[1]; }

__global__ void expl_sampled_finalize_kernel(ExplSampledDev p) {
  const size_t total = (size_t)(p.full_nodes - 1) * p.H;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / p.H) + 1, hd = (int)(i % p.H);
    const float den = p.sum_r[(size_t)p.full_parent[c] * p.H + hd] + 1e-6f;
    p.strategy[i] = (double)(p.sum_s[i] / den);
  }
}

}  // namespace cfrb
