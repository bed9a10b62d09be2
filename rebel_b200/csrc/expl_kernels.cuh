// Recursive to-leaf walk on the device (cfrb_to_leaf_exploitability): compute_strategy_recursive_to_leaf with the average strategy
// (recursive_solving.cc:76-134, as RecursiveEvaluator::strategyToLeaf runs it on the host) for games whose full tree is too large
// for a dense [N][H][A] strategy.  Level l holds the subgames rooted at the non-terminal full-tree nodes of depth l * max_depth, in
// full-tree node order; each wave of a level is solved by the handle's CFR / FP solver (LevelWalk in cfrb_api.cu), then
//
//   expl_begin    per subgame: template, player, act_iteration (the sampled walk's draw, else -1) and (real) root beliefs of the
//                 wave, from the level's roots and fp64 beliefs.  The every-node and sampled walks begin their waves with it too
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
  const int pos = p.off + k;
  const int node = p.roots[pos];
  p.sg_tmpl[k] = p.full_act_lo[node];          // = last_bid + 1 (0 at the game root)
  p.sg_player[k] = p.full_depth[node] & 1;     // the game root is player 0's node
  p.sg_act[k] = p.draws ? p.draws[(long long)(pos % p.b) * p.draws_stride + p.level_base + pos / p.b] : -1;
  const double* b = p.bel + (size_t)pos * 2 * p.H;
  for (int i = 0; i < 2 * p.H; ++i) wave_beliefs[(size_t)k * 2 * p.H + i] = (real)b[i];
}

// The full-tree node of every template node of the subgame at level position pos, by the whole CTA: child j of n is child j of n's
// full-tree node (same bid range, same order).
__device__ __forceinline__ void template_fid(const ExplDev& p, const TemplateDev& t, int pos, int* fid) {
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ level_begin = p.level_begin + t.level_off;
  if (threadIdx.x == 0) fid[0] = p.roots[pos];
  __syncthreads();
  for (int d = 1; d < t.levels; ++d) {
    for (int c = level_begin[d] + threadIdx.x; c < level_begin[d + 1]; c += blockDim.x) {
      const int q = parent[c];
      fid[c] = p.full_child_begin[fid[q]] + (c - child_begin[q]);
    }
    __syncthreads();
  }
}

// One CTA per subgame of the wave.  table: the solver's average-strategy table (CFR: the sum S, normalised here; FP: Sg).
template <typename real>
__global__ void __launch_bounds__(128) expl_expand_kernel(ExplDev p, const real* __restrict__ table, int normalise) {
  const int k = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, H = p.H;
  const TemplateDev t = p.tmpl[p.sg_tmpl[k]];
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  int* fid = p.fid + (size_t)k * p.nmax;
  template_fid(p, t, p.off + k, fid);
  // the average strategy of the inner nodes (avg_row)
  const real* tk = table + (size_t)k * p.table_stride;
  for (int it = tid; it < t.N * H; it += nt) {
    const int nn = it / H, hd = it % H;
    const int nc = nchild[nn];
    if (!nc) continue;
    const int cb = child_begin[nn], f = fid[nn];
    avg_row(p.strategy + (size_t)(p.full_child_begin[f] - 1) * H + hd, tk, cb - 1, hd, H, nc, normalise != 0,
            normalise && p.steps[2 * k + (p.full_depth[f] & 1)] == 0);
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
    sp_normalize(ob, H);
  }
}

__global__ void expl_fill_kernel(ExplDev p) { *p.fill += p.wave[1]; }

// Every-node walk (cfrb_recursive_exploitability): compute_strategy_recursive (recursive_solving.cc:46-74, as
// RecursiveEvaluator::strategyRecursive runs it on the host).  Level d holds the non-terminal full-tree nodes of depth d, in full-tree
// order; each roots a depth-max_depth subgame, solved by expl_begin / sp_scan / the handle's solver like a to-leaf wave, of whose
// average strategy only the root row is kept.  One warp per subgame of the wave:
//   - the root row (avg_row: CFR's sum normalised, FP's Sg as it is) goes to the root's edges of the compact full-tree strategy;
//   - every non-terminal child goes to the next level with the root's beliefs, the acting player's row multiplied by the child's
//     strategy and eps-normalised (normalize_beliefs_inplace), the other row unchanged.  Only the acting row is renormalised, unlike
//     the to-leaf walk's pseudo-leaves.
// Every node below the game root has the liar call, which is terminal, as its last child, and the root has no call.  So a depth-d
// node at level position i follows i call children in the full tree's depth d + 1, and its child c takes next-level slot
// c - level_begin[d + 1] - i (at the root i = 0 and level_begin[1] = 1): the next level comes out in full-tree order without atomics.
// fill only counts the children written, for the host's check of the level's size.
template <typename real>
__global__ void __launch_bounds__(128) rec_expand_kernel(ExplDev p, int n, const real* __restrict__ table, int normalise) {
  const int k = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31, H = p.H;
  if (k >= n) return;                          // whole warps
  const int i = p.off + k, node = p.roots[i];
  const int nc = p.full_nchild[node], cb = p.full_child_begin[node], pl = p.full_depth[node] & 1;
  const real* tk = table + (size_t)k * p.table_stride;   // the template root's edges are its first nc rows
  double* s = p.strategy + (size_t)(cb - 1) * H;
  for (int h = lane; h < H; h += 32) avg_row(s + h, tk, 0, h, H, nc, normalise != 0, normalise && p.steps[2 * k + pl] == 0);
  __syncwarp();
  const int kids = node == 0 ? nc : nc - 1;
  const int first = p.full_level_begin[p.full_depth[node] + 1] + i;
  const double* rb = p.bel + (size_t)i * 2 * H;
  for (int j = lane; j < kids; j += 32) {
    const int slot = cb + j - first;
    if (slot < 0 || slot >= p.cap) continue;   // cannot happen for a level sized by the host; the host checks the count
    p.next_roots[slot] = cb + j;
    double* ob = p.next_bel + (size_t)slot * 2 * H;
    for (int x = 0; x < 2 * H; ++x) ob[x] = rb[x];
    double* a = ob + (size_t)pl * H;
    const double* sj = s + (size_t)j * H;
    for (int h = 0; h < H; ++h) a[h] *= sj[h];
    sp_normalize(a, H);
  }
  if (lane == 0) atomicAdd(p.fill, kids);
}

// Sampled recursive to-leaf walk on the device (cfrb_to_leaf_sampled): recursive_eval's --num_repeats evaluation
// (recursive_eval.cc:331-369: compute_sampled_strategy_recursive_to_leaf, recursive_solving.cc:301-327 with :76-134, and the
// float32 reach-weighted sums of :138-148, 349-355, as RecursiveEvaluator::run does it on the host) for games whose full tree is
// too large for dense [N][H][A] sums.  A batch of b repeats is walked level by level like the average policy; a level holds, for
// each subgame root in full-tree node order, its b repeats next to each other in repeat order.  Each wave (whole root groups) is
// begun by expl_begin, whose act_iteration is the repeat's mt19937 draw for that root, solved by the handle's CFR / FP solver up to
// the largest act_iteration of the wave, and ended by expl_fill after
//
//   expl_sampled_expand   one CTA per root group, its repeats in order: summed_reach[node] += float(reach[player(node)]) at every
//                         node of the subgame but its non-terminal pseudo-leaves, summed_strategy[edge] += float(s) * float(reach)
//                         at every inner edge, s the repeat's snapshot strategy (the sampling strategy at act_iteration); then the
//                         fp64 beliefs (unnormalised down the subgame, eps-normalised at the leaf) and reach (never normalised) of
//                         its non-terminal pseudo-leaves, appended to the next level at fill + group row offset + leaf * b + repeat
//
// Every (node, hand) entry of the accumulators gets one contribution per repeat, and a root's repeats are added by one CTA in
// repeat order, batches in order: the float32 sums are the host's bit for bit.  Every fp64 operation is the host walk's, in its
// order.  At a checkpoint expl_sampled_finalize divides the sums in float32 (recursive_eval.cc:362-363) and widens the result into
// the compact strategy the best response (br_kernel) reads.

// v and w times the snapshot strategy of every edge on the path from the root to template node nn whose parent player pl acts
// on, from the root down (the host's copy-then-multiply per child, recursive_eval.h expand)
template <typename real>
__device__ __forceinline__ void sampled_path(const ExplDev& p, const int* __restrict__ parent, const int* __restrict__ fid,
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
__global__ void __launch_bounds__(128) expl_sampled_expand_kernel(ExplDev p, const real* __restrict__ snap) {
  const int g = blockIdx.x, tid = threadIdx.x, nt = blockDim.x, H = p.H, k0 = g * p.b;
  const TemplateDev t = p.tmpl[p.sg_tmpl[k0]];
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  int* fid = p.fid + (size_t)g * p.nmax;
  template_fid(p, t, p.off + k0, fid);
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
      sp_normalize(ob, H);
    }
    __syncthreads();                           // repeat j + 1 adds to the entries repeat j has just added to
  }
}

__global__ void expl_sampled_finalize_kernel(ExplDev p) {
  const size_t total = (size_t)(p.full_nodes - 1) * p.H;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(i / p.H) + 1, hd = (int)(i % p.H);
    const float den = p.sum_r[(size_t)p.full_parent[c] * p.H + hd] + 1e-6f;
    p.strategy[i] = (double)(p.sum_s[i] / den);
  }
}

}  // namespace cfrb
