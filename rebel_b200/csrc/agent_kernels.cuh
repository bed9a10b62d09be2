// A ReBeL agent driven from outside (cfrb_agent_*): T independent tables, each a game between the agent (one handle) and an
// external player (a person, another program's policy, a tournament harness), advanced one action per call.
//
// The agent plays as in a head-to-head match (match_kernels.cuh): the reference's recursive to-leaf strategy restricted to the
// path played.  At the game root and at every pseudo-leaf of its previous subgame it solves the subgame rooted at the current
// public node from its own beliefs, acts there with the subgame's strategy for its hand, and updates both players' beliefs with
// its own strategy: unnormalised inside the subgame, eps-normalised at its leaves.  Unlike a match, the tables of one call stand
// at different points of their subgames and the wave positions of a call's solves change from call to call, so the handle's
// tables cannot be read in place later: right after every solve agent_capture copies each solved subgame's acting strategy into
// a per-table fp64 cache, and every later step reads only the cache.
//
//   agent_new       per listed table: seat, hand, uniform beliefs, the table's mt19937 stream keyed by (seed, key)
//   agent_scan      one CTA: wave index of every listed table that stands at an unsolved root and the packed value-net row offsets
//   agent_begin     per listed table that needs a solve: subgame descriptor (template, player, fp64 -> real beliefs) and, in
//                   sampled mode, act_iteration ~ weight i/2 + 1 on even i < num_iters drawn from the table's stream
//   agent_capture   warp per solved table: the acting strategy into the cache (capture_levels), entry (child - 1) * H + hand;
//                   average mode = avg_row of S (CFR) or Sg (FP); sampled mode = the act_iteration snapshot
//   agent_step      per listed table: one action (given, or drawn for the agent's hand), the mover's belief row times the
//                   strategy of that action, the next node; at a pseudo-leaf both rows eps-normalised and the table unsolved
//   agent_policy    per (listed table, hand): the strategy of the player to move at the table's node
//
// An every-node agent (CFRB_MATCH_EVERY_NODE, compute_strategy_recursive) has an unsolved subgame root at every node: it caches the
// root row only, and after every action eps-normalises the mover's row and stands at an unsolved root again.
//
// A blueprint agent (cfrb_agent_create_blueprint) never solves: `cache` is the blueprint's full-tree table (stride 0), `node` a
// full-tree node (bp_child_begin non-null), and no node is a pseudo-leaf, so step and policy read the table at every node.
//
// This header is compiled into the -fmad=false translation unit: the belief arithmetic is the match walk's, bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cfr_types.h"
#include "match_kernels.cuh"
#include "selfplay_kernels.cuh"

namespace cfrb {

constexpr uint64_t kAgentStreamTag = 3;   // match_stream_seed tags 1 and 2 are the match's deal and game streams

__global__ void __launch_bounds__(128) agent_new_kernel(AgentDev p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int t = p.ids[i], H = p.H;
  mt_seed_strided(p.mt + t, p.T, match_stream_seed(p.seed, p.keys[i], kAgentStreamTag));
  p.mt_idx[t] = 624;
  p.seat[t] = p.io[i]; p.hand[t] = p.hands[i];
  p.last_bid[t] = -1; p.player[t] = 0; p.ply[t] = 0;
  p.root_lb[t] = -1; p.root_player[t] = 0; p.node[t] = 0; p.depth[t] = 0;
  p.act[t] = -1; p.status[t] = 1; p.subgames[t] = 0;
  for (int k = 0; k < 2 * H; ++k) p.root_bel[(size_t)t * 2 * H + k] = p.bel[(size_t)t * 2 * H + k] = 1.0 / H;
}

// Wave index of every listed table at an unsolved root (list order) and the exclusive prefix sum of their pseudo-leaf counts.
__global__ void __launch_bounds__(1024) agent_scan_kernel(AgentDev p) {
  __shared__ int part[2 * 1024];
  const int t = threadIdx.x, per = (p.n + 1023) / 1024;
  const int b = t * per, e = min(p.n, b + per);
  int n = 0, r = 0;
  for (int i = b; i < e; ++i) {
    const int id = p.ids[i];
    if (p.status[id] == 1) { ++n; r += p.tmpl[p.last_bid[id] + 1].L; }
  }
  int x[2] = {n, r};                                 // tables to solve, rows
  sp_block_scan(part, x);
  int w = x[0] - n, off = x[1] - r;
  for (int i = b; i < e; ++i) {
    const int id = p.ids[i];
    if (p.status[id] != 1) { p.widx[i] = -1; continue; }
    p.widx[i] = w;
    p.sg_row_off[w] = off;
    ++w;
    off += p.tmpl[p.last_bid[id] + 1].L;
  }
  if (t == 1023) { p.wave[0] = x[0]; p.wave[1] = x[1]; }
}

template <typename real>
__global__ void __launch_bounds__(128) agent_begin_kernel(AgentDev p, MatchTabs<real> tb) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int w = p.widx[i];
  if (w < 0) return;
  const int t = p.ids[i], H = p.H;
  int act = -1;
  if (p.sampled) {
    SpRng rng{p.mt + t, p.T, p.mt_idx[t]};
    act = sp_act_iteration(rng, p.iters);
    p.mt_idx[t] = rng.idx;
  }
  p.sg_tmpl[w] = p.last_bid[t] + 1;
  p.sg_player[w] = p.player[t];
  p.sg_act[w] = act;
  p.act[t] = act;
  p.root_lb[t] = p.last_bid[t]; p.root_player[t] = p.player[t]; p.node[t] = 0; p.depth[t] = 0;
  p.subgames[t] += 1;
  const double* b = p.root_bel + (size_t)t * 2 * H;
  for (int k = 0; k < 2 * H; ++k) tb.wave_beliefs[0][(size_t)w * 2 * H + k] = (real)b[k];
}

// One warp per listed table.
template <typename real>
__global__ void __launch_bounds__(128) agent_capture_kernel(AgentDev p, MatchTabs<real> tb) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= p.n) return;
  const int w = p.widx[i];
  if (w < 0) return;
  const int t = p.ids[i];
  const TemplateDev tp = p.tmpl[p.root_lb[t] + 1];
  capture_levels(lane, tp, p.child_begin, p.nchild, p.level_begin, p.H, tb.table[0] + (size_t)w * p.table_stride,
                 tb.normalise[0] != 0, p.steps + 2 * w, p.root_player[t], p.every_node ? 1 : tp.levels,   // every-node: the root row only
                 p.cache + (size_t)t * p.stride);
  if (lane == 0) p.status[t] = 2;
}

// The first child and the child count of table t's node: in its subgame template, or in the blueprint's full tree.
__device__ __forceinline__ void agent_node(const AgentDev& p, int t, int& cb, int& nc) {
  const int node = p.node[t];
  if (p.bp_child_begin) {
    const int lb = p.last_bid[t];
    cb = p.bp_child_begin[node]; nc = lb < 0 ? p.A - 1 : p.A - 1 - lb;   // bids lo .. A - 1, no liar call at the game root
    return;
  }
  const TemplateDev tp = p.tmpl[p.root_lb[t] + 1];
  cb = p.child_begin[tp.node_off + node]; nc = p.nchild[tp.node_off + node];
}

__global__ void __launch_bounds__(128) agent_step_kernel(AgentDev p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n) return;
  const int t = p.ids[i], H = p.H, A = p.A;
  const int lb = p.last_bid[t], actor = p.player[t];
  int cb, nc;
  agent_node(p, t, cb, nc);
  const int lo = lb < 0 ? 0 : lb + 1;
  const double* __restrict__ c = p.cache + (size_t)t * p.stride + (size_t)(cb - 1) * H;   // c[j * H + hand]
  const bool mine = actor == p.seat[t];
  const int hand = p.hand[t];
  int a = p.io[i];
  if (a < 0) {
    SpRng rng{p.mt + t, p.T, p.mt_idx[t]};
    a = lo + sp_discrete(rng, nc, [&](int j) { return c[(size_t)j * H + hand]; });
    p.mt_idx[t] = rng.idx;
  }
  const int j = a - lo;
  if (p.probs) {
    double* pr = p.probs + (size_t)i * A;
    for (int k = 0; k < A; ++k)
      pr[k] = !mine ? __longlong_as_double(0x7ff8000000000000ll) : (k >= lo && k < lo + nc) ? c[(size_t)(k - lo) * H + hand] : 0.0;
  }
  double* bel = p.bel + (size_t)t * 2 * H;
  for (int h = 0; h < H; ++h) bel[actor * H + h] *= c[(size_t)j * H + h];
  const int depth = p.depth[t] + 1;
  p.node[t] = cb + j; p.depth[t] = depth;
  p.last_bid[t] = a; p.player[t] = actor ^ 1; p.ply[t] += 1;
  int flags = 0;
  if (a == A - 1) {                                  // liar call: the game is over
    p.status[t] = 0;
    flags = 1;
  } else if (p.every_node) {                         // every node roots the agent's next subgame: the mover's row eps-normalised
    double* root = p.root_bel + (size_t)t * 2 * H;
    sp_normalize(bel + actor * H, H);
    for (int k = 0; k < 2 * H; ++k) root[k] = bel[k];
    p.status[t] = 1;
    flags = 2;
  } else if (depth >= p.max_depth) {                 // pseudo-leaf: root of the agent's next subgame
    double* root = p.root_bel + (size_t)t * 2 * H;
    for (int r = 0; r < 2; ++r) sp_normalize(bel + r * H, H);
    for (int k = 0; k < 2 * H; ++k) root[k] = bel[k];
    p.status[t] = 1;
    flags = 2;
  }
  p.io[i] = a;
  p.flags[i] = flags;
}

__global__ void __launch_bounds__(128) agent_policy_kernel(AgentDev p) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= p.n * p.H) return;
  const int i = g / p.H, hand = g - i * p.H, t = p.ids[i], H = p.H, A = p.A;
  const int lb = p.last_bid[t];
  int cb, nc;
  agent_node(p, t, cb, nc);
  const int lo = lb < 0 ? 0 : lb + 1;
  const double* __restrict__ c = p.cache + (size_t)t * p.stride + (size_t)(cb - 1) * H;
  double* out = p.pol + (size_t)g * A;
  for (int k = 0; k < A; ++k) out[k] = (k >= lo && k < lo + nc) ? c[(size_t)(k - lo) * H + hand] : 0.0;
}

}  // namespace cfrb
