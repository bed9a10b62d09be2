// Per-ply head-to-head matches (cfrb_match_create2 when either agent plays CFRB_MATCH_EVERY_NODE or the two policies differ), one
// thread per game slot.  A round is one ply of every running game: the agents no longer solve the same public nodes, so each
// gets its own wave.
//
//   every-node agent   compute_strategy_recursive (recursive_solving.cc:46-74) along the path played: at every node it solves
//                      the subgame rooted there from its own beliefs and acts with the average strategy of that subgame's root,
//                      read in place from this round's table.  After an action it multiplies the mover's belief row by its root
//                      row and eps-normalises that row (normalize_beliefs_inplace); the other row is unchanged.
//   to-leaf agent      the walk of match_kernels.cuh: a solve at the game root and at every pseudo-leaf of its previous subgame,
//                      the acting strategy of that solve (normalised CFR average, FP average or act_iteration snapshot) copied
//                      into a per-slot fp64 cache right after it (the handle's tables are rebuilt every round), beliefs
//                      multiplied unnormalised inside the subgame and both of its rows eps-normalised at its pseudo-leaf.
//   blueprint agent    a fixed full-tree table (cfrb_blueprint, cfrb_match_create3): it never solves and keeps no beliefs; each
//                      slot holds the full-tree node its game stands at (0 at the game root, child_begin[node] + j after action j),
//                      and the agent acts with bp[(child_begin[node] + j - 1) * H + hand].  Its trace act_iteration is -2 on
//                      every ply and its traced beliefs stay uniform.  A match between two blueprints has no handle and no
//                      templates: scan and begin only pack empty waves and write the trace.
//
//   ply_scan      one CTA: per agent, the wave index of every running slot where it solves and the packed value-net row offsets
//   ply_begin     per slot: each solving agent's subgame descriptor (and, sampled, its act_iteration), the trace of the ply's beliefs
//   ply_capture   warp per (to-leaf agent, solving slot): the acting strategy into the cache (capture_levels)
//   ply_advance   per slot: one action of the mover's agent for the mover's hand, both agents' belief updates, and at a liar call
//                 the payoff and the slot's next game (match_start)
//
// Draws of game g come from match_kernels.cuh's (seed, g) streams in a fixed order per ply: agent 0's act_iteration when it starts
// a sampled subgame, agent 1's, then the action; so results do not depend on n_slots.  This header is compiled into the
// -fmad=false translation unit: every belief operation is the host walks', bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cfr_types.h"
#include "match_kernels.cuh"
#include "selfplay_kernels.cuh"

namespace cfrb {

constexpr int kPlySampled = 1, kPlyEveryNode = 2;   // CFRB_MATCH_SAMPLED, CFRB_MATCH_EVERY_NODE

// An every-node agent's update of the mover's belief row after an action: times sig(h), then eps-normalised.
template <typename Sig>
__device__ __forceinline__ void en_update_row(double* row, int H, Sig sig) {
  for (int h = 0; h < H; ++h) row[h] *= sig(h);
  sp_normalize(row, H);
}

// Does agent k solve at slot s this round?  An every-node agent at every node, a to-leaf one when it has no solved subgame there.
__device__ __forceinline__ bool ply_solves(const MatchDev& p, int k, int s) {
  return p.game[s] >= 0 && p.policy[k] != kPlyBlueprint && (p.policy[k] == kPlyEveryNode || p.sub_node[k][s] < 0);
}

// Game g in slot s (match_start), neither agent holding a subgame, a blueprint agent at the full tree's root.
__device__ void ply_start(const MatchDev& p, int s, int g) {
  match_start(p, s, g);
  p.sub_node[0][s] = p.sub_node[1][s] = -1;
  for (int k = 0; k < 2; ++k)
    if (p.bp_node[k]) p.bp_node[k][s] = 0;
}

// Per agent: the wave index of every slot it solves (slot order) and the exclusive prefix sum of their pseudo-leaf counts; one CTA.
__global__ void __launch_bounds__(1024) ply_scan_kernel(MatchDev p) {
  __shared__ int part[5 * 1024];
  const int t = threadIdx.x, per = (p.S + 1023) / 1024;
  const int b = t * per, e = min(p.S, b + per);
  int v[5] = {0, 0, 0, 0, 0};                        // agent 0 slots, rows; agent 1 slots, rows; running slots
  for (int s = b; s < e; ++s) {
    if (p.game[s] < 0) continue;
    for (int k = 0; k < 2; ++k)
      if (ply_solves(p, k, s)) { v[2 * k] += 1; v[2 * k + 1] += p.tmpl[p.last_bid[s] + 1].L; }
    v[4] += 1;
  }
  int x[5] = {v[0], v[1], v[2], v[3], v[4]};        // inclusive sums; v stays for the exclusive offsets
  sp_block_scan(part, x);
  int w[2], off[2];
  for (int k = 0; k < 2; ++k) { w[k] = x[2 * k] - v[2 * k]; off[k] = x[2 * k + 1] - v[2 * k + 1]; }
  for (int s = b; s < e; ++s) {
    for (int k = 0; k < 2; ++k) {
      if (!ply_solves(p, k, s)) { p.awidx[k][s] = -1; continue; }
      p.awidx[k][s] = w[k];
      p.sg_row_off[k][w[k]] = off[k];
      ++w[k];
      off[k] += p.tmpl[p.last_bid[s] + 1].L;
    }
  }
  if (t == 1023) {
    for (int k = 0; k < 2; ++k)
      if (p.wave[k]) { p.wave[k][0] = x[2 * k]; p.wave[k][1] = x[2 * k + 1]; }   // a blueprint has no wave
    *p.running = x[4];
  }
}

template <typename real>
__global__ void __launch_bounds__(128) ply_begin_kernel(MatchDev p, MatchTabs<real> tb) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  const int g = p.game[s];
  if (g < 0) return;
  const int H = p.H, r = p.round[s];
  SpRng rng{p.mt + s, p.S, p.mt_idx[s]};
  const double* b = p.bel + (size_t)s * 4 * H;
  const bool traced = g < p.trace_games;
  for (int k = 0; k < 2; ++k) {
    const int w = p.awidx[k][s];
    int act = -2;                                    // -2: k plays on inside its to-leaf subgame
    if (w >= 0) {
      act = -1;
      if (p.policy[k] == kPlySampled) act = sp_act_iteration(rng, p.iters[k]);
      p.sg_tmpl[k][w] = p.last_bid[s] + 1;
      p.sg_player[k][w] = p.player[s];
      p.sg_act[k][w] = act;
      for (int i = 0; i < 2 * H; ++i) tb.wave_beliefs[k][(size_t)w * 2 * H + i] = (real)b[k * 2 * H + i];
      if (p.policy[k] != kPlyEveryNode) {
        p.sub_lb[k][s] = p.last_bid[s]; p.sub_player[k][s] = p.player[s]; p.sub_node[k][s] = 0; p.sub_depth[k][s] = 0;
      }
      p.solves[k][g] += 1;
    }
    if (traced) {
      const size_t rec = (size_t)g * p.A + r;
      p.tr_act[rec * 2 + k] = act;
      for (int i = 0; i < 2 * H; ++i) p.tr_bel[(rec * 2 + k) * 2 * H + i] = b[k * 2 * H + i];
    }
  }
  if (traced) p.tr_rounds[g] = r + 1;
  p.mt_idx[s] = rng.idx;
}

// One warp per (to-leaf agent, slot it solved at); the lanes stride over the (node, hand) pairs of one level, hands innermost.
template <typename real>
__global__ void __launch_bounds__(128) ply_capture_kernel(MatchDev p, MatchTabs<real> tb) {
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (i >= 2 * p.S) return;
  const int k = i / p.S, s = i - k * p.S;
  if (!p.cache[k]) return;                           // every-node agents read their tables in place
  const int w = p.awidx[k][s];
  if (w < 0) return;
  const TemplateDev tp = p.tmpl[p.sub_lb[k][s] + 1];
  capture_levels(lane, tp, p.child_begin, p.nchild, p.level_begin, p.H, tb.table[k] + (size_t)w * p.table_stride,
                 tb.normalise[k] != 0, p.steps[k] + 2 * w, p.sub_player[k][s], tp.levels, p.cache[k] + (size_t)s * p.table_stride);
}

template <typename real>
__global__ void __launch_bounds__(128) ply_advance_kernel(MatchDev p, MatchTabs<real> tb) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  const int g = p.game[s];
  if (g < 0) return;
  const int H = p.H, A = p.A;
  SpRng rng{p.mt + s, p.S, p.mt_idx[s]};
  const int lb = p.last_bid[s], actor = p.player[s];
  const int agent = actor ^ (g & 1);                 // agent A (0) sits in seat 0 in even games
  const int hand = p.hands[2 * s + actor];
  const int lo = lb < 0 ? 0 : lb + 1;
  // children of this public node (the root of a subgame rooted here; bids lo .. A - 1, no liar call at the game root)
  const int nc = p.tmpl ? p.nchild[p.tmpl[lb + 1].node_off] : lb < 0 ? A - 1 : A - 1 - lb;
  // the edges of this node in each agent's strategy: an every-node agent's root row in this round's table (row j = edge j), a
  // to-leaf agent's node in its cache, a blueprint's node in its table
  const real* T[2] = {nullptr, nullptr};
  const double* c[2] = {nullptr, nullptr};
  bool untouched[2] = {false, false};
  int bcb[2] = {0, 0};                               // a blueprint's first child of its node
  for (int k = 0; k < 2; ++k) {
    if (p.policy[k] == kPlyBlueprint) {
      bcb[k] = p.bp_child_begin[k][p.bp_node[k][s]];
      c[k] = p.bp[k] + (size_t)(bcb[k] - 1) * H;
    } else if (p.policy[k] == kPlyEveryNode) {
      const int w = p.awidx[k][s];
      T[k] = tb.table[k] + (size_t)w * p.table_stride;
      untouched[k] = tb.normalise[k] && p.steps[k][2 * w + actor] == 0;
    } else {
      const int cb = p.child_begin[p.tmpl[p.sub_lb[k][s] + 1].node_off + p.sub_node[k][s]];
      c[k] = p.cache[k] + (size_t)s * p.table_stride + (size_t)(cb - 1) * H;
    }
  }
  // agent k's probability of edge j for hand h: the every-node root row, or the cached entry
  auto sig = [&](int k, int h, int j) -> double {
    if (c[k]) return c[k][(size_t)j * H + h];
    return avg_prob(T[k], 0, h, H, nc, tb.normalise[k] != 0, untouched[k], j);
  };
  const int j = sp_discrete(rng, nc, [&](int i) { return sig(agent, hand, i); });
  const int ply = p.ply[s], a = lo + j;
  const bool terminal = a == A - 1;
  if (g < p.trace_games && ply < A) {
    int* rec = p.tr_ply + ((size_t)g * A + ply) * 6;
    rec[0] = agent; rec[1] = lb; rec[2] = actor; rec[3] = hand; rec[4] = a; rec[5] = p.round[s];
    p.tr_prob[(size_t)g * A + ply] = sig(agent, hand, j);
  }
  double* bel = p.bel + (size_t)s * 4 * H;           // [agent][player][hand]
  for (int k = 0; k < 2; ++k) {
    if (p.policy[k] == kPlyBlueprint) { p.bp_node[k][s] = bcb[k] + j; continue; }   // no beliefs to update
    double* bk = bel + (k * 2 + actor) * H;
    if (!c[k]) {
      en_update_row(bk, H, [&](int h) { return sig(k, h, j); });
      continue;
    }
    for (int h = 0; h < H; ++h) bk[h] *= sig(k, h, j);
    const int node = p.sub_node[k][s], depth = p.sub_depth[k][s] + 1;
    p.sub_node[k][s] = p.child_begin[p.tmpl[p.sub_lb[k][s] + 1].node_off + node] + j;
    p.sub_depth[k][s] = depth;
    if (!terminal && depth >= p.max_depth) {         // pseudo-leaf: the root of k's next subgame
      for (int i = 0; i < 2; ++i) sp_normalize(bel + (k * 2 + i) * H, H);
      p.sub_node[k][s] = -1;
    }
  }
  if (!terminal) match_continue(p, s, a, actor ^ 1, ply + 1, p.round[s] + 1, rng.idx);
  else match_settle<ply_start>(p, s, g, lb, actor, ply + 1, p.round[s] + 1);
}

}  // namespace cfrb
