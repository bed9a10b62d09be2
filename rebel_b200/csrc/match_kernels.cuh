// Head-to-head matches between two ReBeL agents (cfrb_match_*), one thread per game slot.
//
// An agent is a solver configuration plus a value net, i.e. one handle.  It plays the reference's recursive to-leaf strategy
// (compute_strategy_recursive_to_leaf / compute_sampled_strategy_recursive_to_leaf, recursive_solving.cc:76-134, 301-327)
// restricted to the path actually played: at the game root and at every pseudo-leaf of its previous subgame it solves the
// subgame rooted at the current public node from its OWN beliefs, acts inside that subgame with the subgame's strategy for the
// hand dealt to its seat, and propagates both players' beliefs with its own strategy — unnormalised inside the subgame,
// eps-normalised at the subgame's leaf (RecursiveEvaluator::expand).  Both agents update their beliefs at every node, whoever
// acts there.  A round is one wave per agent (the subgames of every running game) followed by the walk below.
//
//   match_scan      one CTA: wave index of every running slot (finished slots drop out) and the packed value-net row offsets,
//                   written into both handles' wave descriptors (both agents solve the same public nodes)
//   match_begin     per slot: the subgame descriptor of each agent (template, player, fp64 -> real beliefs) and, in sampled
//                   mode, each agent's act_iteration ~ weight i/2 + 1 on even i < num_iters (recursive_solving.cc:304-319)
//   match_advance   per slot: at most max_depth plies from the subgame root, reading both handles' tables in place; at a
//                   terminal the payoff, and the next game of the slot's quota (seeded and dealt by match_start)
//
// Reproducibility: every draw of game g comes from an mt19937 keyed by (seed, g) (the deal from one keyed by (seed, g / 2)),
// consumed in a fixed per-game order, so a game's result does not depend on the slot it runs in or on how many run at once.
// Unbiased stopping: slot s plays games s, s + S, s + 2S, ... < G, each to its end; a slot whose quota is done drops out.
// This header is compiled into the -fmad=false translation unit: the belief arithmetic is the host restatement's, bit for bit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cfr_types.h"
#include "selfplay_kernels.cuh"

namespace cfrb {

// A 32-bit mt19937 seed for stream `tag` of key `key` (splitmix64 finaliser over the three words).
__device__ __forceinline__ uint32_t match_stream_seed(uint64_t seed, uint64_t key, uint64_t tag) {
  uint64_t z = seed * 0x9E3779B97F4A7C15ull + key * 0xD1B54A32D192ED03ull + tag * 0x8CB92BA72F3D8DD7ull + 0x632BE59BD9B4E019ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)z ^ (uint32_t)(z >> 32);
}

// std::mt19937(x) into the interleaved state of slot s
__device__ __forceinline__ void match_mt_seed(const MatchDev& p, int s, uint32_t x) {
  mt_seed_strided(p.mt + s, p.S, x);
  p.mt_idx[s] = 624;
}

// Start game g in slot s: deal (both seats' hands from the pair's stream), uniform beliefs, then the game's own stream.
__device__ void match_start(const MatchDev& p, int s, int g) {
  match_mt_seed(p, s, match_stream_seed(p.seed, (uint64_t)(g >> 1), 1));
  SpRng deal{p.mt + s, p.S, 624};
  p.hands[2 * s] = deal.uniform_int(0, p.H - 1);
  p.hands[2 * s + 1] = deal.uniform_int(0, p.H - 1);
  match_mt_seed(p, s, match_stream_seed(p.seed, (uint64_t)g, 2));
  p.game[s] = g; p.last_bid[s] = -1; p.player[s] = 0; p.ply[s] = 0; p.round[s] = 0;
  double* b = p.bel + (size_t)s * 4 * p.H;
  for (int i = 0; i < 4 * p.H; ++i) b[i] = 1.0 / p.H;
}

// The start of a game in a slot: match_start, or ply_start for the per-ply walk (ply_kernels.cuh).
using MatchStart = void (*)(const MatchDev&, int, int);

// Game s in slot s, or the slot retired when there are fewer games than slots.
template <MatchStart start>
__global__ void __launch_bounds__(128) match_deal_kernel(MatchDev p) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  if (s < p.G) start(p, s, s);
  else p.game[s] = -1;
}

// Slot s stops at the root of its next subgame: public node (last_bid, player), plies and rounds so far, and its stream position.
__device__ __forceinline__ void match_continue(const MatchDev& p, int s, int last_bid, int player, int ply, int round, int mt_idx) {
  p.last_bid[s] = last_bid; p.player[s] = player; p.ply[s] = ply; p.round[s] = round;
  p.mt_idx[s] = mt_idx;
  atomicAdd(p.left, 1);
}

// The liar call of seat `caller` on bid `bid` ends game g in slot s after `plies` plies and `rounds` rounds: the bidder wins iff
// both hands together hold at least `quantity` dice of `face`, and the payoff is agent 0's (seat 0 in even games).  The slot then
// starts its next game, or retires when its quota is done.
template <MatchStart start>
__device__ __forceinline__ void match_settle(const MatchDev& p, int s, int g, int bid, int caller, int plies, int rounds) {
  const int quantity = 1 + bid / p.F, face = bid % p.F;
  const int count = (int)p.matches[p.hands[2 * s] * p.F + face] + (int)p.matches[p.hands[2 * s + 1] * p.F + face];
  const int winner = count >= quantity ? caller ^ 1 : caller;
  p.payoff[g] = (winner ^ (g & 1)) == 0 ? 1.f : -1.f;
  p.plies[g] = plies;
  p.rounds[g] = rounds;
  if (g < p.trace_games) p.tr_plies[g] = plies;
  const int next = g + p.S;
  if (next < p.G) {
    start(p, s, next);
    atomicAdd(p.left, 1);
  } else {
    p.game[s] = -1;
  }
}

// Levels [0, levels) of the acting strategy (avg_row) of the subgame with template tp solved in one wave slot, into a cache row c,
// entry (child - 1) * H + hand; by one warp, whose lanes stride over the (node, hand) pairs of a level, hands innermost.  T is the
// slot's table, steps its two step counters, root_player the player to move at the subgame's root.  The per-ply walk and the agent
// (agent_kernels.cuh) cache their solves through this.
template <typename real>
__device__ __forceinline__ void capture_levels(int lane, const TemplateDev& tp, const int* __restrict__ child_begin,
                                               const int* __restrict__ nchild, const int* __restrict__ level_begin, int H,
                                               const real* __restrict__ T, bool normalise, const int* __restrict__ steps,
                                               int root_player, int levels, double* __restrict__ c) {
  child_begin += tp.node_off; nchild += tp.node_off;
  const int* __restrict__ level = level_begin + tp.level_off;
  for (int d = 0; d < levels; ++d) {
    const int nb = level[d], ne = level[d + 1];
    const bool untouched = normalise && steps[root_player ^ (d & 1)] == 0;
    for (int e = nb * H + lane; e < ne * H; e += 32) {
      const int node = e / H, hand = e - node * H;
      const int cb = child_begin[node], nc = nchild[node];
      if (nc == 0) continue;
      const size_t at = (size_t)(cb - 1) * H + hand;
      avg_row(c + at, T + at, 0, 0, H, nc, normalise, untouched);
    }
  }
}

// Wave index of every running slot (slot order) and the exclusive prefix sum of their pseudo-leaf counts; one CTA.
__global__ void __launch_bounds__(1024) match_scan_kernel(MatchDev p) {
  __shared__ int part[2 * 1024];
  const int t = threadIdx.x, per = (p.S + 1023) / 1024;
  const int b = t * per, e = min(p.S, b + per);
  int n = 0, r = 0;
  for (int s = b; s < e; ++s)
    if (p.game[s] >= 0) { ++n; r += p.tmpl[p.last_bid[s] + 1].L; }
  int x[2] = {n, r};                                 // running slots, rows
  sp_block_scan(part, x);
  int w = x[0] - n, off = x[1] - r;
  for (int s = b; s < e; ++s) {
    if (p.game[s] < 0) { p.widx[s] = -1; continue; }
    p.widx[s] = w;
    for (int k = 0; k < 2; ++k) p.sg_row_off[k][w] = off;
    ++w;
    off += p.tmpl[p.last_bid[s] + 1].L;
  }
  if (t == 1023) {
    for (int k = 0; k < 2; ++k) { p.wave[k][0] = x[0]; p.wave[k][1] = x[1]; }
    *p.running = x[0];
  }
}

template <typename real>
__global__ void __launch_bounds__(128) match_begin_kernel(MatchDev p, MatchTabs<real> tb) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  const int g = p.game[s];
  if (g < 0) return;
  const int w = p.widx[s], H = p.H;
  SpRng rng{p.mt + s, p.S, p.mt_idx[s]};
  const double* b = p.bel + (size_t)s * 4 * H;
  const int r = p.round[s];
  const bool traced = g < p.trace_games;
  for (int k = 0; k < 2; ++k) {
    const int act = p.sampled ? sp_act_iteration(rng, p.iters[k]) : -1;
    p.sg_tmpl[k][w] = p.last_bid[s] + 1;
    p.sg_player[k][w] = p.player[s];
    p.sg_act[k][w] = act;
    p.act[2 * s + k] = act;
    for (int i = 0; i < 2 * H; ++i) tb.wave_beliefs[k][(size_t)w * 2 * H + i] = (real)b[k * 2 * H + i];
    if (traced) {
      const size_t rec = (size_t)g * p.A + r;
      p.tr_act[rec * 2 + k] = act;
      for (int i = 0; i < 2 * H; ++i) p.tr_bel[(rec * 2 + k) * 2 * H + i] = b[k * 2 * H + i];
    }
  }
  if (traced) p.tr_rounds[g] = r + 1;
  p.mt_idx[s] = rng.idx;
}

template <typename real>
__global__ void __launch_bounds__(128) match_advance_kernel(MatchDev p, MatchTabs<real> tb) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  const int g = p.game[s];
  if (g < 0) return;
  const int w = p.widx[s], H = p.H, A = p.A;
  SpRng rng{p.mt + s, p.S, p.mt_idx[s]};
  int lb = p.last_bid[s];
  const int root_player = p.player[s];
  const TemplateDev t = p.tmpl[lb + 1];
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  double* bel = p.bel + (size_t)s * 4 * H;         // [agent][player][hand]
  const bool traced = g < p.trace_games;
  // strategy of agent k at (node, hand, child j): average mode = avg_prob of S (CFR) or Sg (FP); sampled mode = the act_iteration
  // snapshot, as it is
  auto sig = [&](int k, int node, int actor, int hand, int j) -> double {
    const real* T = tb.table[k] + (size_t)w * p.table_stride;
    return avg_prob(T, child_begin[node] - 1, hand, H, nchild[node], tb.normalise[k] != 0,
                    tb.normalise[k] && p.steps[k][2 * w + actor] == 0, j);
  };
  int node = 0, depth = 0, ply = p.ply[s], prev_bid = lb, caller = 0;
  bool terminal = false;
  while (depth < p.max_depth) {
    const int nc = nchild[node], lo = lb < 0 ? 0 : lb + 1;
    const int actor = root_player ^ (depth & 1);
    const int agent = actor ^ (g & 1);               // agent A (0) sits in seat 0 in even games
    const int hand = p.hands[2 * s + actor];
    const int j = sp_discrete(rng, nc, [&](int i) { return sig(agent, node, actor, hand, i); });
    if (traced && ply < A) {
      int* rec = p.tr_ply + ((size_t)g * A + ply) * 6;
      rec[0] = agent; rec[1] = lb; rec[2] = actor; rec[3] = hand; rec[4] = lo + j; rec[5] = p.round[s];
      p.tr_prob[(size_t)g * A + ply] = sig(agent, node, actor, hand, j);
    }
    for (int k = 0; k < 2; ++k) {
      double* bk = bel + (k * 2 + actor) * H;
      for (int h = 0; h < H; ++h) bk[h] *= sig(k, node, actor, h, j);
    }
    prev_bid = lb; caller = actor;
    node = child_begin[node] + j;
    lb = lo + j;
    ++depth; ++ply;
    if (lb == A - 1) { terminal = true; break; }
  }
  if (!terminal) {                                   // pseudo-leaf: root of both agents' next subgames
    for (int i = 0; i < 4; ++i) sp_normalize(bel + i * H, H);
    match_continue(p, s, lb, root_player ^ (depth & 1), ply, p.round[s] + 1, rng.idx);
    return;
  }
  match_settle<match_start>(p, s, g, prev_bid, caller, ply, p.round[s] + 1);
}

}  // namespace cfrb
