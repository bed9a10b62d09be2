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

// std::mt19937(x) into an interleaved state whose words lie `stride` apart (word i at st[i * stride])
__device__ __forceinline__ void mt_seed_strided(uint32_t* st, int stride, uint32_t x) {
  st[0] = x;
  for (int i = 1; i < 624; ++i) { x = 1812433253u * (x ^ (x >> 30)) + (uint32_t)i; st[(size_t)i * stride] = x; }
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

__global__ void __launch_bounds__(128) match_deal_kernel(MatchDev p) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= p.S) return;
  if (s < p.G) match_start(p, s, s);
  else p.game[s] = -1;
}

// Wave index of every running slot (slot order) and the exclusive prefix sum of their pseudo-leaf counts; one CTA.
__global__ void __launch_bounds__(1024) match_scan_kernel(MatchDev p) {
  __shared__ int part_n[1024], part_r[1024];
  const int t = threadIdx.x, per = (p.S + 1023) / 1024;
  const int b = t * per, e = min(p.S, b + per);
  int n = 0, r = 0;
  for (int s = b; s < e; ++s)
    if (p.game[s] >= 0) { ++n; r += p.tmpl[p.last_bid[s] + 1].L; }
  part_n[t] = n; part_r[t] = r;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const int vn = t >= d ? part_n[t - d] : 0, vr = t >= d ? part_r[t - d] : 0;
    __syncthreads();
    part_n[t] += vn; part_r[t] += vr;
    __syncthreads();
  }
  int w = part_n[t] - n, off = part_r[t] - r;
  for (int s = b; s < e; ++s) {
    if (p.game[s] < 0) { p.widx[s] = -1; continue; }
    p.widx[s] = w;
    for (int k = 0; k < 2; ++k) p.sg_row_off[k][w] = off;
    ++w;
    off += p.tmpl[p.last_bid[s] + 1].L;
  }
  if (t == 1023) {
    for (int k = 0; k < 2; ++k) { p.wave[k][0] = part_n[1023]; p.wave[k][1] = part_r[1023]; }
    *p.running = part_n[1023];
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
    int act = -1;
    if (p.sampled) {
      const int n = p.iters[k];
      act = sp_discrete(rng, n, [](int i) { return i % 2 ? 0.0 : (i / 2. + 1); });
    }
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
  // strategy of agent k at (node, hand, child j): average mode = normalise(S) with cfrb_fetch_compact(..., 4)'s operation order
  // and uniform-until-first-update rule (CFR) or the average table itself (FP); sampled mode = the act_iteration snapshot
  auto sig = [&](int k, int node, int actor, int hand, int j) -> double {
    const real* T = tb.table[k] + (size_t)w * p.table_stride;
    const int cb = child_begin[node], nc = nchild[node];
    const double v = (double)T[(size_t)(cb + j - 1) * H + hand];
    if (!tb.normalise[k]) return v;
    if (p.steps[k][2 * w + actor] == 0) return 1.0 / nc;
    double sum = 0;
    for (int i = 0; i < nc; ++i) sum += (double)T[(size_t)(cb + i - 1) * H + hand];
    return sum > 0 ? v / sum : 1.0 / nc;
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
    p.last_bid[s] = lb; p.player[s] = root_player ^ (depth & 1); p.ply[s] = ply; p.round[s] += 1;
    p.mt_idx[s] = rng.idx;
    atomicAdd(p.left, 1);
    return;
  }
  // liar call on bid prev_bid: the bidder wins iff both hands together hold at least `quantity` dice of `face`
  const int quantity = 1 + prev_bid / p.F, face = prev_bid % p.F;
  const int count = (int)p.matches[p.hands[2 * s] * p.F + face] + (int)p.matches[p.hands[2 * s + 1] * p.F + face];
  const int winner = count >= quantity ? caller ^ 1 : caller;
  p.payoff[g] = (winner ^ (g & 1)) == 0 ? 1.f : -1.f;
  p.plies[g] = ply;
  p.rounds[g] = p.round[s] + 1;
  if (traced) p.tr_plies[g] = ply;
  const int next = g + p.S;
  if (next < p.G) {
    match_start(p, s, next);
    atomicAdd(p.left, 1);
  } else {
    p.game[s] = -1;
  }
}

}  // namespace cfrb
