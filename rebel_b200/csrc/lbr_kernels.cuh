// Local best response (Lisý & Bowling, 2017) against one ReBeL agent (cfrb_match_create_lbr), one thread per game slot.
//
// The agent plays exactly as in a head-to-head match with the AVERAGE policy (match_kernels.cuh): it re-solves at the game root
// and at every pseudo-leaf of its previous subgame from its own beliefs and updates both players' beliefs with its own strategy.
// LBR keeps an fp64 belief beta over the agent's hand (uniform, times the agent's strategy after each agent action, renormalised)
// and at each of its decisions plays the argmax over
//   liar:     sum_h beta[h] (b true ? -1 : +1)
//   raise a:  sum_h beta[h] sum_{a' legal after a} sigma(child(a), h, a') u(h, a'),   u = +-1: the agent's liar call on a is
//             settled at once, any raise a' of the agent is called by LBR (the rollout assumption)
// where sigma(child(a)) is the agent's strategy there: from its current table inside the subgame, or, when child(a) is a
// pseudo-leaf, from the root of the agent's subgame at child(a) ("what-if" solve, one per raise).  The what-if solve of the
// chosen raise is the agent's next subgame; the walk continues in it.
//
//   lbr_scan      one CTA: each running slot asks for 1 subgame (game start / pseudo-leaf) or m (a pending LBR decision with m
//                 legal raises); slots are admitted round-robin from after the last slot admitted in the previous round until
//                 the handle's capacity K is full, the others wait a round.  Wave ranges and packed value-net row offsets.
//   lbr_begin     per admitted slot: the descriptor of the agent's next subgame, or the m what-if descriptors with the agent's
//                 beliefs propagated through its own strategy for LBR's seat and eps-normalised (fp64 -> real)
//   lbr_advance   per admitted slot: resolves a pending decision, then walks up to max_depth plies; stops at a pseudo-leaf, at
//                 an LBR decision whose raises lead to pseudo-leaves (pending), or at the liar call (payoff, next game)
//
// Against an EVERY_NODE agent (cfrb_match_create_lbr2) the agent plays as in a per-ply match (ply_kernels.cuh): it solves the
// subgame rooted at every node of the path, whoever moves, and acts and updates the mover's belief row with that root's row
// (avg_prob, en_update_row).  The LBR rule is the same; sigma(child(a)) is always the root row of a what-if solve at child(a):
//   phase 1       LBR to move at X with m > 0 legal raises: one subgame rooted at X from the agent's beliefs; its root row for
//                 LBR's seat goes to sigx (what the agent would multiply LBR's row by after each raise)
//   phase 2       m what-if subgames rooted at the children: the agent's own row as it is, LBR's row times sigx[a], eps-normalised
//                 (the row the agent holds if LBR raises to a; kept in sigx[a])
//   decide, act   LBR values its actions from the what-if roots and chooses.  After a raise the chosen what-if is the agent's
//                 subgame at child(a): it acts for its hand from that root row, updates its own row with it, LBR updates beta,
//                 and the slot waits for phase 1 at LBR's next decision.  At bid A - 2 LBR has no raise and calls at once.
// The agent moving first solves at the game root and acts.  A slot still asks for 1 subgame (phase 1, root) or m (phase 2) a
// round, so lbr_scan and its admission serve both walks unchanged.
//
// Against a blueprint (cfrb_match_create_lbr_blueprint) nothing is solved: sigma is the blueprint's table everywhere, so
//   lbr_blueprint plays a slot's whole game in one round (no scan, no begin, no wave): the agent acts from its row at the slot's
//                 full-tree node, LBR's beta is updated with that row, and LBR values its actions from the rows at the children
// in the order and arithmetic of lbr_advance; a blueprint holding an AVERAGE or EVERY_NODE agent's walked policy gives that
// agent's LBR games bit for bit.
//
// LBR draws no random numbers, so the agent's draws consume the match's (seed, g) streams exactly as in a match.  Compiled into
// the -fmad=false translation unit: every sum runs in the order stated, in fp64, without contraction.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "cfr_types.h"
#include "match_kernels.cuh"
#include "ply_kernels.cuh"

namespace cfrb {

// Subgames (n) and value-net rows (r) slot s asks for in this round.
__device__ __forceinline__ void lbr_need(const LbrDev& p, int s, int& n, int& r) {
  n = 0; r = 0;
  if (p.m.game[s] < 0) return;
  const int lb = p.m.last_bid[s];
  if (!p.pend[s]) { n = 1; r = p.m.tmpl[lb + 1].L; return; }
  for (int a = lb < 0 ? 0 : lb + 1; a <= p.m.A - 2; ++a) { ++n; r += p.m.tmpl[a + 1].L; }
}

__global__ void __launch_bounds__(1024) lbr_scan_kernel(LbrDev p) {
  __shared__ int part[2 * 1024];
  __shared__ int end_n, end_r, last_pos, deferred;
  const MatchDev& q = p.m;
  const int S = q.S, t = threadIdx.x, per = (S + 1023) / 1024, start = *p.rr;
  if (t == 0) { end_n = 0; end_r = 0; last_pos = -1; deferred = 0; }
  const int b = t * per, e = min(S, b + per);
  int n = 0, r = 0;
  for (int i = b; i < e; ++i) {
    int ni, ri;
    lbr_need(p, (start + i) % S, ni, ri);
    n += ni; r += ri;
  }
  int x[2] = {n, r};                                 // subgames, rows
  sp_block_scan(part, x);
  // the needs are >= 0, so the admitted slots (exclusive prefix + need <= K) are a prefix of the rotated order
  int w = x[0] - n, off = x[1] - r, dn = 0;
  for (int i = b; i < e; ++i) {
    const int s = (start + i) % S;
    int ni, ri;
    lbr_need(p, s, ni, ri);
    if (ni > 0 && w + ni <= p.K) {
      q.widx[s] = w; p.nsg[s] = ni;
      if (!p.pend[s]) {
        q.sg_row_off[0][w] = off;
      } else {
        const int lb = q.last_bid[s];
        int o = off;
        for (int a = lb < 0 ? 0 : lb + 1, j = 0; a <= q.A - 2; ++a, ++j) { q.sg_row_off[0][w + j] = o; o += q.tmpl[a + 1].L; }
      }
      atomicMax(&end_n, w + ni); atomicMax(&end_r, off + ri); atomicMax(&last_pos, i);
    } else {
      q.widx[s] = -1; p.nsg[s] = 0;
      if (ni > 0) ++dn;
    }
    w += ni; off += ri;
  }
  if (dn) atomicAdd(&deferred, dn);
  __syncthreads();
  if (t == 0) {
    q.wave[0][0] = end_n; q.wave[0][1] = end_r;
    *q.running = end_n;
    if (last_pos >= 0) *p.rr = (start + last_pos + 1) % S;
    *p.deferred += (unsigned long long)deferred;
  }
}

template <typename real>
__global__ void __launch_bounds__(128) lbr_begin_kernel(LbrDev p, MatchTabs<real> tb) {
  const MatchDev& q = p.m;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= q.S) return;
  const int g = q.game[s], n = g < 0 ? 0 : p.nsg[s];
  if (n == 0) return;
  const int w = q.widx[s], H = q.H, A = q.A, lb = q.last_bid[s], pl = q.player[s];
  const double* b = q.bel + (size_t)s * 4 * H;
  real* wb = tb.wave_beliefs[0];
  if (!p.pend[s]) {                                  // the agent's next subgame
    q.sg_tmpl[0][w] = lb + 1; q.sg_player[0][w] = pl; q.sg_act[0][w] = -1;
    for (int i = 0; i < 2 * H; ++i) wb[(size_t)w * 2 * H + i] = (real)b[i];
    const int r = q.round[s];
    if (g < q.trace_games) {
      const size_t rec = (size_t)g * A + r;
      q.tr_act[rec * 2] = -1; q.tr_act[rec * 2 + 1] = 0;
      for (int i = 0; i < 2 * H; ++i) q.tr_bel[rec * 2 * 2 * H + i] = b[i];
      q.tr_rounds[g] = r + 1;
    }
  } else {                                           // one what-if subgame per raise of LBR (seat pl)
    const int lo = lb < 0 ? 0 : lb + 1;
    for (int a = lo; a <= A - 2; ++a) {
      const int ws = w + a - lo;
      q.sg_tmpl[0][ws] = a + 1; q.sg_player[0][ws] = pl ^ 1; q.sg_act[0][ws] = -1;
      if (p.every_node) {                            // sigx[a] becomes LBR's row times it, eps-normalised (the product commutes,
        double* x = p.sigx + ((size_t)s * A + a) * H;   // so these are ply_advance's bits); the agent's own row as it is
        en_update_row(x, H, [&](int h) { return b[pl * H + h]; });
        for (int k = 0; k < 2; ++k)
          for (int h = 0; h < H; ++h) wb[((size_t)ws * 2 + k) * H + h] = (real)(k == pl ? x[h] : b[k * H + h]);
        continue;
      }
      const double* sx = p.sigx + ((size_t)s * A + a) * H;
      for (int k = 0; k < 2; ++k) {                  // sp_normalize of row k (LBR's row times the agent's strategy)
        const double* bk = b + k * H;
        double sum = 0;
        for (int h = 0; h < H; ++h) sum += (k == pl ? bk[h] * sx[h] : bk[h]) + 1e-80;
        for (int h = 0; h < H; ++h) wb[((size_t)ws * 2 + k) * H + h] = (real)(((k == pl ? bk[h] * sx[h] : bk[h]) + 1e-80) / sum);
      }
    }
    p.whatif[g] += n;
  }
  p.solves[g] += n;
}

template <typename real>
__global__ void __launch_bounds__(128) lbr_advance_kernel(LbrDev p, MatchTabs<real> tb) {
  const MatchDev& q = p.m;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= q.S) return;
  const int g = q.game[s];
  if (g < 0) return;
  if (p.nsg[s] == 0) { atomicAdd(q.left, 1); return; }   // not admitted this round: waits
  const int H = q.H, A = q.A, F = q.F;
  const int me = g & 1;                              // the agent sits in seat 0 in even games
  const int hand_a = q.hands[2 * s + me], hand_l = q.hands[2 * s + (me ^ 1)];
  SpRng rng{q.mt + s, q.S, q.mt_idx[s]};
  double* bel = q.bel + (size_t)s * 4 * H;           // the agent's beliefs [player][hand]
  double* beta = bel + 2 * H;                        // LBR's belief over the agent's hand
  const bool traced = g < q.trace_games;
  int w = q.widx[s], lb = q.last_bid[s], root_player = q.player[s], ply = q.ply[s], round = q.round[s];
  int prev_bid = lb, caller = 0;
  bool terminal = false;
  auto is_true = [&](int bid, int h) {
    const int f = bid % F;
    return (int)q.matches[hand_l * F + f] + (int)q.matches[h * F + f] >= 1 + bid / F;
  };
  auto trace_ply = [&](int who, int bid, int actor, int hand, int action, double prob) {
    if (!traced || ply >= A) return;
    int* rec = q.tr_ply + ((size_t)g * A + ply) * 6;
    rec[0] = who; rec[1] = bid; rec[2] = actor; rec[3] = hand; rec[4] = action; rec[5] = round;
    q.tr_prob[(size_t)g * A + ply] = prob;
  };
  // LBR's decision at a node with last bid b: child(a, wc, cb, nc) gives raise a's node as (wave slot, first child, children)
  auto decide = [&](int b, auto child) -> int {
    const int lo = b < 0 ? 0 : b + 1;
    double* tv = traced && ply < A ? p.tr_val + ((size_t)g * A + ply) * A : nullptr;
    if (tv) for (int h = 0; h < H; ++h) p.tr_beta[((size_t)g * A + ply) * H + h] = beta[h];
    int best = -1;
    double bv = 0;
    for (int a = lo; a <= A - 2; ++a) {
      int wc, cb, nc;
      child(a, wc, cb, nc);
      const real* T = tb.table[0] + (size_t)wc * q.table_stride;
      const bool norm = tb.normalise[0] != 0, untouched = norm && q.steps[0][2 * wc + me] == 0;   // the agent acts at child(a)
      double v = 0;
      for (int h = 0; h < H; ++h) {
        double sum = 0;
        if (norm && !untouched) sum = avg_row_sum(T, cb - 1, h, H, nc);   // once per hand, not per child
        const double ua = is_true(a, h) ? 1.0 : -1.0;
        double inner = 0;
        for (int i = 0; i < nc; ++i) {               // bids a + 1 .. A - 1, the liar call last
          const double sg = avg_entry((double)T[(size_t)(cb - 1 + i) * H + h], sum, nc, norm, untouched);
          const int a2 = a + 1 + i;
          const double u = a2 == A - 1 ? ua : (is_true(a2, h) ? -1.0 : 1.0);
          inner += sg * u;
        }
        v += beta[h] * inner;
      }
      if (tv) tv[a] = v;
      if (best < 0 || v > bv) { best = a; bv = v; }
    }
    if (b >= 0) {
      double v = 0;
      for (int h = 0; h < H; ++h) v += beta[h] * (is_true(b, h) ? -1.0 : 1.0);
      if (tv) tv[A - 1] = v;
      if (best < 0 || v > bv) { best = A - 1; bv = v; }
    }
    return best;
  };
  if (p.pend[s]) {                                   // the what-if solves of the pending decision are in slots w ..
    const int actor = root_player, lo = lb < 0 ? 0 : lb + 1;
    const int a = decide(lb, [&](int a, int& wc, int& cb, int& nc) {
      const int off = q.tmpl[a + 1].node_off;
      wc = w + a - lo; cb = q.child_begin[off]; nc = q.nchild[off];
    });
    trace_ply(1, lb, actor, hand_l, a, 1.0);
    p.pend[s] = 0;
    prev_bid = lb; caller = actor; ++ply;
    if (a == A - 1) {
      terminal = true;
    } else {                                         // the chosen raise's what-if subgame is the agent's next subgame
      const double* sx = p.sigx + ((size_t)s * A + a) * H;
      if (p.every_node) {                            // lbr_begin left the agent's updated row for LBR's seat there
        for (int h = 0; h < H; ++h) bel[actor * H + h] = sx[h];
      } else {
        for (int h = 0; h < H; ++h) bel[actor * H + h] *= sx[h];
        sp_normalize(bel, H); sp_normalize(bel + H, H);
      }
      w += a - lo; lb = a; root_player = actor ^ 1; ++round;
      if (traced) {
        const size_t rec = (size_t)g * A + round;
        q.tr_act[rec * 2] = -1; q.tr_act[rec * 2 + 1] = 0;
        for (int i = 0; i < 2 * H; ++i) q.tr_bel[rec * 2 * 2 * H + i] = bel[i];
        q.tr_rounds[g] = round + 1;
      }
    }
  }
  if (p.every_node && !terminal) {                   // the subgame in slot w is rooted at the slot's node (lb, root_player)
    const int lo = lb < 0 ? 0 : lb + 1, nc = q.nchild[q.tmpl[lb + 1].node_off];
    const real* T = tb.table[0] + (size_t)w * q.table_stride;
    const bool norm = tb.normalise[0] != 0, untouched = norm && q.steps[0][2 * w + root_player] == 0;
    auto sig = [&](int h, int j) { return avg_prob(T, 0, h, H, nc, norm, untouched, j); };
    if (root_player != me) {                         // phase 1: the agent's root row for LBR's seat, per raise
      for (int a = lo; a <= A - 2; ++a)
        for (int h = 0; h < H; ++h) p.sigx[((size_t)s * A + a) * H + h] = sig(h, a - lo);
      p.pend[s] = 1;
      atomicAdd(q.left, 1);
      return;
    }
    const int j = sp_discrete(rng, nc, [&](int i) { return sig(hand_a, i); });   // the agent acts at the root
    trace_ply(0, lb, me, hand_a, lo + j, sig(hand_a, j));
    en_update_row(bel + me * H, H, [&](int h) { return sig(h, j); });
    for (int h = 0; h < H; ++h) beta[h] *= sig(h, j);
    double sum = 0;
    for (int h = 0; h < H; ++h) sum += beta[h];
    for (int h = 0; h < H; ++h) beta[h] /= sum;
    prev_bid = lb; caller = me; lb = lo + j; ++ply;
    if (lb == A - 2) {                               // LBR has no raise: it calls
      const int a = decide(lb, [](int, int&, int&, int&) {});
      trace_ply(1, lb, me ^ 1, hand_l, a, 1.0);
      prev_bid = lb; caller = me ^ 1; ++ply;
    } else if (lb < A - 2) {                         // LBR's next decision waits for phase 1
      match_continue(q, s, lb, me ^ 1, ply, round + 1, rng.idx);
      return;
    }
    terminal = true;
  }
  int depth = 0;
  if (!terminal) {
    const TemplateDev t = q.tmpl[lb + 1];
    const int* __restrict__ child_begin = q.child_begin + t.node_off;
    const int* __restrict__ nchild = q.nchild + t.node_off;
    int node = 0;
    // the agent's strategy at (node, hand, child j) of the subgame in wave slot w
    auto sig = [&](int cb, int nc, int actor, int hand, int j) {
      return avg_prob(tb.table[0] + (size_t)w * q.table_stride, cb - 1, hand, H, nc, tb.normalise[0] != 0,
                      tb.normalise[0] && q.steps[0][2 * w + actor] == 0, j);
    };
    while (depth < q.max_depth) {
      const int nc = nchild[node], cb = child_begin[node], lo = lb < 0 ? 0 : lb + 1;
      const int actor = root_player ^ (depth & 1);
      int j;
      if (actor == me) {
        j = sp_discrete(rng, nc, [&](int i) { return sig(cb, nc, actor, hand_a, i); });
        trace_ply(0, lb, actor, hand_a, lo + j, sig(cb, nc, actor, hand_a, j));
        for (int h = 0; h < H; ++h) {
          const double sg = sig(cb, nc, actor, h, j);
          bel[actor * H + h] *= sg;
          beta[h] *= sg;
        }
        double sum = 0;
        for (int h = 0; h < H; ++h) sum += beta[h];
        for (int h = 0; h < H; ++h) beta[h] /= sum;
      } else {
        if (depth + 1 == q.max_depth && lo <= A - 2) {   // the raises lead to pseudo-leaves: what-if solves first
          for (int a = lo; a <= A - 2; ++a)
            for (int h = 0; h < H; ++h) p.sigx[((size_t)s * A + a) * H + h] = sig(cb, nc, actor, h, a - lo);
          p.pend[s] = 1;
          match_continue(q, s, lb, actor, ply, round, rng.idx);
          return;
        }
        const int a = decide(lb, [&](int a, int& wc, int& cb2, int& nc2) {
          const int c = cb + a - lo;
          wc = w; cb2 = child_begin[c]; nc2 = nchild[c];
        });
        j = a - lo;
        trace_ply(1, lb, actor, hand_l, a, 1.0);
        for (int h = 0; h < H; ++h) bel[actor * H + h] *= sig(cb, nc, actor, h, j);
      }
      prev_bid = lb; caller = actor;
      node = cb + j;
      lb = lo + j;
      ++depth; ++ply;
      if (lb == A - 1) { terminal = true; break; }
    }
  }
  if (!terminal) {                                   // pseudo-leaf: root of the agent's next subgame (beta stays as it is)
    sp_normalize(bel, H); sp_normalize(bel + H, H);
    match_continue(q, s, lb, root_player ^ (depth & 1), ply, round + 1, rng.idx);
    return;
  }
  match_settle<match_start>(q, s, g, prev_bid, caller, ply, round + 1);   // the agent is agent 0: its payoff
}

// One thread per slot: the slot's game to its end against the blueprint p.bp, then match_settle (its next game waits a round).
__global__ void __launch_bounds__(128) lbr_blueprint_kernel(LbrDev p) {
  const MatchDev& q = p.m;
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= q.S) return;
  const int g = q.game[s];
  if (g < 0) return;
  const int H = q.H, A = q.A, F = q.F;
  const int me = g & 1;                              // the agent sits in seat 0 in even games
  const int hand_a = q.hands[2 * s + me], hand_l = q.hands[2 * s + (me ^ 1)];
  const double* __restrict__ bp = p.bp;
  const int* __restrict__ child_begin = p.bp_child_begin;
  SpRng rng{q.mt + s, q.S, q.mt_idx[s]};
  double* beta = q.bel + (size_t)s * 4 * H + 2 * H;  // LBR's belief over the agent's hand (the agent keeps none)
  const bool traced = g < q.trace_games;
  auto is_true = [&](int bid, int h) {
    const int f = bid % F;
    return (int)q.matches[hand_l * F + f] + (int)q.matches[h * F + f] >= 1 + bid / F;
  };
  int lb = -1, actor = 0, node = 0, ply = 0, prev_bid = -1, caller = 0;
  for (;;) {
    const int lo = lb < 0 ? 0 : lb + 1, nc = lb < 0 ? A - 1 : A - 1 - lb, cb = child_begin[node];
    const double* row = bp + (size_t)(cb - 1) * H;   // row[j * H + hand]: the agent's strategy at this node
    int a;
    if (actor == me) {
      const int j = sp_discrete(rng, nc, [&](int i) { return row[(size_t)i * H + hand_a]; });
      a = lo + j;
      if (traced && ply < A) {
        int* rec = q.tr_ply + ((size_t)g * A + ply) * 6;
        rec[0] = 0; rec[1] = lb; rec[2] = actor; rec[3] = hand_a; rec[4] = a; rec[5] = 0;
        q.tr_prob[(size_t)g * A + ply] = row[(size_t)j * H + hand_a];
      }
      for (int h = 0; h < H; ++h) beta[h] *= row[(size_t)j * H + h];
      double sum = 0;
      for (int h = 0; h < H; ++h) sum += beta[h];
      for (int h = 0; h < H; ++h) beta[h] /= sum;
    } else {                                         // lbr_advance's decide, sigma(child(a)) from the table
      double* tv = traced && ply < A ? p.tr_val + ((size_t)g * A + ply) * A : nullptr;
      if (tv) for (int h = 0; h < H; ++h) p.tr_beta[((size_t)g * A + ply) * H + h] = beta[h];
      int best = -1;
      double bv = 0;
      for (int r = lo; r <= A - 2; ++r) {
        const int cb2 = child_begin[cb + r - lo], nc2 = A - 1 - r;
        const double* row2 = bp + (size_t)(cb2 - 1) * H;
        double v = 0;
        for (int h = 0; h < H; ++h) {
          const double ua = is_true(r, h) ? 1.0 : -1.0;
          double inner = 0;
          for (int i = 0; i < nc2; ++i) {            // bids r + 1 .. A - 1, the liar call last
            const int a2 = r + 1 + i;
            const double u = a2 == A - 1 ? ua : (is_true(a2, h) ? -1.0 : 1.0);
            inner += row2[(size_t)i * H + h] * u;
          }
          v += beta[h] * inner;
        }
        if (tv) tv[r] = v;
        if (best < 0 || v > bv) { best = r; bv = v; }
      }
      if (lb >= 0) {
        double v = 0;
        for (int h = 0; h < H; ++h) v += beta[h] * (is_true(lb, h) ? -1.0 : 1.0);
        if (tv) tv[A - 1] = v;
        if (best < 0 || v > bv) { best = A - 1; bv = v; }
      }
      a = best;
      if (traced && ply < A) {
        int* rec = q.tr_ply + ((size_t)g * A + ply) * 6;
        rec[0] = 1; rec[1] = lb; rec[2] = actor; rec[3] = hand_l; rec[4] = a; rec[5] = 0;
        q.tr_prob[(size_t)g * A + ply] = 1.0;
      }
    }
    prev_bid = lb; caller = actor;
    node = cb + a - lo; lb = a; actor ^= 1; ++ply;
    if (a == A - 1) break;
  }
  match_settle<match_start>(q, s, g, prev_bid, caller, ply, 1);
}

}  // namespace cfrb
