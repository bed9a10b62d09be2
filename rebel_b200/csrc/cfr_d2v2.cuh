// Depth <= 2 CFR iteration kernel, generation 2 (CFR solver; fictitious play stays on cfr_iter_d2_kernel).
//
// Same arithmetic as cfr_backward_d2 / cfr_forward_d2 (cfr_kernels.cuh) — every fp64 operation of the reference's CFR::step
// (subgame_solving.cc:577-664), update_regrets (:538-575), compute_reach_probabilities (:54-78), write_query_to (:104-123),
// query_value_net scaling (:253-269) and compute_expected_terminal_values / compute_win_probability (:80-98, :765-789) in the
// reference's order, so the results are bit-identical — but re-organised around the long-scoreboard stalls (dependent loads) that
// limit generation 1:
//
//  * STAGING BY THE BULK-COPY ENGINE.  Everything a subgame reads in one launch is contiguous in HBM: its strategy table
//    (all edges), the regret / sum-strategy rows of the traverser's level, its value-net output rows, scalers and terminal
//    payoffs.  One lane issues five cp.async.bulk copies (SASS: UBLKCP) onto one mbarrier at kernel entry; every phase then
//    reads shared memory (29 cycles) instead of L2 / HBM (300-800 cycles, one dependent round trip per phase before).
//    Stores stay direct (fire and forget).
//  * FEWER INSTRUCTIONS.  (1) The query rows: the normalised beliefs of the root player are the same for all leaves under
//    one level-1 node, so they are normalised once per level-1 node (12 instead of 66 at 1x6f); rows are assembled from
//    fp16 values kept in shared memory instead of re-deriving every column per (leaf, 16-byte chunk).  (2) Regret matching
//    divides every positive regret by the node's sum; IEEE division is ~50 instructions in fp64.  Here the reciprocal of the
//    sum is formed once per (node, hand) with a true division and every quotient is obtained from it with two fused
//    multiply-add correction steps (Markstein), which yields the correctly rounded quotient — the same bits as `/`.
//  * One warp per CTA: shared memory per subgame grows to ~19 KB (11 warps per SM instead of 32), but a warp no longer waits
//    on memory between phases, and CTAs of one warp retire independently (no round quantisation inside a CTA).
#pragma once
#include "cfr_kernels.cuh"

namespace cfrb {

__device__ __forceinline__ uint32_t d2v2_smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void d2v2_bulk(void* smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(d2v2_smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(bar) : "memory");
}

// Shared memory of one subgame (bytes, every region 16-byte aligned).
struct D2v2Layout {
  int off_val, off_bel, off_sg, off_r, off_s, off_io, off_bar, bytes;
  int io_net, io_scal, io_vterm;             // staging view of the io region
  int io_hist, io_par, io_qpar, io_qown;     // forward-half view of the same region
  __host__ __device__ D2v2Layout(int sz, int Nmax, int H, int Hout, int Lmax, int Tmax, int n1max, int stride) {
    auto up = [](int x) { return (x + 15) & ~15; };
    int o = 0;
    off_val = o; o += up(Nmax * H * sz);
    off_bel = o; o += up(2 * H * sz);
    off_sg = o; o += up(stride * sz);
    off_r = o; o += up(stride * sz) + 16;
    off_s = o; o += up(stride * sz) + 16;
    off_io = o;
    io_net = 0;
    io_scal = up(Lmax * Hout * 4);
    io_vterm = io_scal + up((Lmax + 4) * sz);
    const int stage_end = io_vterm + up((Tmax * H + 4) * sz);
    io_hist = 0;
    io_par = up(10 * Tmax * sz);                       // [3][n1max] reals: sum, sum + eps, 1 / (sum + eps)
    io_qpar = io_par + up(3 * n1max * sz);            // [n1max][H] halves
    io_qown = io_qpar + up(n1max * H * 2);            // [Lmax][H] halves
    const int fwd_end = io_qown + up(Lmax * H * 2);
    o += stage_end > fwd_end ? stage_end : fwd_end;
    off_bar = o; o += 16;
    bytes = o;
  }
};

// GT = threads per subgame (= per CTA): 32, 64 or 128.  More threads shorten every phase of the one subgame the CTA owns (its
// staged tables are shared), at the price of idle lanes in the short phases.
template <typename real, int HC, int GT>
__global__ void __launch_bounds__(GT, 8) cfr_iter_d2v2_kernel(CfrDev<real> p, int iter, int do_b, int do_f, int n1max) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  asm volatile("griddepcontrol.launch_dependents;");
  const int lane = threadIdx.x;
  const int k = blockIdx.x;
  if (k >= *p.wave_n) return;
  constexpr int G = GT;
  auto group_sync = [] { if (GT == 32) __syncwarp(); else __syncthreads(); };
  constexpr int kAl = 16 / (int)sizeof(real);          // elements per 16 bytes
  const int H = HC > 0 ? HC : p.H;
  const TemplateDev t = p.tmpl[p.sg_tmpl[k]];
  const int rp = p.sg_player[k];
  const int row0 = p.sg_row_off[k];
  const D2Levels lv = d2_levels(p.level_begin, t);
  const int n1 = lv.n1e - lv.n1b;                      // level-1 nodes are 1 .. n1
  const int E = t.N - 1;
  const int tb = (iter - 1) & 1, tf = iter & 1;
  const bool mine0 = rp == tb;                         // the backward half's traverser acts at the root (else on level 1)
  const D2v2Layout Lo((int)sizeof(real), p.nh_max / p.H, p.H, p.Hout, p.lmax, p.tmax, n1max, p.table_stride);
  real* val = reinterpret_cast<real*>(smem_raw + Lo.off_val);
  real* bel = reinterpret_cast<real*>(smem_raw + Lo.off_bel);
  real* sgs = reinterpret_cast<real*>(smem_raw + Lo.off_sg);
  real* rs = reinterpret_cast<real*>(smem_raw + Lo.off_r);
  real* ss = reinterpret_cast<real*>(smem_raw + Lo.off_s);
  unsigned char* io = smem_raw + Lo.off_io;
  const uint32_t bar = d2v2_smem_u32(smem_raw + Lo.off_bar);
  const int* __restrict__ parent = p.parent + t.node_off;
  const int* __restrict__ nchild = p.nchild + t.node_off;
  const int* __restrict__ child_begin = p.child_begin + t.node_off;
  const int* __restrict__ pleaf = p.pleaf_node + t.pleaf_off;
  const int* __restrict__ term = p.term_node + t.term_off;
  real* Rg = p.R + (size_t)k * p.table_stride;
  real* Sgg = p.Sg + (size_t)k * p.table_stride;
  real* Sg_ = p.S + (size_t)k * p.table_stride;

  // ---- staging.  Edge ranges: level 1 = [0, n1), level 2 = [n1, E).  The traverser of the backward half owns [e0, e1).
  const int e0 = mine0 ? 0 : n1, e1 = mine0 ? n1 : E;
  const int ra = (e0 * H) & ~(kAl - 1);                // aligned start of the regret / sum rows that are staged
  const int scal_a = row0 & ~(kAl - 1);
  if (lane == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  group_sync();
  // the previous kernels' outputs (value-net rows; tables written by the previous CFR launch) are read from here on
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (lane == 0) {
    const uint32_t b_sg = (uint32_t)(((E * H + kAl - 1) & ~(kAl - 1)) * sizeof(real));
    uint32_t total = b_sg, b_rs = 0, b_net = 0, b_scal = 0, b_vt = 0;
    if (do_b) {
      b_rs = (uint32_t)((((e1 * H + kAl - 1) & ~(kAl - 1)) - ra) * sizeof(real));
      total += 2 * b_rs;
      if (t.L > 0 && p.use_net) {
        b_net = (uint32_t)(t.L * p.Hout * 4);
        b_scal = (uint32_t)((((row0 + t.L + kAl - 1) & ~(kAl - 1)) - scal_a) * sizeof(real));
        total += b_net + b_scal;
      }
      if (t.T > 0) { b_vt = (uint32_t)(((t.T * H + kAl - 1) & ~(kAl - 1)) * sizeof(real)); total += b_vt; }
    }
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(total) : "memory");
    d2v2_bulk(sgs, Sgg, b_sg, bar);
    if (b_rs) { d2v2_bulk(rs, Rg + ra, b_rs, bar); d2v2_bulk(ss, Sg_ + ra, b_rs, bar); }
    if (b_net) {
      d2v2_bulk(io + Lo.io_net, p.net_out + (size_t)row0 * p.Hout, b_net, bar);
      d2v2_bulk(io + Lo.io_scal, p.scaler + scal_a, b_scal, bar);
    }
    if (b_vt) d2v2_bulk(io + Lo.io_vterm, p.vterm + (size_t)k * p.vterm_stride, b_vt, bar);
  }
  for (int i = lane; i < 2 * H; i += G) bel[i] = p.beliefs[(size_t)k * 2 * H + i];
  const int s_steps = do_b ? p.steps[2 * k + tb] : 0;
  {   // wait for the bytes (phase 0 of a freshly initialised barrier)
    uint32_t done = 0;
    while (!done)
      asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar) : "memory");
  }
  group_sync();
  const real* rsv = rs - ra;                           // rsv[e * H + h] for the staged edges
  const real* ssv = ss - ra;

  if (do_b) {
    const int trav = tb;
    // ---- leaf values = (float)(net(query) * scaler) (subgame_solving.cc:266-282); terminals from the previous forward half
    {
      const float* net_s = reinterpret_cast<const float*>(io + Lo.io_net);
      const real* scal_s = reinterpret_cast<const real*>(io + Lo.io_scal) + (row0 - scal_a);
      for (int it = lane; it < t.L * H; it += G) {
        const int r = it / H, h = it % H;
        val[pleaf[r] * H + h] = p.use_net ? (real)(float)((real)net_s[r * p.Hout + h] * scal_s[r]) : (real)0;
      }
      const real* vt_s = reinterpret_cast<const real*>(io + Lo.io_vterm);
      for (int it = lane; it < t.T * H; it += G) {
        const int z = it / H, h = it % H;
        val[term[z] * H + h] = vt_s[it];
      }
    }
    group_sync();
    // ---- bottom-up (update_regrets :538-575): level-1 node values, then the root
    if (lv.n2e > lv.n1e) {
      for (int it = lane; it < n1 * H; it += G) {
        const int n = 1 + it / H, h = it % H;
        const int nc = nchild[n];
        if (!nc) continue;
        const int c0 = child_begin[n];
        real v = 0;
        if (!mine0) { for (int j = 0; j < nc; ++j) v += val[(c0 + j) * H + h] * sgs[(c0 + j - 1) * H + h]; }
        else        { for (int j = 0; j < nc; ++j) v += val[(c0 + j) * H + h]; }
        val[n * H + h] = v;
      }
      group_sync();
      if (!mine0) {   // new regrets of the level-1 actions, kept in the child's slot
        for (int it = lane; it < (lv.n2e - lv.n1e) * H; it += G) {
          const int c = lv.n1e + it / H, h = it % H;
          val[c * H + h] = (rsv[(c - 1) * H + h] + val[c * H + h]) - val[parent[c] * H + h];
        }
      }
    }
    for (int h = lane; h < H; h += G) {
      real v = 0;
      if (mine0) { for (int n = 1; n <= n1; ++n) v += val[n * H + h] * sgs[(n - 1) * H + h]; }
      else       { for (int n = 1; n <= n1; ++n) v += val[n * H + h]; }
      val[h] = v;
    }
    group_sync();
    if (mine0) {
      for (int it = lane; it < n1 * H; it += G) {
        const int n = 1 + it / H, h = it % H;
        val[n * H + h] = (rsv[(n - 1) * H + h] + val[n * H + h]) - val[h];
      }
    }
    // ---- root value running mean (:579-590) and discounts (:592-617)
    const int s = s_steps;
    {
      const real alpha = p.linear ? (real)2 / (s + 2) : (real)1 / (s + 1);
      real* mu = p.mu + ((size_t)k * 2 + trav) * H;
      for (int h = lane; h < H; h += G) mu[h] += (val[h] - mu[h]) * alpha;
    }
    real pos = 1, neg = 1, strat = 1;
    {
      const real ns = (real)(s + 1);
      if (p.linear) {
        pos = neg = strat = ns / (ns + 1);
      } else if (p.dcfr) {
        pos = p.dcfr_alpha >= 5 ? (real)1 : rpow(ns, p.dcfr_alpha) / (rpow(ns, p.dcfr_alpha) + 1);
        neg = p.dcfr_beta <= -5 ? (real)0 : rpow(ns, p.dcfr_beta) / (rpow(ns, p.dcfr_beta) + 1);
        strat = rpow(ns / (ns + 1), p.dcfr_gamma);
      }
    }
    group_sync();
    // ---- regret matching (:619-634): per acting (node, hand) the sum of max(R, 1e-80) and its reciprocal
    real* rcp = rs;                                      // the staged regrets are dead: reuse the region, indexed like val's parents
    const real* bt = bel + trav * H;
    const int pb = mine0 ? 0 : 1, pe = mine0 ? 1 : lv.n1e;            // acting nodes
    const int cb = mine0 ? 1 : lv.n1e, ce = mine0 ? lv.n1e : lv.n2e;  // their children
    for (int it = lane; it < (pe - pb) * H; it += G) {
      const int n = pb + it / H, h = it % H;
      const int nc = nchild[n];
      if (!nc) continue;
      const int c0 = child_begin[n];
      real sum = 0;
      for (int j = 0; j < nc; ++j) {
        const real r = val[(c0 + j) * H + h];
        sum += Eps<real>::kLiteral ? (r > Eps<real>::v ? r : Eps<real>::v) : rmax0(r);   // max(R, 1e-80) (:626-629)
      }
      val[n * H + h] = sum;
      rcp[n * H + h] = (real)1 / sum;
    }
    group_sync();
    // ---- new strategy, regret discount and sum-strategy update (:639-661) on the traverser's level; the child's slot receives
    // belief * new strategy = the traverser's reach under the new strategy (:636-638), which the forward half reuses
    for (int it = lane; it < (ce - cb) * H; it += G) {
      const int c = cb + it / H, h = it % H;
      const int e = (c - 1) * H + h, par = parent[c];
      const real r = val[c * H + h], sum = val[par * H + h], rn = bt[h];
      const real sg = Eps<real>::kLiteral ? div_by_rcp(r > Eps<real>::v ? r : Eps<real>::v, sum, rcp[par * H + h])
                                          : (sum > 0 ? rmax0(r) / sum : (real)1 / nchild[par]);
      Sgg[e] = sg;
      Rg[e] = r * (r > 0 ? pos : neg);
      Sg_[e] = ssv[e] * strat + rn * sg;
      val[c * H + h] = rn * sg;
    }
    if (lane == 0) p.steps[2 * k + trav] = s + 1;
    group_sync();
  }
  // ---- sampling-strategy snapshot for RlRunner (recursive_solving.cc:168-174): state after `iter` iterations
  if (p.sg_act_iter[k] == iter) {
    real* __restrict__ Sn = p.Snap + (size_t)k * p.table_stride;
    for (int i = lane; i < E * H; i += G) Sn[i] = (do_b && i >= e0 * H && i < e1 * H) ? Sgg[i] : sgs[i];
  }
  if (!do_f) return;

  // ================= forward half of iteration `iter` (traverser tf) =================
  const int trav = tf;
  const int have = do_b ? (mine0 ? 0 : 1) : -1;        // level whose slots already hold belief * strategy
  if (have != 0) {
    const real* b0 = bel + rp * H;
    for (int it = lane; it < n1 * H; it += G) val[H + it] = b0[it % H] * sgs[it];
  }
  if (have != 1) {
    const real* b1 = bel + (1 - rp) * H;
    for (int it = lane; it < (lv.n2e - lv.n1e) * H; it += G) val[lv.n1e * H + it] = b1[it % H] * sgs[n1 * H + it];
  }
  group_sync();
  // Reach rows: the root player's reach at a level-2 node is its parent's level-1 slot, the other player's is the node's own
  // slot; at a level-1 node the root player's is the node's slot, the other player's is its root belief.
  real* hist = reinterpret_cast<real*>(io + Lo.io_hist);
  real* par_sum = reinterpret_cast<real*>(io + Lo.io_par);
  real* par_inv = par_sum + n1max;
  __half* qpar = reinterpret_cast<__half*>(io + Lo.io_qpar);
  __half* qown = reinterpret_cast<__half*>(io + Lo.io_qown);
  const int opp = 1 - trav;
  // ---- level-1 nodes: sum / normalisation of the root player's reach, shared by all leaves below the node (:257-265)
  for (int i = lane; i < n1; i += G) {
    const real* r = val + (1 + i) * H;
    real s0 = 0, e0s = 0;
    for (int h = 0; h < H; ++h) { s0 += r[h]; e0s += r[h] + Eps<real>::v; }
    const real inv = (real)1 / e0s;
    par_sum[i] = s0; par_inv[i] = inv;
    for (int h = 0; h < H; ++h) {
      float f;
      if (Eps<real>::kLiteral) f = (float)((r[h] + Eps<real>::v) * inv);                  // util.h:68-78
      else f = isfinite(inv) ? (float)(r[h] * inv) : 1.f / H;
      qpar[i * H + h] = __float2half_rn(f);
    }
  }
  group_sync();
  // ---- pseudo-leaves: the other player's sums, the scaler (sum of the opponent's reach, :264-268) and its fp16 columns
  for (int r = lane; r < t.L; r += G) {
    const int n = pleaf[r];
    const real* ro = val + n * H;
    real s1 = 0, e1s = 0;
    for (int h = 0; h < H; ++h) { s1 += ro[h]; e1s += ro[h] + Eps<real>::v; }
    const real inv = (real)1 / e1s;
    p.scaler[row0 + r] = (opp == rp) ? par_sum[parent[n] - 1] : s1;
    for (int h = 0; h < H; ++h) {
      float f;
      if (Eps<real>::kLiteral) f = (float)((ro[h] + Eps<real>::v) * inv);
      else f = isfinite(inv) ? (float)(ro[h] * inv) : 1.f / H;
      qown[r * H + h] = __float2half_rn(f);
    }
  }
  group_sync();
  // ---- query rows (write_query_to :104-123), fp16 tile in wgmma K-major core-matrix order, one 16-byte store per (row, 8
  // columns): constant columns from the per-template table, flags, and the two belief blocks from the fp16 values above
  const int leaf_player = rp ^ ((t.levels - 1) & 1);
  const int Qp = p.Qpad;
  if (p.Xh != nullptr) {
    const int kc = Qp >> 3;
    const int qb0 = 2 + p.A, qb1 = qb0 + H, qb2 = qb1 + H;
    const __half* __restrict__ qconst = p.qconst + t.qconst_off;
    for (int it = lane; it < t.L * kc; it += G) {
      const int k8 = it / t.L, r = it % t.L;
      union { int4 v; __half h[8]; } c;
      c.v = *reinterpret_cast<const int4*>(qconst + (size_t)r * Qp + k8 * 8);
      const int q0 = k8 * 8;
      if (q0 == 0) { c.h[0] = __float2half_rn((float)leaf_player); c.h[1] = __float2half_rn((float)trav); }
      if (q0 + 8 > qb0 && q0 < qb2) {
        const __half* mine = qown + r * H;                                   // player 1 - rp
        const __half* theirs = qpar + (parent[pleaf[r]] - 1) * H;            // player rp
        const __half* p0 = rp == 0 ? theirs : mine;
        const __half* p1 = rp == 0 ? mine : theirs;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int q = q0 + j;
          if (q >= qb0 && q < qb1) c.h[j] = p0[q - qb0];
          else if (q >= qb1 && q < qb2) c.h[j] = p1[q - qb1];
        }
      }
      const int Rr = row0 + r, rr = Rr & 127;
      *reinterpret_cast<int4*>(p.Xh + (size_t)(Rr >> 7) * 128 * Qp + k8 * 1024 + (rr >> 3) * 64 + (rr & 7) * 8) = c.v;
    }
  } else if (p.X != nullptr) {
    // fp32 parity net: the same columns in fp32, recomputed like generation 1 (this path is not the performance path)
    for (int it = lane; it < t.L * Qp; it += G) {
      const int r = it / Qp, q = it % Qp;
      const int n = pleaf[r];
      const real* r0 = d2_reach_row(val, bel, parent, n, lv.n1e, 0, rp, H);
      const real* r1 = d2_reach_row(val, bel, parent, n, lv.n1e, 1, rp, H);
      real s0 = 0, s1 = 0;
      for (int h = 0; h < H; ++h) { s0 += r0[h] + Eps<real>::v; s1 += r1[h] + Eps<real>::v; }
      p.X[(size_t)(row0 + r) * Qp + q] = query_value(p, q, leaf_player, trav, p.last_bid[t.node_off + n], r0, r1, (real)1 / s0, (real)1 / s1);
    }
  }
  // ---- terminals (compute_expected_terminal_values :80-98; win probability :765-789), as in cfr_forward_d2
  constexpr int kMaxBins = 9;
  real* __restrict__ vt = p.vterm + (size_t)k * p.vterm_stride;
  for (int z = lane; z < t.T; z += G) {
    const int n = term[z];
    const int face = term[t.T + z] % p.F;
    const real* ro = d2_reach_row(val, bel, parent, n, lv.n1e, opp, rp, H);
    real cnt[kMaxBins];
#pragma unroll
    for (int m = 0; m < kMaxBins; ++m) cnt[m] = 0;
    real tot = 0;
    for (int g = 0; g < H; ++g) {
      const real r = ro[g];
      const int mg = (int)p.matches[g * p.F + face];
      tot += r;
#pragma unroll
      for (int m = 0; m < kMaxBins; ++m) cnt[m] += (m == mg) ? r : (real)0;
    }
#pragma unroll
    for (int m = kMaxBins - 2; m >= 0; --m) cnt[m] += cnt[m + 1];
#pragma unroll
    for (int m = 0; m < kMaxBins; ++m) hist[z * (kMaxBins + 1) + m] = cnt[m];
    hist[z * (kMaxBins + 1) + kMaxBins] = tot;
  }
  group_sync();
  for (int it = lane; it < t.T * H; it += G) {
    const int z = it / H, h = it % H;
    const int pbid = term[t.T + z];
    const int ndepth = term[2 * t.T + z];
    const int quantity = 1 + pbid / p.F, face = pbid % p.F;
    int left = quantity - (int)p.matches[h * p.F + face];
    left = left < 0 ? 0 : (left > kMaxBins - 1 ? kMaxBins - 1 : left);
    const real win = hist[z * (kMaxBins + 1) + left], tot = hist[z * (kMaxBins + 1) + kMaxBins];
    const real v = (real)(float)win * 2 - tot;
    const int pl = rp ^ (ndepth & 1);
    vt[z * H + h] = (pl != trav) ? -v : v;
  }
}

}  // namespace cfrb
