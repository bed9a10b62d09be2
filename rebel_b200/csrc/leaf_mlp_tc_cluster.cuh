// Tensor-core value net on a cluster of two CTAs, for games whose Net2 weights do not fit one SM's shared memory (2x7f, 3x4f,
// 6x2f, 4x3f, 7x2f, 2x8f .. 2x11f, 3x5f, one-die games 1x33f .. 1x96f) -- and every smaller game, so that it can be compared
// with the resident and wide kernels.  Same Net2, fp16 operands, fp32 accumulation, mean-free fp32 LayerNorm and the fp32 tanh
// GELU (kGelu 2, CFRB_NET_TC_F16X2's default) as leaf_mlp_tc.cuh, whose helpers it reuses.
//
// Feature split.  CTA r of the cluster keeps, for the kernel's lifetime, hidden features [128 r, 128 r + 128): those rows of W1
// (bias column included) and of W2 (at full K = 256), its half of the output columns of W3 (at full K), and its halves of bias 2,
// the LayerNorm parameters and bias 3 (ClusterLayout).  Both CTAs take the same 128-row query tiles; warpgroup w of each runs
// rows 64w .. 64w + 63 of a tile, so a warpgroup's partner is the warpgroup w of the other CTA, which holds the same rows.
//
// Exchange protocol, per warpgroup and tile (a layer's accumulators are this CTA's 128 features of the warpgroup's 64 rows):
//   * LayerNorm: the host centres W1 / W2 and the biases over all 256 features, so the row mean is zero by construction.  Each
//     warpgroup writes its per-row sum of squares into the partner's `ss` slot (st.shared::cluster) and both add the two halves in
//     rank order, so both CTAs compute the same 1 / std.
//   * Activations: after its epilogue a warpgroup writes its 128 fp16 features of the 64 rows into the partner's `xa` buffer, in
//     the A-fragment order of the next wgmma (K-step i, thread lt: 16 bytes at [i][lt]), so the partner reads its own fragments back
//     with one 16-byte load per K-step.  The next layer then takes its own eight K-steps from registers and the partner's eight
//     from those loads: own features first, then the partner's (the order of the K-steps is fixed per CTA, so the results do not
//     depend on which tiles a cluster takes).
//   * Every write is followed by a remote mbarrier arrival with release semantics at cluster scope (128 per exchange); the reader
//     waits with acquire at cluster scope.  The two exchanges alternate on two mbarriers per warpgroup (ss: bar_ss, activations:
//     bar_xa), two phases of each per tile.  No "empty" barrier is needed: a warpgroup writes a buffer again only after it has
//     received the partner's next exchange, which the partner sends only after it has read that buffer.  Nor can a barrier run two
//     phases ahead of its reader: the partner's next exchange on the same barrier needs this warpgroup's exchange in between.
//
// Both CTAs of a cluster read the same row count and take the same tiles, so they leave together; every CTA passes a final
// cluster barrier, so none exits while its partner may still write into its shared memory.
#pragma once
#include "leaf_mlp_tc_wide.cuh"

namespace cfrb {
namespace tc {

constexpr int kClusterCtas = 2;
constexpr int kHalfHid = kHid / kClusterCtas;   // hidden features per CTA
constexpr int kClusterKChunk = 8;               // layer-1 K-steps loaded into registers at once (Kp is unbounded here)

// Shared memory of one CTA (bytes).  The weight blob in global memory is the two CTAs' blobs one after the other, each exactly the
// smem layout up to blob_bytes.  Nh = output columns per CTA: roundup(H, 32) / 2, at most 64.
struct ClusterLayout {
  int Kp, Nh;
  int off_w1, off_w2, off_w3, off_b2, off_ln1, off_ln2, off_b3, blob_bytes, off_xa, off_ss, off_bar, smem_bytes;
  __host__ __device__ ClusterLayout(int kp, int nh) : Kp(kp), Nh(nh) {
    off_w1 = 0;                                   // [128 x Kp]  fp16, column Q holds bias 1
    off_w2 = off_w1 + kHalfHid * kp * 2;          // [128 x 256] fp16
    off_w3 = off_w2 + kHalfHid * kHid * 2;        // [Nh x 256]  fp16
    off_b2 = off_w3 + nh * kHid * 2;              // float [128]
    off_ln1 = off_b2 + kHalfHid * 4;              // float4 {gamma_j, gamma_j+1, beta_j, beta_j+1} per feature pair
    off_ln2 = off_ln1 + kHalfHid * 8;
    off_b3 = off_ln2 + kHalfHid * 8;              // float [Nh]
    blob_bytes = off_b3 + nh * 4;                 // a multiple of 16 (Nh a multiple of 16): the second CTA's blob stays aligned
    off_xa = (blob_bytes + 127) / 128 * 128;      // per warpgroup [8 K-steps][128 threads] x 16 B: the partner's activations
    off_ss = off_xa + 2 * 8 * 128 * 16;           // per warpgroup float [64]: the partner's per-row sums of squares
    off_bar = off_ss + 2 * kWgRows * 4;           // mbarriers: weights, bar_ss[2], bar_xa[2]
    smem_bytes = off_bar + 5 * 8;
  }
};
__host__ __device__ inline int cluster_nh(int H) { return (H + 31) / 32 * 32 / 2; }

// ---------------------------------------------------------------- cluster PTX
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_id_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%clusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_count_x() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%nclusterid.x;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// The shared::cluster address of the same offset in CTA `rank`'s shared memory.
__device__ __forceinline__ uint32_t map_peer(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_u4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared::cluster.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) {
  asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "CWAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra CWAIT_DONE;\n\t"
      "bra CWAIT_LOOP;\n\t"
      "CWAIT_DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}

// Per-row sums of squares of a warpgroup's 64 x 128 accumulators (rows r, r + 8 of the thread), reduced over the quad.
__device__ __forceinline__ void half_sumsq(const float (&acc)[64], float& lo, float& hi) {
  float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int c = (i & 1) * 2;
    s[c] = fmaf(acc[4 * i], acc[4 * i], s[c]);
    s[c] = fmaf(acc[4 * i + 1], acc[4 * i + 1], s[c]);
    s[c + 1] = fmaf(acc[4 * i + 2], acc[4 * i + 2], s[c + 1]);
    s[c + 1] = fmaf(acc[4 * i + 3], acc[4 * i + 3], s[c + 1]);
  }
  lo = s[0] + s[2];
  hi = s[1] + s[3];
  lo += __shfl_xor_sync(0xffffffffu, lo, 1);
  hi += __shfl_xor_sync(0xffffffffu, hi, 1);
  lo += __shfl_xor_sync(0xffffffffu, lo, 2);
  hi += __shfl_xor_sync(0xffffffffu, hi, 2);
}
// LayerNorm affine + GELU of the 128 features, given 1 / std of the two rows: A fragments act[4i .. 4i+3] of K-step i (0 .. 7).
__device__ __forceinline__ void half_affine_gelu(const float (&acc)[64], const float4* __restrict__ ln, int q, float rstd_lo,
                                                 float rstd_hi, uint32_t (&act)[32]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float4 pp = ln[i * 4 + q];
    act[2 * i] = act_pair<2>(__fmaf_rn(__fmul_rn(acc[4 * i], rstd_lo), pp.x, pp.z), __fmaf_rn(__fmul_rn(acc[4 * i + 1], rstd_lo), pp.y, pp.w));
    act[2 * i + 1] = act_pair<2>(__fmaf_rn(__fmul_rn(acc[4 * i + 2], rstd_hi), pp.x, pp.z),
                                 __fmaf_rn(__fmul_rn(acc[4 * i + 3], rstd_hi), pp.y, pp.w));
  }
}

// Output layer of one CTA: kNh columns as one chain (16, 32, 48) or two (64 = 48 + 16).
template <int kNh>
struct OutChains {
  static constexpr int N1 = kNh > 48 ? 48 : kNh, N2 = kNh - N1;
  static_assert(kNh % 16 == 0 && kNh >= 16 && kNh <= 64, "output columns per CTA: 16, 32, 48 or 64");
  float o1[N1 / 2];
  float o2[N2 > 0 ? N2 / 2 : 1];
};

template <int kNh>
__global__ void __launch_bounds__(kThreads, 1) leaf_mlp_tc_cluster_kernel(TcArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const ClusterLayout L(a.Kp, kNh);
  const int tid = threadIdx.x, wg = __shfl_sync(0xffffffffu, tid >> 7, 0), lt = tid & 127, warp = lt >> 5, lane = tid & 31;
  const uint32_t rank = __shfl_sync(0xffffffffu, cluster_ctarank(), 0), peer = rank ^ 1u;
  const int ksteps = a.Kp / 16;

  const uint32_t bar_w = smem_u32(smem + L.off_bar), bar_ss = bar_w + 8 + 8 * wg, bar_xa = bar_w + 24 + 8 * wg;
  if (tid == 0) {
    mbar_init(bar_w, 1);
    for (int w = 0; w < 2; ++w) { mbar_init(bar_w + 8 + 8 * w, 128); mbar_init(bar_w + 24 + 8 * w, 128); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // weights of this CTA's half: fetched while the CFR kernel before this launch drains (programmatic dependent launch)
  if (tid == 0) {
    const uint8_t* src = a.blob + (size_t)rank * L.blob_bytes;
    mbar_expect_tx(bar_w, (uint32_t)L.blob_bytes);
    for (int o = 0; o < L.blob_bytes; o += 32768) bulk_g2s(smem_u32(smem + o), src + o, (uint32_t)min(32768, L.blob_bytes - o), bar_w);
  }
  cluster_sync();                                 // both CTAs' mbarriers are initialised before any remote arrival
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;");
  const int rows = __shfl_sync(0xffffffffu, *a.rows_ptr, 0);
  const int ntiles = (rows + kTileM - 1) / kTileM;
  const int cl = (int)cluster_id_x(), ncl = (int)cluster_count_x();
  const int J = cl < ntiles ? (ntiles - 1 - cl) / ncl + 1 : 0;   // tiles of this cluster: cl + j * ncl (the same for both CTAs)
  mbar_wait(bar_w, 0);

  const uint32_t sw1 = smem_u32(smem + L.off_w1), sw2 = smem_u32(smem + L.off_w2), sw3 = smem_u32(smem + L.off_w3);
  const float4* ln1 = reinterpret_cast<const float4*>(smem + L.off_ln1);
  const float4* ln2 = reinterpret_cast<const float4*>(smem + L.off_ln2);
  const float* b2 = reinterpret_cast<const float*>(smem + L.off_b2);
  const float* b3 = reinterpret_cast<const float*>(smem + L.off_b3);
  const int q = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);
  const uint32_t lbo_w = (kHalfHid / 8) * 128, lbo_w3 = (kNh / 8) * 128;
  // exchange slots: what the partner writes here (own, read back) and where this warpgroup writes (the partner's, remote)
  const uint32_t xa_own = smem_u32(smem + L.off_xa) + (uint32_t)(wg * 8 * 128 + lt) * 16u;
  const uint32_t xa_peer = map_peer(xa_own, peer);
  float* ss_own = reinterpret_cast<float*>(smem + L.off_ss) + wg * kWgRows;
  const uint32_t ss_peer = map_peer(smem_u32(ss_own), peer);
  const uint32_t bar_ss_peer = map_peer(bar_ss, peer), bar_xa_peer = map_peer(bar_xa, peer);
  const uint32_t* xw = reinterpret_cast<const uint32_t*>(a.Xh) + wg * 256 + warp * 64 + lane;
  const int tile_words = kTileM * a.Kp / 2;

  float acc[64];
  uint32_t act[32], pa[32];
  uint32_t xa[4 * kClusterKChunk];

  // 1 / std of the thread's two rows from its own half's sums of squares and the partner's (phase `ph` of bar_ss); the sum is
  // taken in rank order, so both CTAs get the same bits
  auto layer_norm_scale = [&](uint32_t ph, float& rstd_lo, float& rstd_hi) {
    float lo, hi;
    half_sumsq(acc, lo, hi);
    if (q == 0) { st_cluster_f32(ss_peer + 4u * r_lo, lo); st_cluster_f32(ss_peer + 4u * (r_lo + 8), hi); }
    mbar_arrive_remote(bar_ss_peer);
    mbar_wait_cluster(bar_ss, ph);
    const float plo = ss_own[r_lo], phi = ss_own[r_lo + 8];
    const float tlo = rank == 0 ? lo + plo : plo + lo, thi = rank == 0 ? hi + phi : phi + hi;
    rstd_lo = rsqrtf(tlo * (1.f / kHid) + 1e-5f);
    rstd_hi = rsqrtf(thi * (1.f / kHid) + 1e-5f);
  };
  // this warpgroup's activations to the partner, the partner's into pa (phase `ph` of bar_xa)
  auto exchange_act = [&](uint32_t ph) {
#pragma unroll
    for (int i = 0; i < 8; ++i) st_cluster_u4(xa_peer + i * 128 * 16, act[4 * i], act[4 * i + 1], act[4 * i + 2], act[4 * i + 3]);
    mbar_arrive_remote(bar_xa_peer);
    mbar_wait_cluster(bar_xa, ph);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const uint4 v = *reinterpret_cast<const uint4*>(smem + L.off_xa + (size_t)(wg * 8 * 128 + lt) * 16 + i * 128 * 16);
      pa[4 * i] = v.x; pa[4 * i + 1] = v.y; pa[4 * i + 2] = v.z; pa[4 * i + 3] = v.w;
    }
  };
  // the layer-2 turns of leaf_mlp_tc_kernel: warpgroup 0 takes J - 1 turns and passes J, warpgroup 1 takes J and passes J - 1
  auto take_turn = [&] { asm volatile("bar.sync %0, 256;" ::"r"(kBarTurn + wg) : "memory"); };
  auto pass_turn = [&] { asm volatile("bar.arrive %0, 256;" ::"r"(kBarTurn + (wg ^ 1)) : "memory"); };
  const uint32_t k_own = rank * 8, k_peer = peer * 8;   // K-steps of layers 2 and 3 fed by this CTA's / the partner's features

  for (int j = 0; j < J; ++j) {
    const int tile = cl + j * ncl;
    const uint32_t* xt = xw + (size_t)tile * tile_words;
    // ---- layer 1: D1 = X W1'^T for this CTA's 128 features, A from the query tile in chunks of kClusterKChunk K-steps
    for (int k0 = 0; k0 < ksteps; k0 += kClusterKChunk) {
#pragma unroll
      for (int kk = 0; kk < kClusterKChunk; ++kk) {
        const bool in = k0 + kk < ksteps;
        const uint32_t* p = xt + (k0 + kk) * 1024;
        xa[4 * kk] = in ? p[0] : 0u;
        xa[4 * kk + 1] = in ? p[32] : 0u;
        xa[4 * kk + 2] = in ? p[512] : 0u;
        xa[4 * kk + 3] = in ? p[544] : 0u;
      }
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kClusterKChunk; ++kk)
        if (k0 + kk < ksteps) wgmma_rs_n128_sd(acc, xa + 4 * kk, make_desc(sw1 + (k0 + kk) * 2 * lbo_w, lbo_w, 128), k0 + kk > 0);
      wgmma_commit();
      wgmma_wait_all();
      fence_regs(acc); fence_regs(xa);
    }
    if (wg == 1 && j == 0) take_turn();
    float rlo, rhi;
    layer_norm_scale(0, rlo, rhi);
    half_affine_gelu(acc, ln1, q, rlo, rhi, act);
    exchange_act(0);
    // ---- layer 2: D2 = bias2 + A2 W2'^T, own K-steps from act, the partner's from pa
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float2 bb = *reinterpret_cast<const float2*>(b2 + i * 8 + 2 * q);
      acc[4 * i] = bb.x; acc[4 * i + 1] = bb.y; acc[4 * i + 2] = bb.x; acc[4 * i + 3] = bb.y;
    }
    if (j > 0) take_turn();
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < 8; ++i) wgmma_rs_n128(acc, act + 4 * i, make_desc(sw2 + (k_own + i) * 2 * lbo_w, lbo_w, 128));
#pragma unroll
    for (int i = 0; i < 8; ++i) wgmma_rs_n128(acc, pa + 4 * i, make_desc(sw2 + (k_peer + i) * 2 * lbo_w, lbo_w, 128));
    wgmma_commit();
    if (wg == 0 || j + 1 < J) pass_turn();
    int dst[2];                                   // output rows of this thread's two rows (row_src: compacted tiles), -1 = none
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int row = tile * kTileM + wg * kWgRows + r_lo + 8 * e;
      dst[e] = row < rows ? (a.row_src != nullptr ? __ldg(a.row_src + row) : row) : -1;
    }
    wgmma_wait_all();
    fence_regs(acc); fence_regs(act); fence_regs(pa);
    // ---- epilogue 2 and layer 3: this CTA's kNh output columns at full K
    layer_norm_scale(1, rlo, rhi);
    half_affine_gelu(acc, ln2, q, rlo, rhi, act);
    exchange_act(1);
    OutChains<kNh> oc;
    constexpr int N1 = OutChains<kNh>::N1, N2 = OutChains<kNh>::N2;
#pragma unroll
    for (int i = 0; i < N1 / 2; ++i) oc.o1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (N2 > 0 ? N2 / 2 : 1); ++i) oc.o2[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const uint32_t* f = i < 8 ? act + 4 * i : pa + 4 * (i - 8);
      const uint32_t kk = i < 8 ? k_own + i : k_peer + i - 8;
      wgmma_rs_out<N1>(oc.o1, f, make_desc(sw3 + kk * 2 * lbo_w3, lbo_w3, 128));
      if constexpr (N2 > 0) wgmma_rs_out<N2>(oc.o2, f, make_desc(sw3 + kk * 2 * lbo_w3 + (N1 / 8) * 128, lbo_w3, 128));
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(oc.o1); fence_regs(oc.o2); fence_regs(act); fence_regs(pa);
    const int c0 = (int)rank * kNh;               // first output column of this CTA
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (dst[e] >= 0) {                          // rows are Hout floats apart, Hout a multiple of 4
        float* orow = a.out + (size_t)dst[e] * a.Hout;
#pragma unroll
        for (int i = 0; i < N1 / 8; ++i) {
          const int c = i * 8 + 2 * q;
          if (c0 + c < a.Hout) *reinterpret_cast<float2*>(orow + c0 + c) = make_float2(oc.o1[4 * i + 2 * e] + b3[c], oc.o1[4 * i + 2 * e + 1] + b3[c + 1]);
        }
        if constexpr (N2 > 0) {
#pragma unroll
          for (int i = 0; i < N2 / 8; ++i) {
            const int c = N1 + i * 8 + 2 * q;
            if (c0 + c < a.Hout) *reinterpret_cast<float2*>(orow + c0 + c) = make_float2(oc.o2[4 * i + 2 * e] + b3[c], oc.o2[4 * i + 2 * e + 1] + b3[c + 1]);
          }
        }
      }
    }
  }
  cluster_sync();                                 // no CTA leaves while its partner may still write into its shared memory
}

// Host side (leaf_mlp_tc_cluster.cu): the instantiations for Nh = 16, 32, 48, 64.
cudaError_t cluster_configure(int nh, int smem_bytes, int* max_clusters);
cudaError_t cluster_launch(const cudaLaunchConfig_t& lc, const TcArgs& a, int nh);

}  // namespace tc
}  // namespace cfrb
