// Tensor-core value net for games whose weights leave no room for query tiles in shared memory (more than 16 hands: 2x5f, 3x3f,
// 5x2f, 2x6f, one-die games up to 1x32f).  Same Net2, same fp16 operands, fp32 accumulation and epilogues as leaf_mlp_tc_kernel
// (leaf_mlp_tc.cuh, whose helpers it reuses); two things differ:
//
//   * the output layer is one m64nNk16 chain with N = kNo = roundup(H, 16) columns (16, 32 or 48), W3 stored with kNo rows;
//   * layer 1 is an RS wgmma: each thread loads its A fragments straight from the query tiles in global memory (Xh, written by
//     the CFR forward kernel in K-major core-matrix order) into registers.  A fragment of K-step kk is (row g, cols 2q, 2q+1),
//     (g + 8, same), (g, 8 + 2q ..), (g + 8, 8 + 2q ..): four 4-byte loads, and across a warp each of them reads exactly one
//     128-byte core matrix, so they coalesce.  No query buffers, refill counter or per-tile mbarrier: shared memory holds the
//     weights only, W1 [256 x Kp] + W2 + W3 [kNo x 256] + 5 KB of biases and LayerNorm parameters (WideLayout).
//
// Layer 1 accumulates over K in the order of the SS form of leaf_mlp_tc_kernel, layers 2 and 3 are issued the same way, so on a
// shape both kernels accept (H <= 16, kNo = 16) the outputs are bit-identical.  The two warpgroups keep the layer-2 turns of
// leaf_mlp_tc_kernel (one warpgroup's loads and epilogues run under the other's MMAs).
#pragma once
#include "leaf_mlp_tc.cuh"

namespace cfrb {
namespace tc {

constexpr int kWideMaxKSteps = 10;        // layer-1 K-steps held in registers: Kp <= 160
constexpr int kSmemOptinSm90 = 232448;    // dynamic shared memory a block may opt into on sm_90 (227 KB)

struct WideLayout {
  int Kp, Nout;
  int off_w1, off_w2, off_w3, off_b2, off_ln1, off_ln2, off_b3, blob_bytes, off_bar, smem_bytes;
  __host__ __device__ WideLayout(int kp, int nout) : Kp(kp), Nout(nout) {
    off_w1 = 0;                               // [256 x Kp]   fp16, column Q holds bias 1
    off_w2 = off_w1 + kHid * kp * 2;          // [256 x 256]  fp16
    off_w3 = off_w2 + kHid * kHid * 2;        // [Nout x 256] fp16
    off_b2 = off_w3 + nout * kHid * 2;        // float [256]
    off_ln1 = off_b2 + kHid * 4;              // float4 {gamma_j, gamma_j+1, beta_j, beta_j+1} per feature pair
    off_ln2 = off_ln1 + kHid * 8;
    off_b3 = off_ln2 + kHid * 8;              // float [Nout]
    blob_bytes = off_b3 + nout * 4;
    off_bar = (blob_bytes + 15) / 16 * 16;    // mbarrier of the weight copy
    smem_bytes = off_bar + 8;
  }
};

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, A in registers; scale_d = 0 overwrites D (the first K-step of layer 1).
__device__ __forceinline__ void wgmma_rs_n128_sd(float (&d)[64], const uint32_t* a, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(scale_d));
}
// D[64 x 32] += A[64 x 16] * B[32 x 16]^T, A in registers.
__device__ __forceinline__ void wgmma_rs_n32(float (&d)[16], const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1u));
}
// D[64 x 48] += A[64 x 16] * B[48 x 16]^T, A in registers.
__device__ __forceinline__ void wgmma_rs_n48(float (&d)[24], const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1u));
}
template <int kNo>
__device__ __forceinline__ void wgmma_rs_out(float (&d)[kNo / 2], const uint32_t* a, uint64_t b_desc) {
  static_assert(kNo == 16 || kNo == 32 || kNo == 48, "output layer: N = 16, 32 or 48");
  if constexpr (kNo == 16) wgmma_rs_n16(d, a, b_desc);
  else if constexpr (kNo == 32) wgmma_rs_n32(d, a, b_desc);
  else wgmma_rs_n48(d, a, b_desc);
}

template <bool kDebug, int kGelu, int kNo>
__global__ void __launch_bounds__(kThreads, 1) leaf_mlp_tc_wide_kernel(TcArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const WideLayout L(a.Kp, kNo);
  // warp-uniform through a shuffle, as in leaf_mlp_tc_kernel: branches on wg do not serialise the wgmmas
  const int tid = threadIdx.x, wg = __shfl_sync(0xffffffffu, tid >> 7, 0), lt = tid & 127, warp = lt >> 5, lane = tid & 31;
  const int ksteps = a.Kp / 16;

  const uint32_t bar_w = smem_u32(smem + L.off_bar);
  if (tid == 0) {
    mbar_init(bar_w, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // weights: fetched while the CFR kernel before this launch drains (programmatic dependent launch); the query rows are read
  // only after griddepcontrol.wait
  if (tid == 0) {
    mbar_expect_tx(bar_w, (uint32_t)L.blob_bytes);
    for (int o = 0; o < L.blob_bytes; o += 32768)
      bulk_g2s(smem_u32(smem + o), a.blob + o, (uint32_t)min(32768, L.blob_bytes - o), bar_w);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;");
  // the row count may come from the CFR kernel before this launch (compacted query tiles): read only after the wait.  A CTA
  // without tiles lets its weight copy land before it exits.
  const int rows = __shfl_sync(0xffffffffu, *a.rows_ptr, 0);
  const int ntiles = (rows + kTileM - 1) / kTileM;
  if ((int)blockIdx.x >= ntiles) {
    mbar_wait(bar_w, 0);
    return;
  }
  const int J = (ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1;      // tiles of this CTA: blockIdx.x + j * gridDim.x
  mbar_wait(bar_w, 0);

  const uint32_t sw1 = smem_u32(smem + L.off_w1), sw2 = smem_u32(smem + L.off_w2), sw3 = smem_u32(smem + L.off_w3);
  const float4* ln1 = reinterpret_cast<const float4*>(smem + L.off_ln1);
  const float4* ln2 = reinterpret_cast<const float4*>(smem + L.off_ln2);
  const float* b2 = reinterpret_cast<const float*>(smem + L.off_b2);
  const float* b3 = reinterpret_cast<const float*>(smem + L.off_b3);
  const int q = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);     // this thread's rows within the warpgroup's 64: r_lo and r_lo + 8
  const uint32_t lbo_w = (kHid / 8) * 128, lbo_w3 = (kNo / 8) * 128;
  // A fragments of layer 1 in the tile's K-major core-matrix order (umma_kmajor_offset_halves with R = 128), in 32-bit words:
  // K-step kk starts at kk * 1024; the thread's core matrices at (wg * 8 + warp * 2) * 32, word lane within each; + 32 for rows
  // g + 8, + 512 for columns 8 .. 15 of the step
  const uint32_t* xw = reinterpret_cast<const uint32_t*>(a.Xh) + wg * 256 + warp * 64 + lane;
  const int tile_words = kTileM * a.Kp / 2;
  auto tile_of = [&](int j) { return (int)blockIdx.x + j * (int)gridDim.x; };
  float acc[2][64];
  uint32_t act[64];
  uint32_t xa[4 * kWideMaxKSteps];

#define CFRB_TRACE(e)                                                                                 \
  do {                                                                                                \
    if (kDebug && a.trace && blockIdx.x == 0 && lt == 0 && j < 64) a.trace[wg * 1024 + j * 8 + (e)] = clock64(); \
  } while (0)
  auto tap = [&](float* dbg, int tile) {        // raw accumulators of tile 0 (debug build)
    if (kDebug && dbg && tile == 0) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 16; ++i)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            dbg[(wg * kWgRows + r_lo + (e >> 1) * 8) * kHid + h * 128 + i * 8 + 2 * q + (e & 1)] = acc[h][4 * i + e];
    }
  };
  // layer-2 turns exactly as in leaf_mlp_tc_kernel (see there): warpgroup 0 takes J - 1 turns and passes J, warpgroup 1 takes J
  // (its first before epilogue 1 of its first tile) and passes J - 1
  auto take_turn = [&] { asm volatile("bar.sync %0, 256;" ::"r"(kBarTurn + wg) : "memory"); };
  auto pass_turn = [&] { asm volatile("bar.arrive %0, 256;" ::"r"(kBarTurn + (wg ^ 1)) : "memory"); };

  for (int j = 0; j < J; ++j) {
    const int tile = tile_of(j);
    const uint32_t* xt = xw + (size_t)(tile * tile_words);
    // (fragments past Kp are set, not left over from the previous tile: nothing is carried from one tile to the next)
#pragma unroll
    for (int kk = 0; kk < kWideMaxKSteps; ++kk) {
      const bool in = kk < ksteps;
      xa[4 * kk] = in ? xt[kk * 1024] : 0u;
      xa[4 * kk + 1] = in ? xt[kk * 1024 + 32] : 0u;
      xa[4 * kk + 2] = in ? xt[kk * 1024 + 512] : 0u;
      xa[4 * kk + 3] = in ? xt[kk * 1024 + 544] : 0u;
    }
    CFRB_TRACE(0);
    // ---- layer 1: D1 = X W1'^T (bias 1 through the constant-1 query column), A from registers
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kWideMaxKSteps; ++kk)
      if (kk < ksteps) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          wgmma_rs_n128_sd(acc[h], xa + 4 * kk, make_desc(sw1 + kk * 2 * lbo_w + h * 2048, lbo_w, 128), kk > 0);
      }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(acc[0]); fence_regs(acc[1]);
    tap(a.dbg_d1, tile);
    CFRB_TRACE(1);
    if (wg == 1 && j == 0) take_turn();
    ln_gelu<kGelu>(acc, ln1, q, act);
    CFRB_TRACE(2);
    // ---- layer 2: D2 = bias2 + A2 W2'^T, A2 from registers
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float2 bb = *reinterpret_cast<const float2*>(b2 + h * 128 + i * 8 + 2 * q);
        acc[h][4 * i] = bb.x; acc[h][4 * i + 1] = bb.y; acc[h][4 * i + 2] = bb.x; acc[h][4 * i + 3] = bb.y;
      }
    if (j > 0) take_turn();
    CFRB_TRACE(3);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kHid / 16; ++kk) {
#pragma unroll
      for (int h = 0; h < 2; ++h) wgmma_rs_n128(acc[h], act + 4 * kk, make_desc(sw2 + kk * 2 * lbo_w + h * 2048, lbo_w, 128));
    }
    wgmma_commit();
    if (wg == 0 || j + 1 < J) pass_turn();
    CFRB_TRACE(4);
    int dst[2];                                 // output rows of this thread's two rows (row_src: compacted tiles), -1 = none
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int row = tile * kTileM + wg * kWgRows + r_lo + 8 * e;
      dst[e] = row < rows ? (a.row_src != nullptr ? __ldg(a.row_src + row) : row) : -1;
    }
    wgmma_wait_all();
    fence_regs(acc[0]); fence_regs(acc[1]); fence_regs(act);
    tap(a.dbg_d2, tile);
    CFRB_TRACE(5);
    // ---- epilogue 2 and layer 3: each half of the m64nNk16 chain is issued as soon as epilogue 2 has produced its A fragments
    float o[kNo / 2];
#pragma unroll
    for (int i = 0; i < kNo / 2; ++i) o[i] = 0.f;
    ln_gelu<kGelu>(acc, ln2, q, act, [&](int h) {
      wgmma_fence();
#pragma unroll
      for (int kk = 8 * h; kk < 8 * h + 8; ++kk) wgmma_rs_out<kNo>(o, act + 4 * kk, make_desc(sw3 + kk * 2 * lbo_w3, lbo_w3, 128));
    });
    wgmma_commit();
    CFRB_TRACE(6);
    wgmma_wait_all();
    fence_regs(o); fence_regs(act);
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (dst[e] >= 0) {                        // rows are Hout floats apart, Hout a multiple of 4
        float* orow = a.out + (size_t)dst[e] * a.Hout;
#pragma unroll
        for (int i = 0; i < kNo / 8; ++i) {
          const int c = i * 8 + 2 * q;
          if (c < a.Hout) *reinterpret_cast<float2*>(orow + c) = make_float2(o[4 * i + 2 * e] + b3[c], o[4 * i + 2 * e + 1] + b3[c + 1]);
        }
      }
    }
    CFRB_TRACE(7);
  }
#undef CFRB_TRACE
}

// Host side (leaf_mlp_tc_wide.cu): the instantiations for kNo = 16, 32, 48 live in their own translation unit.
cudaError_t wide_configure(int nout, int smem_bytes);
cudaError_t wide_launch(const cudaLaunchConfig_t& lc, const TcArgs& a, int nout, int gelu, bool dbg);

}  // namespace tc
}  // namespace cfrb
