// Tensor-core evaluation of the leaf value net (Net2: Linear -> LayerNorm -> GELU -> Linear -> LayerNorm -> GELU -> Linear,
// cfvpy/models.py:64-94) for all pseudo-leaf query rows of a wave — the one dense contraction of the CFR hot path and,
// at 148k FLOP per row, its dominant cost.  Hopper-native: wgmma.mma_async (fp16 operands, fp32 accumulation in registers),
// weights resident in shared memory for the lifetime of a persistent CTA, activations never leave the registers:
//
//   X tile [128 x Kp] fp16 (smem, K-major core-matrix order, written in that order by the CFR forward kernel; bulk-copied,
//   double-buffered)
//     --wgmma SS-->  D1 [64 x 256] fp32 per warpgroup (two m64n128k16 halves, 128 registers per thread)
//     --epilogue (LayerNorm, GELU, -> fp16 A fragments in registers)-->
//     --wgmma RS (A from registers, W2 from smem; accumulators preloaded with bias 2)-->  D2 [64 x 256]
//     --epilogue-->  --wgmma RS (N = 16)-->  D3 [64 x 16]  --(+ bias 3)-->  out[rows][Hout] fp32
//
// CTA = two warpgroups; warpgroup w owns rows 64w..64w+63 of every 128-row tile and runs all three layers of them on its own,
// so the tensor cores work for one warpgroup while the other one is in its epilogue.  The fp32 accumulator fragment of a
// wgmma is, converted to fp16, exactly the A-register fragment of the next one (a thread holds two rows and, per 8 columns, a
// column pair), so LayerNorm is a reduction over the four threads of a quad and nothing goes through shared memory.
// Bias 1 rides on the tensor cores through a constant-1 query column (written by the CFR kernel) against a bias column in W1.
//
// LayerNorm without the mean: the rows of W1 / W2 and the biases are centred over the 256 output features on the host
// (W'[j][k] = W[j][k] - mean_j W[j][k]), so sum_j y_j = 0 by construction and LayerNorm needs only sum_j y_j^2.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace cfrb {
namespace tc {

constexpr int kHid = 256;
constexpr int kTileM = 128;               // rows of a query tile (the CFR kernel writes tiles of this height)
constexpr int kWgRows = 64;               // rows per warpgroup (wgmma M)
constexpr int kNout = 16;                 // output features padded to a wgmma N
constexpr int kThreads = 2 * 128;         // two warpgroups

// ---- shared-memory / weight-blob layout (bytes).  The blob in global memory has exactly the smem layout up to off_x.
struct BlobLayout {
  int Kp;            // padded query width (multiple of 16, with at least one spare column for the constant 1)
  int off_w1, off_w2, off_w3, off_b2, off_ln1, off_ln2, off_b3, blob_bytes, x_bytes, off_x, off_xcnt, off_bar, smem_bytes;
  __host__ __device__ explicit BlobLayout(int kp) : Kp(kp) {
    off_w1 = 0;                               // [256 x Kp]  fp16, column Q holds bias 1
    off_w2 = off_w1 + kHid * kp * 2;          // [256 x 256] fp16
    off_w3 = off_w2 + kHid * kHid * 2;        // [16 x 256]  fp16
    off_b2 = off_w3 + kNout * kHid * 2;       // float [256]: bias 2 (rounded to fp16 like the weights)
    off_ln1 = off_b2 + kHid * 4;              // float4 {gamma_j, gamma_j+1, beta_j, beta_j+1} per feature pair
    off_ln2 = off_ln1 + kHid * 8;
    off_b3 = off_ln2 + kHid * 8;
    blob_bytes = off_b3 + kNout * 4;
    x_bytes = kTileM * kp * 2;
    off_x = (blob_bytes + 127) / 128 * 128;   // two query-tile buffers
    off_xcnt = off_x + 2 * x_bytes;           // per buffer: warpgroups done with it (monotonic)
    off_bar = off_xcnt + 16;                  // mbarriers: weights, x[0], x[1]
    smem_bytes = off_bar + 3 * 8;
  }
};

// Element (row r, col k) of a K-major [R x K] fp16 operand in the no-swizzle core-matrix order of wgmma:
// 8x8 core matrices of 128 contiguous bytes; row-groups are 128 B apart (SBO), K-chunks R/8*128 B apart (LBO).
__host__ __device__ inline int umma_kmajor_offset_halves(int r, int k, int R) {
  return (k >> 3) * (R >> 3) * 64 + (r >> 3) * 64 + (r & 7) * 8 + (k & 7);
}

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bulk copy global -> shared (the TMA engine without a tensor map); completion is signalled on the mbarrier as transaction bytes.
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(gsrc),
               "r"(bytes), "r"(bar) : "memory");
}

// wgmma shared-memory matrix descriptor, K-major, no swizzle: start>>4 [0,14), LBO>>4 [16,30) (between the two K core
// matrices of a K=16 step), SBO>>4 [32,46) (between 8-row groups), layout type 0 [62,64).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Keeps the compiler from moving register reads / writes across the asynchronous wgmma (issue ... wait) window.
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N>
__device__ __forceinline__ void fence_regs(uint32_t (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

// D[64 x 128] (+)= A[64 x 16] * B[128 x 16]^T, A and B in shared memory (descriptors); scale_d = 0 overwrites D.
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a_desc), "l"(b_desc), "r"(scale_d));
}
// D[64 x 128] += A[64 x 16] * B[128 x 16]^T, A in registers (the accumulator layout of the previous layer, packed to fp16).
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1u));
}
// D[64 x 16] += A[64 x 16] * B[16 x 16]^T, A in registers.
__device__ __forceinline__ void wgmma_rs_n16(float (&d)[8], const uint32_t* a, uint64_t b_desc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc), "r"(1u));
}

// GELU(y) = y * Phi(y), Phi(y) = 0.5 (1 + erf(y / sqrt 2)).  erf(z) = tanh(z (a + b z^2 + c z^4)) to 1.0e-4 (fitted, max error
// of the resulting GELU 2.5e-5 absolute — 20x below the fp16 rounding of the activation it feeds), evaluated as a logistic
// with ex2 / rcp so it is branch-free: y / (1 + 2^(-2 log2(e) u)), u = y (c0 + c1 y^2 + c2 y^4).
__device__ __forceinline__ float gelu_tc(float y) {
  const float y2 = fminf(y * y, 52.f);                              // beyond |y| ~ 7.2 the logistic is saturated anyway
  // -2 log2(e) * (c0 + c1 y^2 + c2 y^4)
  const float p = fmaf(y2, fmaf(y2, 1.014244e-3f, -1.0677588e-1f), -2.3011216f);
  const float t = y * p;
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(t));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(e + 1.0f));
  return y * r;
}

// GELU(y) for a packed pair given hy = y / 2:  hy + hy * tanh(hy (c0 + c1 hy^2 + c2 hy^4)) (clamp hy^2 <= 13), with HFMA2
// arithmetic and one tanh.approx.f16x2 per pair.
__device__ __forceinline__ uint32_t gelu_hy_x2(float hy0, float hy1) {
  const __half2 hy = __floats2half2_rn(hy0, hy1);
  const __half2 s = __hmin2(__hmul2(hy, hy), __float2half2_rn(13.f));
  const __half2 p = __hfma2(s, __hfma2(s, __float2half2_rn(-1.124832e-2f), __float2half2_rn(2.960456e-1f)), __float2half2_rn(1.594992f));
  const __half2 u = __hmul2(hy, p);
  uint32_t t;
  asm("tanh.approx.f16x2 %0, %1;" : "=r"(t) : "r"(*reinterpret_cast<const uint32_t*>(&u)));
  const __half2 g = __hfma2(hy, *reinterpret_cast<const __half2*>(&t), hy);
  return *reinterpret_cast<const uint32_t*>(&g);
}

// The same function with fp32 arithmetic (tanh.approx.f32) and ONE rounding to fp16 at the end.  tanh.approx.f16x2 truncates
// towards zero (mean error -2.4e-4 sign(u) on 0.25 <= |u| < 4, one fp16 ulp at most), which gives gelu_hy_x2 a coherent
// negative bias of 1.6e-4 .. 3.9e-4 on every activation with |y| > 0.5; the data-generation statistics of the self-play loop
// respond to that bias (tests/test_rela_module.py P5), not to the rounding noise.
__device__ __forceinline__ float gelu_hy_f32(float hy) {
  const float s = fminf(__fmul_rn(hy, hy), 13.f);
  const float p = __fmaf_rn(s, __fmaf_rn(s, -1.124832e-2f, 2.960456e-1f), 1.594992f);
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(__fmul_rn(hy, p)));
  return __fmaf_rn(hy, t, hy);
}
__device__ __forceinline__ uint32_t gelu_hy_t32(float hy0, float hy1) {
  const __half2 g = __floats2half2_rn(gelu_hy_f32(hy0), gelu_hy_f32(hy1));
  return *reinterpret_cast<const uint32_t*>(&g);
}

// kGelu: 0 = fp32 logistic GELU of y (CFRB_NET_TC_F16); 1 = packed-half GELU, 2 = fp32 tanh GELU (both CFRB_NET_TC_F16X2:
// the LayerNorm parameters in the blob are gamma / 2, beta / 2, so the affine yields hy = y / 2)
template <int kGelu>
__device__ __forceinline__ uint32_t act_pair(float y0, float y1) {
  if (kGelu == 1) return gelu_hy_x2(y0, y1);
  if (kGelu == 2) return gelu_hy_t32(y0, y1);
  const __half2 h = __floats2half2_rn(gelu_tc(y0), gelu_tc(y1));
  return *reinterpret_cast<const uint32_t*>(&h);
}

// LayerNorm (eps 1e-5, mean-free, see above) + GELU of a warpgroup's 64 x 256 accumulators, packed to fp16 as the A fragments of
// the next layer's wgmma: K-step kk = 8h + i/2 takes act[4kk .. 4kk+3].  A thread holds rows r and r + 8 (d[4i], d[4i+1] and
// d[4i+2], d[4i+3]) at columns 128h + 8i + 2q + {0, 1}, q = lane & 3; the four threads of a quad share the rows.
// ln: float4 {gamma_j, gamma_j+1, beta_j, beta_j+1} per feature pair.  half_ready(h) runs as soon as act[32h .. 32h+31] (K-steps
// 8h .. 8h+7) are written: layer 3 issues its first eight K-steps there, so they run under the second half of the GELU.
struct NoHalf {
  __device__ __forceinline__ void operator()(int) const {}
};
template <int kGelu, typename Half = NoHalf>
__device__ __forceinline__ void ln_gelu(const float (&acc)[2][64], const float4* __restrict__ ln, int q, uint32_t (&act)[64],
                                        Half half_ready = Half()) {
  float s[4] = {0.f, 0.f, 0.f, 0.f};        // (row r, row r + 8) x two independent chains
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int c = (i & 1) * 2;
      s[c] = fmaf(acc[h][4 * i], acc[h][4 * i], s[c]);
      s[c] = fmaf(acc[h][4 * i + 1], acc[h][4 * i + 1], s[c]);
      s[c + 1] = fmaf(acc[h][4 * i + 2], acc[h][4 * i + 2], s[c + 1]);
      s[c + 1] = fmaf(acc[h][4 * i + 3], acc[h][4 * i + 3], s[c + 1]);
    }
  float lo = s[0] + s[2], hi = s[1] + s[3];
  lo += __shfl_xor_sync(0xffffffffu, lo, 1);
  hi += __shfl_xor_sync(0xffffffffu, hi, 1);
  lo += __shfl_xor_sync(0xffffffffu, lo, 2);
  hi += __shfl_xor_sync(0xffffffffu, hi, 2);
  // the rows of W and the biases are centred over the features on the host: the mean of the 256 accumulators is zero
  const float rstd_lo = rsqrtf(lo * (1.f / kHid) + 1e-5f), rstd_hi = rsqrtf(hi * (1.f / kHid) + 1e-5f);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float4 pp = ln[h * 64 + i * 4 + q];
      act[h * 32 + 2 * i] = act_pair<kGelu>(__fmaf_rn(__fmul_rn(acc[h][4 * i], rstd_lo), pp.x, pp.z),
                                            __fmaf_rn(__fmul_rn(acc[h][4 * i + 1], rstd_lo), pp.y, pp.w));
      act[h * 32 + 2 * i + 1] = act_pair<kGelu>(__fmaf_rn(__fmul_rn(acc[h][4 * i + 2], rstd_hi), pp.x, pp.z),
                                                __fmaf_rn(__fmul_rn(acc[h][4 * i + 3], rstd_hi), pp.y, pp.w));
    }
    half_ready(h);
  }
}

struct TcArgs {
  const uint8_t* blob;      // weights in smem layout (BlobLayout)
  const __half* Xh;         // [tiles][Kp/8][16][8][8] fp16 query tiles
  const int* rows_ptr;      // rows to evaluate (read on the device)
  const int* row_src;       // output row of each query-tile row (compacted tiles, CfrDev::row_src) -- or nullptr: the same row
  float* out;               // [rows][Hout]
  int Kp, H, Hout;
  float* dbg_d1;            // optional [128][256] raw layer-1 accumulators of tile 0
  float* dbg_d2;            // optional [128][256] raw layer-2 accumulators of tile 0
  long long* trace;         // optional (debug build only): SM clock stamps of CTA 0, [2048]: thread 0 of warpgroup w at
                            // [w * 1024 + j * 8 + e] for its j-th tile (j < 64): e = 0 query tile ready, 1 layer 1 done,
                            // 2 epilogue 1 done, 3 turn taken, 4 layer 2 issued, 5 layer 2 done, 6 epilogue 2 done (layer 3
                            // issued under it), 7 outputs written.  Warpgroup 1 takes its first turn between stamps 1 and 2
                            // of its tile 0.
};

// Named barriers (0 is __syncthreads): kBarWg + w gathers the four warps of warpgroup w; kBarTurn + w is warpgroup w's turn
// to issue its layer-2 chain (bar.sync by w, bar.arrive by the other warpgroup: 256 threads).
constexpr int kBarWg = 1;
constexpr int kBarTurn = 3;

template <bool kDebug, int kGelu>
__global__ void __launch_bounds__(kThreads, 1) leaf_mlp_tc_kernel(TcArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const BlobLayout L(a.Kp);
  // wg and rows through a shuffle: ptxas then knows they are warp-uniform, and the branches on them (the turns below) do not
  // make it serialise the wgmmas (C7520) or spill
  const int tid = threadIdx.x, wg = __shfl_sync(0xffffffffu, tid >> 7, 0), lt = tid & 127, warp = lt >> 5, lane = tid & 31;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bar);
  const uint32_t bar_w = smem_u32(bars + 0), bar_x = smem_u32(bars + 1);   // x buffer b: bar_x + 8 b
  int* xcnt = reinterpret_cast<int*>(smem + L.off_xcnt);
  if (tid == 0) {
    mbar_init(bar_w, 1); mbar_init(bar_x, 1); mbar_init(bar_x + 8, 1);
    xcnt[0] = 0; xcnt[1] = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // weights: independent of the CFR kernel that precedes this launch -> fetched while that kernel drains (programmatic
  // dependent launch); the query tiles are read only after griddepcontrol.wait
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

  const uint32_t sx = smem_u32(smem + L.off_x), sw1 = smem_u32(smem + L.off_w1), sw2 = smem_u32(smem + L.off_w2),
                 sw3 = smem_u32(smem + L.off_w3);
  const uint8_t* xg = reinterpret_cast<const uint8_t*>(a.Xh);
  auto tile_of = [&](int j) { return (int)blockIdx.x + j * (int)gridDim.x; };
  auto fetch_x = [&](int j) {                   // query tile of the CTA's j-th tile -> x buffer j & 1
    const uint32_t b = bar_x + 8 * (j & 1);
    mbar_expect_tx(b, (uint32_t)L.x_bytes);
    bulk_g2s(sx + (j & 1) * (uint32_t)L.x_bytes, xg + (size_t)tile_of(j) * L.x_bytes, (uint32_t)L.x_bytes, b);
  };
  if (tid == 0) {
    fetch_x(0);
    if (J > 1) fetch_x(1);
  }
  mbar_wait(bar_w, 0);

  const float4* ln1 = reinterpret_cast<const float4*>(smem + L.off_ln1);
  const float4* ln2 = reinterpret_cast<const float4*>(smem + L.off_ln2);
  const float* b2 = reinterpret_cast<const float*>(smem + L.off_b2);
  const float* b3 = reinterpret_cast<const float*>(smem + L.off_b3);
  const int q = lane & 3;
  const int r_lo = warp * 16 + (lane >> 2);     // this thread's rows within the warpgroup's 64: r_lo and r_lo + 8
  // K-major core-matrix strides: LBO = next 8 columns of K, SBO = next 8 rows
  const uint32_t lbo_x = (kTileM / 8) * 128, lbo_w = (kHid / 8) * 128, lbo_w3 = (kNout / 8) * 128;
  float acc[2][64];
  uint32_t act[64];

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

  // Ping-pong: the layer-2 chains of the two warpgroups take turns on the tensor cores.  A warpgroup takes its turn before it
  // issues layer 2 and passes it on as soon as the chain is issued.  Warpgroup 0 has the first turn; warpgroup 1 takes its
  // first turn already before epilogue 1 of its first tile, so that it starts one phase behind, its first epilogue under
  // warpgroup 0's first layer 2.  (Holding the turn through epilogue 1 on every tile, which keeps the two epilogues apart, was
  // slower: an epilogue is bound by the latency of its own dependent instructions, not by issue slots, and two of them side by
  // side, one warp of each warpgroup per SM sub-partition, cover each other's latency.)  Both warpgroups run the same J tiles;
  // warpgroup 0 takes J - 1 turns (none at j = 0) and passes J, warpgroup 1 takes J and passes J - 1 (none after its last
  // chain), so every bar.arrive meets its bar.sync before exit, and neither warpgroup can arrive twice before the other has
  // synchronised once.
  auto take_turn = [&] { asm volatile("bar.sync %0, 256;" ::"r"(kBarTurn + wg) : "memory"); };
  auto pass_turn = [&] { asm volatile("bar.arrive %0, 256;" ::"r"(kBarTurn + (wg ^ 1)) : "memory"); };

  for (int j = 0; j < J; ++j) {
    const int tile = tile_of(j), buf = j & 1;
    const uint32_t xb = sx + buf * (uint32_t)L.x_bytes + wg * (kWgRows / 8) * 128;
    mbar_wait(bar_x + 8 * buf, (j >> 1) & 1);
    CFRB_TRACE(0);
    // ---- layer 1: D1 = X W1'^T (bias 1 through the constant-1 query column)
    wgmma_fence();
#pragma unroll 1
    for (int kk = 0; kk < a.Kp / 16; ++kk) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
        wgmma_ss_n128(acc[h], make_desc(xb + kk * 2 * lbo_x, lbo_x, 128), make_desc(sw1 + kk * 2 * lbo_w + h * 2048, lbo_w, 128), kk > 0);
    }
    wgmma_commit();
    wgmma_wait_all();
    fence_regs(acc[0]); fence_regs(acc[1]);
    // wgmma.wait_group covers only the calling warp's reads of the buffer: all four warps of the warpgroup meet first (named
    // barrier kBarWg + wg), then the second warpgroup to get here refills the buffer with the tile two ahead.  The layer-2
    // issues of the two warpgroups alternate, so neither gets more than two tiles ahead of the other: a warpgroup waits for
    // tile j + 2 only after both have passed layer 1 of tile j, never for tile j + 4 of the same buffer.
    asm volatile("bar.sync %0, 128;" ::"r"(kBarWg + wg) : "memory");
    if (lt == 0 && (atomicAdd(&xcnt[buf], 1) & 1) && j + 2 < J) fetch_x(j + 2);
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
    // ---- epilogue 2 and layer 3 (raw net outputs; the CFR backward kernel multiplies by the opponent-reach scaler): each half
    // of the m64n16k16 chain is issued as soon as epilogue 2 has produced its A fragments; the steps still accumulate in K order.
    // (A fence per K-step, i.e. issuing each step as soon as its four registers exist, splits the GELU into sixteen short
    // scheduling windows and made epilogue 2 about twice as long.)
    float o[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o[i] = 0.f;
    ln_gelu<kGelu>(acc, ln2, q, act, [&](int h) {
      wgmma_fence();
#pragma unroll
      for (int kk = 8 * h; kk < 8 * h + 8; ++kk) wgmma_rs_n16(o, act + 4 * kk, make_desc(sw3 + kk * 2 * lbo_w3, lbo_w3, 128));
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
        for (int i = 0; i < 2; ++i) {
          const int c = i * 8 + 2 * q;
          if (c < a.Hout) *reinterpret_cast<float2*>(orow + c) = make_float2(o[4 * i + 2 * e] + b3[c], o[4 * i + 2 * e + 1] + b3[c + 1]);
        }
      }
    }
    CFRB_TRACE(7);
  }
#undef CFRB_TRACE
}

}  // namespace tc
}  // namespace cfrb
