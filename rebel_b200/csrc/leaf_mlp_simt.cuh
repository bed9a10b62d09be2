// fp32 SIMT evaluation of the leaf value net (Net2: Linear -> LayerNorm -> GELU(erf) -> Linear -> LayerNorm ->
// GELU -> Linear, cfvpy/models.py:64-94) over the packed query rows of a whole wave.  This is the PARITY path
// (CFRB_NET_FP32): same arithmetic type as the reference's libtorch fp32 forward
// (rela/model_locker.h:85-95), summation in k-order like a scalar dot product.  The tensor-core path lives in
// leaf_mlp_tc.cuh.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace cfrb {

struct NetDev {
  int Qpad, hidden, Hout;
  const float* w1t;   // [Qpad][hidden]   (transposed body.0.weight, zero rows for q >= Q)
  const float *b1, *g1, *be1;
  const float* w2t;   // [hidden][hidden] (transposed body.4.weight)
  const float *b2, *g2, *be2;
  const float* w3t;   // [hidden][Hout]   (transposed output.weight)
  const float* b3;
};

constexpr int kMlpRows = 32;   // rows per CTA

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// One dense layer for a 32-row tile: thread j owns output feature j for all rows.
// xs: [K][32] (k-major), wt: [K][HID] global.  Result left in acc[].  The bias is added after the dot product, as libtorch's
// addmm does: started from a large bias (a common offset of every feature, which LayerNorm removes) the sum would be rounded at
// the bias's ulp K times.
template <int HID>
__device__ __forceinline__ void dense_tile(const float* __restrict__ xs, const float* __restrict__ wt, int K, float bias,
                                           float (&acc)[kMlpRows], int j) {
#pragma unroll
  for (int r = 0; r < kMlpRows; ++r) acc[r] = 0.f;
  for (int k = 0; k < K; ++k) {
    const float w = __ldg(wt + (size_t)k * HID + j);
    const float4* xv = reinterpret_cast<const float4*>(xs + k * kMlpRows);
#pragma unroll
    for (int i = 0; i < kMlpRows / 4; ++i) {
      const float4 x = xv[i];
      acc[4 * i + 0] += x.x * w; acc[4 * i + 1] += x.y * w; acc[4 * i + 2] += x.z * w; acc[4 * i + 3] += x.w * w;
    }
  }
#pragma unroll
  for (int r = 0; r < kMlpRows; ++r) acc[r] += bias;
}

// LayerNorm(eps 1e-5, biased variance, affine) + GELU over ys[r][0..HID) for the 32 rows; writes xs[j][r].
template <int HID>
__device__ __forceinline__ void ln_gelu_tile(float (&acc)[kMlpRows], float* ys, float* stats, float* xs, const float* g,
                                             const float* be, int j) {
  constexpr int LD = HID + 1;
#pragma unroll
  for (int r = 0; r < kMlpRows; ++r) ys[r * LD + j] = acc[r];
  __syncthreads();
  const int warp = j >> 5, lane = j & 31, nwarps = HID / 32;
  for (int r = warp; r < kMlpRows; r += nwarps) {
    float s = 0.f;
    for (int i = lane; i < HID; i += 32) s += ys[r * LD + i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / HID;
    float v = 0.f;
    for (int i = lane; i < HID; i += 32) { const float d = ys[r * LD + i] - mean; v += d * d; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) { stats[2 * r] = mean; stats[2 * r + 1] = rsqrtf(v / HID + 1e-5f); }
  }
  __syncthreads();
  const float gj = g[j], bj = be[j];
#pragma unroll
  for (int r = 0; r < kMlpRows; ++r) {
    const float y = (acc[r] - stats[2 * r]) * stats[2 * r + 1] * gj + bj;
    xs[j * kMlpRows + r] = gelu_erf(y);
  }
  __syncthreads();
}

template <int HID>
__global__ void __launch_bounds__(HID) leaf_mlp_fp32_kernel(NetDev w, const float* __restrict__ X, const int* __restrict__ rows_ptr,
                                                            float* __restrict__ out) {
  extern __shared__ float sm[];
  float* xs = sm;                               // [HID][32]
  float* ys = xs + HID * kMlpRows;              // [32][HID+1]
  float* stats = ys + kMlpRows * (HID + 1);     // [32][2]
  const int rows = *rows_ptr;
  const int row0 = blockIdx.x * kMlpRows;
  if (row0 >= rows) return;
  const int j = threadIdx.x;
  // stage the query tile k-major
  for (int idx = j; idx < kMlpRows * w.Qpad; idx += HID) {
    const int r = idx / w.Qpad, q = idx % w.Qpad;
    xs[q * kMlpRows + r] = (row0 + r < rows) ? X[(size_t)(row0 + r) * w.Qpad + q] : 0.f;
  }
  __syncthreads();
  float acc[kMlpRows];
  dense_tile<HID>(xs, w.w1t, w.Qpad, w.b1[j], acc, j);
  __syncthreads();
  ln_gelu_tile<HID>(acc, ys, stats, xs, w.g1, w.be1, j);
  dense_tile<HID>(xs, w.w2t, HID, w.b2[j], acc, j);
  __syncthreads();
  ln_gelu_tile<HID>(acc, ys, stats, xs, w.g2, w.be2, j);
  for (int idx = j; idx < kMlpRows * w.Hout; idx += HID) {
    const int r = idx / w.Hout, o = idx % w.Hout;
    if (row0 + r >= rows) continue;
    float a = w.b3[o];
    for (int k = 0; k < HID; ++k) a += xs[k * kMlpRows + r] * __ldg(w.w3t + (size_t)k * w.Hout + o);
    out[(size_t)(row0 + r) * w.Hout + o] = a;
  }
}

inline size_t leaf_mlp_fp32_smem(int hid) { return sizeof(float) * ((size_t)hid * kMlpRows + (size_t)kMlpRows * (hid + 1) + 2 * kMlpRows); }

}  // namespace cfrb
