// One optimisation step of the value net on the GPU: the reference trainer's loop body (cfvpy/selfplay.py:409-438) for
// Net2(n_hidden=256, n_layers=2, use_layer_norm=True) — forward (Linear -> LayerNorm -> GELU(erf), twice, then Linear), the
// huber or mse loss of selfplay.py:135-149, backward through every parameter, clip_grad_norm_ (selfplay.py:636-651) and
// torch.optim.Adam with its defaults (betas 0.9 / 0.999, eps 1e-8, no weight decay, bias correction).
//
// Everything is fp32 operands with fp32 accumulation, like the reference's PyTorch training.  Every sum (the GEMMs' dot
// products, the batch reductions of the weight and bias gradients, the LayerNorm row statistics, the norms, the batch loss) is
// compensated: fp32 error-free transformations (TwoSum, TwoProduct by FMA) carry each rounding error along and add it back at
// the end, so a sum is about as accurate as if it had been accumulated in twice the precision.  That matters where sums cancel:
// a gradient element not much larger than Adam's eps = 1e-8 moves its parameter by lr * g / (|g| + eps), which magnifies the
// absolute error of g.  The step is deterministic: no atomics, and every sum runs in an order fixed by the shapes alone, so the
// same state and batch give the same bits on every run, eager or replayed from a CUDA graph.  All kernels run on the caller's stream and read the Adam step count and
// the clipping coefficient from device memory, so a step needs no host synchronisation.
//
// Parameters, gradients and Adam moments are each ONE flat fp32 buffer in Net2 state_dict order (include/cfrb200.h).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "leaf_mlp_simt.cuh"

namespace cfrb {
namespace train {

constexpr int kHid = 256;
constexpr int kParams = 10;   // tensors in FLAT_ORDER

// Offsets of the ten tensors of the flat buffer for a game with query width Q and H outputs.
struct Layout {
  int64_t off[kParams + 1];
  Layout() = default;
  Layout(int Q, int H) {
    const int64_t len[kParams] = {(int64_t)kHid * Q, kHid, kHid, kHid, (int64_t)kHid * kHid, kHid, kHid, kHid, (int64_t)H * kHid, H};
    off[0] = 0;
    for (int i = 0; i < kParams; ++i) off[i + 1] = off[i] + len[i];
  }
  int64_t total() const { return off[kParams]; }
};
enum { W1 = 0, B1, G1, BE1, W2, B2, G2, BE2, W3, B3 };

// A compensated fp32 sum: the value is s + c, where c collects the exact rounding error of every addition (TwoSum) and product
// (TwoProduct: fma(a, b, -a b)).  The _rn intrinsics keep the compiler from contracting a product into the next addition, which
// would break the error-free transformations.  combine() is exactly commutative, so butterfly reductions give every lane the
// same bits.
struct Sum {
  float s = 0.f, c = 0.f;
  __device__ __forceinline__ void add(float x) {
    const float t = __fadd_rn(s, x), bb = __fsub_rn(t, s);
    c = __fadd_rn(c, __fadd_rn(__fsub_rn(s, __fsub_rn(t, bb)), __fsub_rn(x, bb)));
    s = t;
  }
  __device__ __forceinline__ void add_prod(float a, float b) {
    const float p = __fmul_rn(a, b);
    c = __fadd_rn(c, __fmaf_rn(a, b, -p));
    add(p);
  }
  __device__ __forceinline__ float value() const { return __fadd_rn(s, c); }
};
__device__ __forceinline__ Sum combine(const Sum& a, const Sum& b) {
  Sum r;
  r.s = __fadd_rn(a.s, b.s);
  const float bb = __fsub_rn(r.s, a.s);
  const float e = __fadd_rn(__fsub_rn(a.s, __fsub_rn(r.s, bb)), __fsub_rn(b.s, bb));   // exact: (a.s + b.s) - r.s
  r.c = __fadd_rn(__fadd_rn(a.c, b.c), e);
  return r;
}

// ---------------------------------------------------------------------------------------------------------------- GEMM
// C[m][n] = sum_k A(m, k) B(k, n) (+ bias[n]) with A(m, k) = A[m * sam + k * sak], B(k, n) = B[k * sbk + n * sbn]: every
// product of the step (forward X W^T, input gradients dY W, weight gradients dY^T X) is this with its own strides.  One thread
// owns a 2 x 2 block of C and sums over k in increasing order, compensated (Sum).
struct Gemm {
  const float* A; int64_t sam, sak;
  const float* B; int64_t sbk, sbn;
  float* C; int64_t ldc;
  const float* bias;
  int M, N, K;
};
struct GemmPair { Gemm g[2]; };

constexpr int kT = 32;   // tile edge (M, N and K)

__global__ void __launch_bounds__(256) gemm_kernel(GemmPair p) {
  const Gemm& g = p.g[blockIdx.z];
  const int m0 = blockIdx.y * kT, n0 = blockIdx.x * kT;
  if (m0 >= g.M || n0 >= g.N) return;
  __shared__ float As[kT][kT + 1], Bs[kT][kT + 1];   // [k][m], [k][n]
  const int tid = threadIdx.x, ty = tid / 16, tx = tid % 16;
  Sum acc[2][2];
  const bool a_kfast = g.sak == 1, b_nfast = g.sbn == 1;
  for (int k0 = 0; k0 < g.K; k0 += kT) {
#pragma unroll
    for (int r = 0; r < kT * kT / 256; ++r) {
      const int idx = tid + r * 256;
      const int i = idx / kT, j = idx % kT;          // j is the coalesced index
      {
        const int m = a_kfast ? i : j, k = a_kfast ? j : i;
        const int gm = m0 + m, gk = k0 + k;
        As[k][m] = (gm < g.M && gk < g.K) ? g.A[gm * g.sam + gk * g.sak] : 0.f;
      }
      {
        const int n = b_nfast ? j : i, k = b_nfast ? i : j;
        const int gn = n0 + n, gk = k0 + k;
        Bs[k][n] = (gn < g.N && gk < g.K) ? g.B[gk * g.sbk + gn * g.sbn] : 0.f;
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < kT; ++k) {
      const float a0 = As[k][2 * ty], a1 = As[k][2 * ty + 1], b0 = Bs[k][2 * tx], b1 = Bs[k][2 * tx + 1];
      acc[0][0].add_prod(a0, b0); acc[0][1].add_prod(a0, b1);
      acc[1][0].add_prod(a1, b0); acc[1][1].add_prod(a1, b1);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int m = m0 + 2 * ty + i, n = n0 + 2 * tx + j;
      if (m < g.M && n < g.N) {
        Sum r = acc[i][j];
        if (g.bias) r.add(g.bias[n]);
        g.C[m * g.ldc + n] = r.value();
      }
    }
}

inline cudaError_t launch_gemm(const Gemm* g, int count, cudaStream_t st) {
  GemmPair p{};
  int gx = 1, gy = 1;
  for (int i = 0; i < count; ++i) {
    p.g[i] = g[i];
    gx = max(gx, (g[i].N + kT - 1) / kT);
    gy = max(gy, (g[i].M + kT - 1) / kT);
  }
  gemm_kernel<<<dim3(gx, gy, count), 256, 0, st>>>(p);
  return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------- row-wise kernels
// A warp owns a row of 256 hidden units: lane l holds units l, l + 32, ...  The butterfly sums give every lane the same bits.
__device__ __forceinline__ float warp_sum(Sum x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Sum y;
    y.s = __shfl_xor_sync(0xffffffffu, x.s, o);
    y.c = __shfl_xor_sync(0xffffffffu, x.c, o);
    x = combine(x, y);
  }
  return x.value();
}

constexpr int kRowsPerBlock = 8;   // 8 warps
constexpr float kLnEps = 1e-5f;

// z [n][256] -> xhat = (z - mean) * rstd, rstd [n], act = gelu(xhat * gamma + beta)
__global__ void __launch_bounds__(256) ln_gelu_fwd(const float* __restrict__ z, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* __restrict__ xhat,
                                                   float* __restrict__ rstd, float* __restrict__ act, int n) {
  const int row = blockIdx.x * kRowsPerBlock + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n) return;
  float x[8];
  Sum s;
#pragma unroll
  for (int i = 0; i < 8; ++i) { x[i] = z[(int64_t)row * kHid + lane + 32 * i]; s.add(x[i]); }
  const float mean = warp_sum(s) * (1.0f / kHid);
  Sum s2;
#pragma unroll
  for (int i = 0; i < 8; ++i) { x[i] -= mean; s2.add_prod(x[i], x[i]); }
  const float r = 1.0f / sqrtf(warp_sum(s2) * (1.0f / kHid) + kLnEps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int j = lane + 32 * i;
    const float xh = x[i] * r;
    xhat[(int64_t)row * kHid + j] = xh;
    act[(int64_t)row * kHid + j] = gelu_erf(xh * gamma[j] + beta[j]);
  }
  if (lane == 0) rstd[row] = r;
}

// Backward through GELU and LayerNorm of one row: da = dL/d act -> dy = dL/d(xhat * gamma + beta), dz = dL/dz.
__global__ void __launch_bounds__(256) ln_gelu_bwd(const float* __restrict__ da, const float* __restrict__ xhat,
                                                   const float* __restrict__ rstd, const float* __restrict__ gamma,
                                                   const float* __restrict__ beta, float* __restrict__ dy_out,
                                                   float* __restrict__ dz, int n) {
  const int row = blockIdx.x * kRowsPerBlock + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n) return;
  float xh[8], dxh[8];
  Sum s1, s2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int j = lane + 32 * i;
    const int64_t e = (int64_t)row * kHid + j;
    xh[i] = xhat[e];
    const float y = xh[i] * gamma[j] + beta[j];
    const float cdf = 0.5f * (1.0f + erff(y * 0.70710678118654752440f));
    const float pdf = expf(-0.5f * y * y) * 0.39894228040143267794f;
    const float dy = da[e] * (cdf + y * pdf);
    dy_out[e] = dy;
    dxh[i] = dy * gamma[j];
    s1.add(dxh[i]);
    s2.add_prod(dxh[i], xh[i]);
  }
  const float m1 = warp_sum(s1) * (1.0f / kHid), m2 = warp_sum(s2) * (1.0f / kHid), r = rstd[row];
  // dxh - m1 - xh m2 cancels where the gradient is small: one rounding at the end
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    Sum d;
    d.add(dxh[i]);
    d.add(-m1);
    d.add_prod(-xh[i], m2);
    dz[(int64_t)row * kHid + lane + 32 * i] = r * d.value();
  }
}

enum { LOSS_HUBER = 0, LOSS_MSE = 1 };

// x = values - pred; per element huber (|x| > 1: 2|x| - 1, else x^2) or x^2; row_loss = mean over the H outputs;
// dpred = dL/dpred of the batch mean of row_loss.
__global__ void __launch_bounds__(256) loss_rows(const float* __restrict__ pred, const float* __restrict__ values, int n, int H,
                                                 int kind, float* __restrict__ row_loss, float* __restrict__ dpred) {
  const int row = blockIdx.x * kRowsPerBlock + threadIdx.x / 32, lane = threadIdx.x % 32;
  if (row >= n) return;
  const float gscale = (1.0f / n) / H;   // d(mean over rows of mean over outputs) / d(element loss)
  Sum s;
  for (int h = lane; h < H; h += 32) {
    const int64_t e = (int64_t)row * H + h;
    const float x = values[e] - pred[e], ax = fabsf(x);
    float l, dl;
    if (kind == LOSS_HUBER && ax > 1.f) { l = 2.f * ax - 1.f; dl = copysignf(2.f, x); }
    else { l = x * x; dl = 2.f * x; }
    s.add(l);
    dpred[e] = -(gscale * dl);
  }
  const float t = warp_sum(s);
  if (lane == 0) row_loss[row] = t / H;
}

// Batch sums of per-row columns: out[j] = sum_rows x[r][j] (* y[r][j] when y is given), compensated, rows in increasing order
// within each of the 8 warps and the 8 partial sums combined in warp order.  blockIdx.y picks one of up to 4 jobs; a block covers 32 columns.
struct ColJob { const float* x; const float* y; float* out; int cols; };
struct ColJobs { ColJob j[4]; };

__global__ void __launch_bounds__(256) colsum_kernel(ColJobs jobs, int n) {
  const ColJob& jb = jobs.j[blockIdx.y];
  const int c0 = blockIdx.x * 32;
  if (c0 >= jb.cols) return;
  __shared__ Sum part[8][32];
  const int w = threadIdx.x / 32, lane = threadIdx.x % 32, c = c0 + lane;
  Sum s;
  if (c < jb.cols)
    for (int r = w; r < n; r += 8) {
      const int64_t e = (int64_t)r * jb.cols + c;
      if (jb.y) s.add_prod(jb.x[e], jb.y[e]);
      else s.add(jb.x[e]);
    }
  part[w][lane] = s;
  __syncthreads();
  if (w == 0 && c < jb.cols) {
    Sum t = part[0][lane];
#pragma unroll
    for (int i = 1; i < 8; ++i) t = combine(t, part[i][lane]);
    jb.out[c] = t.value();
  }
}

inline cudaError_t launch_colsum(const ColJob* j, int count, int n, cudaStream_t st) {
  ColJobs p{};
  int gx = 1;
  for (int i = 0; i < count; ++i) { p.j[i] = j[i]; gx = max(gx, (j[i].cols + 31) / 32); }
  colsum_kernel<<<dim3(gx, count), 256, 0, st>>>(p, n);
  return cudaGetLastError();
}

// Fixed-order compensated block sum (256 threads, a power-of-two tree in shared memory).
__device__ __forceinline__ float block_sum(Sum v, Sum* sh) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) sh[threadIdx.x] = combine(sh[threadIdx.x], sh[threadIdx.x + o]);
    __syncthreads();
  }
  const float r = sh[0].value();
  __syncthreads();
  return r;
}

// Blocks 0 .. kParams-1 (training only): squared 2-norm of each parameter's gradient -> sq_norms[p]; block 0 also advances the
// Adam step count.  The last block: batch loss = mean of row_loss -> last[0] and out[0], and the per-row losses -> out[2 ..] (last and out
// may be NULL).
struct FinishArgs {
  const float* grads; Layout L; float* sq_norms; long long* step;
  const float* row_loss; int n; float* last; float* out;
};
__global__ void __launch_bounds__(256) finish_kernel(FinishArgs a) {
  __shared__ Sum sh[256];
  if (blockIdx.x + 1 < gridDim.x) {
    const int p = blockIdx.x;
    Sum s;
    for (int64_t i = a.L.off[p] + threadIdx.x; i < a.L.off[p + 1]; i += 256) s.add_prod(a.grads[i], a.grads[i]);
    const float ss = block_sum(s, sh);
    if (threadIdx.x == 0) {
      a.sq_norms[p] = ss;
      if (p == 0) *a.step += 1;
    }
    return;
  }
  Sum acc;
  for (int r = threadIdx.x; r < a.n; r += 256) acc.add(a.row_loss[r]);
  const float s = block_sum(acc, sh);
  if (threadIdx.x == 0) {
    if (a.last) a.last[0] = s / a.n;
    if (a.out) a.out[0] = s / a.n;
  }
  if (a.out)
    for (int r = threadIdx.x; r < a.n; r += 256) a.out[2 + r] = a.row_loss[r];
}

// clip_grad_norm_ (total norm = sqrt of the sum of the squared per-parameter norms, the 2-norm of the 2-norms) then Adam, element-wise over the flat buffers, in torch's formula order (torch/optim/adam.py,
// _multi_tensor_adam): m = lerp(m, g, 1 - beta1); v = v * beta2 + (1 - beta2) * g * g; denom = sqrt(v) / sqrt(bc2) + eps;
// p += -(lr / bc1) * (m / denom), with the bias corrections in double like torch's Python scalars.  The clipped gradient is
// written back (what p.grad holds after clip_grad_norm_).
struct AdamArgs {
  float* params; float* grads; float* m; float* v; int64_t P;
  const float* sq_norms; const long long* step; double lr; float max_norm;
  float* last; float* out;
};
__global__ void __launch_bounds__(256) adam_kernel(AdamArgs a) {
  Sum ss;
#pragma unroll
  for (int p = 0; p < kParams; ++p) ss.add(a.sq_norms[p]);
  const float total = sqrtf(ss.value());
  // max_norm / (total + 1e-6) as torch evaluates a Python float over a tensor: reciprocal, then the product
  const float coef = (1.0f / (total + 1e-6f)) * a.max_norm;
  const bool clip = a.max_norm > 0.f && coef < 1.f;
  const double t = (double)*a.step;
  const double bc1 = 1.0 - pow(0.9, t), bc2 = 1.0 - pow(0.999, t);
  const float step_size = (float)(-(a.lr / bc1)), bc2_sqrt = (float)sqrt(bc2);
  const float w1 = (float)(1.0 - 0.9), beta2 = 0.999f, w2 = (float)(1.0 - 0.999), eps = 1e-8f;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    a.last[1] = total;
    if (a.out) a.out[1] = total;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < a.P; i += (int64_t)gridDim.x * blockDim.x) {
    float g = a.grads[i];
    if (clip) { g *= coef; a.grads[i] = g; }
    const float m = a.m[i] + w1 * (g - a.m[i]);
    const float v = a.v[i] * beta2 + w2 * g * g;
    a.m[i] = m;
    a.v[i] = v;
    const float denom = sqrtf(v) / bc2_sqrt + eps;
    a.params[i] = a.params[i] + step_size * (m / denom);
  }
}

}  // namespace train
}  // namespace cfrb
