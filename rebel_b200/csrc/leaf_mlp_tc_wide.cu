// Instantiations of the wide tensor-core value net (leaf_mlp_tc_wide.cuh): output layers of 16, 32 and 48 columns, the three
// GELU variants, release and debug (layer taps, phase trace) builds.  A translation unit of its own, so that it compiles in
// parallel with cfrb_api.cu.
#include "leaf_mlp_tc_wide.cuh"

namespace cfrb {
namespace tc {

template <int kNo>
static cudaError_t configure_nout(int smem_bytes) {
  const cudaFuncAttribute at = cudaFuncAttributeMaxDynamicSharedMemorySize;
  cudaError_t e;
  if ((e = cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<false, 0, kNo>, at, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<true, 0, kNo>, at, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<false, 1, kNo>, at, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<true, 1, kNo>, at, smem_bytes)) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<false, 2, kNo>, at, smem_bytes)) != cudaSuccess) return e;
  return cudaFuncSetAttribute(leaf_mlp_tc_wide_kernel<true, 2, kNo>, at, smem_bytes);
}

template <int kNo>
static cudaError_t launch_nout(const cudaLaunchConfig_t& lc, const TcArgs& a, int gelu, bool dbg) {
  if (dbg && gelu == 1) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<true, 1, kNo>, a);
  if (dbg && gelu == 2) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<true, 2, kNo>, a);
  if (dbg) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<true, 0, kNo>, a);
  if (gelu == 1) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<false, 1, kNo>, a);
  if (gelu == 2) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<false, 2, kNo>, a);
  return cudaLaunchKernelEx(&lc, leaf_mlp_tc_wide_kernel<false, 0, kNo>, a);
}

cudaError_t wide_configure(int nout, int smem_bytes) {
  if (nout == 16) return configure_nout<16>(smem_bytes);
  if (nout == 32) return configure_nout<32>(smem_bytes);
  if (nout == 48) return configure_nout<48>(smem_bytes);
  return cudaErrorInvalidValue;
}

cudaError_t wide_launch(const cudaLaunchConfig_t& lc, const TcArgs& a, int nout, int gelu, bool dbg) {
  if (nout == 16) return launch_nout<16>(lc, a, gelu, dbg);
  if (nout == 32) return launch_nout<32>(lc, a, gelu, dbg);
  if (nout == 48) return launch_nout<48>(lc, a, gelu, dbg);
  return cudaErrorInvalidValue;
}

}  // namespace tc
}  // namespace cfrb
