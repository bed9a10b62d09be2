// Instantiations of the two-CTA cluster value net (leaf_mlp_tc_cluster.cuh) for 16, 32, 48 and 64 output columns per CTA.  A
// translation unit of its own, so that it compiles in parallel with cfrb_api.cu.
#include "leaf_mlp_tc_cluster.cuh"

namespace cfrb {
namespace tc {

template <int kNh>
static cudaError_t configure_nh(int smem_bytes, int* max_clusters) {
  cudaError_t e = cudaFuncSetAttribute(leaf_mlp_tc_cluster_kernel<kNh>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
  if (e != cudaSuccess) return e;
  cudaLaunchConfig_t lc{};
  lc.gridDim = dim3(kClusterCtas); lc.blockDim = dim3(kThreads); lc.dynamicSmemBytes = smem_bytes;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = kClusterCtas; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  lc.attrs = at; lc.numAttrs = 1;
  return cudaOccupancyMaxActiveClusters(max_clusters, leaf_mlp_tc_cluster_kernel<kNh>, &lc);
}

cudaError_t cluster_configure(int nh, int smem_bytes, int* max_clusters) {
  if (nh == 16) return configure_nh<16>(smem_bytes, max_clusters);
  if (nh == 32) return configure_nh<32>(smem_bytes, max_clusters);
  if (nh == 48) return configure_nh<48>(smem_bytes, max_clusters);
  if (nh == 64) return configure_nh<64>(smem_bytes, max_clusters);
  return cudaErrorInvalidValue;
}

cudaError_t cluster_launch(const cudaLaunchConfig_t& lc, const TcArgs& a, int nh) {
  if (nh == 16) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_cluster_kernel<16>, a);
  if (nh == 32) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_cluster_kernel<32>, a);
  if (nh == 48) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_cluster_kernel<48>, a);
  if (nh == 64) return cudaLaunchKernelEx(&lc, leaf_mlp_tc_cluster_kernel<64>, a);
  return cudaErrorInvalidValue;
}

}  // namespace tc
}  // namespace cfrb
