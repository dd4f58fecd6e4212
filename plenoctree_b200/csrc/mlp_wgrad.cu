// mlp_wgrad.cu — launch of the weight-gradient contraction; body in wgrad_body.cuh.
#include "wgrad_body.cuh"

namespace pob {

__global__ void __launch_bounds__(WG_THREADS, 1) mlp_wgrad_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  wgrad_body(p, smem, int(blockIdx.x));
}

cudaError_t launch_mlp_wgrad(const WgradParams& p, int num_ctas, cudaStream_t stream) {
  cudaError_t e = cudaFuncSetAttribute(mlp_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)WG_SMEM);
  if (e != cudaSuccess) return e;
  // may start while the preceding mlp_bwd launch runs; the kernel never calls griddepcontrol.wait and synchronises on
  // the per-tile progress counters instead
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr.val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(num_ctas);
  cfg.blockDim = dim3(WG_THREADS);
  cfg.dynamicSmemBytes = WG_SMEM;
  cfg.stream = stream;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, mlp_wgrad_kernel, p);
}

}  // namespace pob
