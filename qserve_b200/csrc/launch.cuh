// qserve_b200 -- the one launch path of every kernel: programmatic dependent launch as pdl_enabled() says, an optional 1-D cluster, and the
// per-device dynamic shared memory limit of a kernel.
#pragma once
#include <cuda_runtime.h>

#include "common.cuh"
#include "launch.h"

namespace qs {

// Launches `kern` on `stream` with the PDL attribute set from pdl_enabled().  cluster > 0 adds a (cluster, 1, 1) cluster dimension, cluster = 0
// none.  Returns QS_OK or the launch error, prefixed with `what`.
template <typename Kern, typename... Args>
int launch(Kern kern, dim3 grid, dim3 block, size_t smem, int cluster, void* stream, const char* what, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = static_cast<cudaStream_t>(stream);
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = cluster;
  attr[1].val.clusterDim.y = 1;
  attr[1].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = cluster > 0 ? 2 : 1;
  return check_cuda(cudaLaunchKernelEx(&cfg, kern, args...), what);
}

// Raises cudaFuncAttributeMaxDynamicSharedMemorySize of `kern` on the current device to at least `bytes` (capi.cu).  The largest value set is
// kept per (kernel address, device): instantiations of one template share a C++ type but not an address, and a kernel whose shared memory
// grows with the input is raised again when a launch needs more.
int raise_smem_limit(const void* kern, size_t bytes, const char* what);
template <typename... P>
int raise_smem_limit(void (*kern)(P...), size_t bytes, const char* what) {
  return raise_smem_limit(reinterpret_cast<const void*>(kern), bytes, what);
}

}  // namespace qs
