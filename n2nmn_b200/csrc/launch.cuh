// Kernel launch with the optional attributes the library uses: programmatic dependent launch
// (the kernel calls griddepcontrol.wait before it reads its predecessor's output) and a thread
// block cluster along x.
#pragma once
#include <cuda_runtime.h>

namespace n2nmn {

struct LaunchAttrs {
  bool pdl = false;
  unsigned cluster = 1;   // CTAs per cluster along x; 1 = no cluster attribute
};

template <class... KArgs, class... Args>
cudaError_t launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                   LaunchAttrs a, Args... args) {
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (a.cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = a.cluster;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  if (a.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = grid; lc.blockDim = block; lc.dynamicSmemBytes = smem; lc.stream = st;
  lc.attrs = attr;
  lc.numAttrs = na;
  return cudaLaunchKernelEx(&lc, kernel, KArgs(args)...);
}

}  // namespace n2nmn
