// Host helpers shared by the C ABI's translation units: error propagation, kernel attribute setup
// and the counted kernel launch with the optional attributes the library uses: programmatic
// dependent launch (the kernel calls griddepcontrol.wait before it reads its predecessor's output)
// and a thread block cluster along x.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/n2nmn_b200.h"

namespace n2nmn {

int fail_with(int code, const std::string& msg);   // capi.cu: sets n2nmn_last_error()

#define CUDA_TRY(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return fail_with(N2NMN_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

#define TRY(expr)                                                                       \
  do {                                                                                  \
    if (int _rc = (expr)) return _rc;                                                   \
  } while (0)

// Maximum dynamic shared memory of a kernel and, if carveout >= 0, its preferred carveout.
template <class... KArgs>
int set_smem(void (*kernel)(KArgs...), int bytes, int carveout = -1) {
  CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  if (carveout >= 0)
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
  return 0;
}

struct LaunchAttrs {
  bool pdl = false;
  unsigned cluster = 1;   // CTAs per cluster along x; 1 = no cluster attribute
};

// Every kernel launch goes through here: counted once in `launches` when the runtime accepted it,
// N2NMN_ERR_CUDA with the runtime's message when it did not.
template <class... KArgs, class... Args>
int launch(int64_t& launches, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
           cudaStream_t st, LaunchAttrs a, Args... args) {
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
  const cudaError_t e = cudaLaunchKernelEx(&lc, kernel, KArgs(args)...);
  if (e != cudaSuccess)
    return fail_with(N2NMN_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(e));
  ++launches;
  return 0;
}

}  // namespace n2nmn
