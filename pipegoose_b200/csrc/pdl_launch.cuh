// Host-side launcher with optional programmatic dependent launch (PDL).
//   default / PIPEGOOSE_B200_PDL=1 : kernels are launched with cudaLaunchAttributeProgrammaticStreamSerialization, so a
//                          kernel's prologue overlaps the tail of its predecessor (every kernel launched through here
//                          calls pdl_launch_dependents() at its start and pdl_wait() before its first dependent access).
//   PIPEGOOSE_B200_PDL=0 : plain stream-ordered launches (the griddepcontrol instructions are no-ops)
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <utility>

namespace pg {

inline bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = std::getenv("PIPEGOOSE_B200_PDL");
    on = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return on == 1;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg;
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace pg
