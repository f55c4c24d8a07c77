// Host-side launch helper: every engine kernel goes through launch_k(), which sets the programmatic-stream-
// serialization attribute (PDL, see device_utils.cuh) unless set_pdl(0) turned it off.  Under stream capture
// consecutive launches become programmatic edges of the CUDA graph.
#pragma once
#include <cuda_runtime.h>

namespace glt {

// Process-wide switch (default on, set_pdl).  Read at every launch, so a caller can turn it off around the
// capture of a CUDA graph: programmatic edges help single-stream chains (hetero engine, the unpipelined step) but can
// cost when two streams interleave kernels (sample || train), because early-launched dependents hold SM slots that
// the other stream's kernels could have used.
int& pdl_flag();
inline bool pdl_enabled() { return pdl_flag() != 0; }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                            Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace glt
