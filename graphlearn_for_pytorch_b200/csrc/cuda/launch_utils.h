// Host-side launch helpers: every engine kernel goes through launch_k(), which sets the programmatic-stream-
// serialization attribute (PDL, see device_utils.cuh) unless set_pdl(0) turned it off.  Under stream capture
// consecutive launches become programmatic edges of the CUDA graph.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

namespace glt {

// Blocks for `items` work items at `per_block` per block, clamped to [1, max_blocks] (default: 16 per SM of a
// 132-SM H100; grid-stride kernels cover the rest).
inline int grid_for(int64_t items, int per_block, int max_blocks = 132 * 16) {
  int64_t b = (items + per_block - 1) / per_block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return static_cast<int>(b);
}

// Lane-group shape of the row-parallel kernels: LPR lanes of a warp share one row of `nvec` 16-byte vectors and each
// lane owns VPL of them (vector c = v * LPR + lane).  LPR is the smallest power of two >= nvec in [MinLPR, 32]; above
// 32 vectors LPR = 32 and VPL = 2, then 4, up to MaxVPL.  Calls f(std::integral_constant<int, LPR>,
// std::integral_constant<int, VPL>) once; only the shapes of this ladder are instantiated.  A kernel whose lanes own
// VPL fixed vectors covers 32 * MaxVPL vectors per row: 128 vectors, i.e. 1024 bf16 columns, at MaxVPL = 4, and the
// same 1024 columns for the MXFP8 ladders (16 elements per vector, MaxVPL = 2).  The width checks in bindings.cc
// reject wider rows before launch.  (The LPR and VPL template parameters are the ladder's current step, not for
// callers to set.)
template <int MinLPR, int MaxVPL, int LPR = MinLPR, int VPL = 1, typename F>
inline void dispatch_lanes(int nvec, F&& f) {
  if constexpr (LPR < 32) {
    if (nvec <= LPR) f(std::integral_constant<int, LPR>(), std::integral_constant<int, 1>());
    else dispatch_lanes<MinLPR, MaxVPL, 2 * LPR, 1>(nvec, f);
  } else if constexpr (VPL < MaxVPL) {
    if (nvec <= 32 * VPL) f(std::integral_constant<int, 32>(), std::integral_constant<int, VPL>());
    else dispatch_lanes<MinLPR, MaxVPL, 32, 2 * VPL>(nvec, f);
  } else {
    f(std::integral_constant<int, 32>(), std::integral_constant<int, MaxVPL>());
  }
}

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
