// The row schedule of the exact full-neighbourhood inference kernels (sage_infer.cu, hetero_infer.cu).
//
// A CTA of kFullRowThreads threads holds G = kFullRowThreads / LPR lane groups of LPR lanes; group g reduces target row
// r0 + blockIdx.x * G + g of the chunk [r0, r1).  Degrees are power-law, so a row of more than kFullRowHubDeg neighbours
// (a hub) is not walked by one group while the rest of the GPU idles: it is queued in shared memory and reduced by the
// whole CTA, group g taking neighbours g, g + G, ..., and the G partials are merged in group order.  Which path a row
// takes depends on its degree alone, and no floating-point atomics are used, so every row has one fixed reduction order:
// results are bitwise identical from call to call and for any chunking.
#pragma once
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

constexpr int kFullRowThreads = 256;
constexpr int kFullRowHubDeg = 256;

// own(r) on the group's row r < r1 when deg(r) <= kFullRowHubDeg (deg may leave what own needs in the caller's
// registers), otherwise r is queued; then hub(r) on the whole CTA for each queued row, each followed by a barrier.
template <int G, typename Deg, typename Own, typename Hub>
__device__ __forceinline__ void full_rows(int64_t r0, int64_t r1, int g, int gl, Deg deg, Own own, Hub hub) {
  __shared__ int64_t s_hub[G];
  __shared__ int s_nhub;
  if (threadIdx.x == 0) s_nhub = 0;
  __syncthreads();
  // 32-bit offset into the chunk: 2^32 output rows would not fit in device memory
  const int64_t r = r0 + (blockIdx.x * G + g);
  if (r < r1) {
    if (deg(r) > kFullRowHubDeg) {
      if (gl == 0) s_hub[atomicAdd(&s_nhub, 1)] = r;
    } else {
      own(r);
    }
  }
  __syncthreads();
  const int nhub = s_nhub;
  for (int h = 0; h < nhub; ++h) {
    hub(s_hub[h]);
    __syncthreads();
  }
}

// Element e of one vector of a lane's registers: a float[N], or a single float (N = 1).
template <typename T>
__device__ __forceinline__ T& vec_elem(T& x, int) { return x; }
template <typename T, int N>
__device__ __forceinline__ T& vec_elem(T (&x)[N], int e) { return x[e]; }

// Hub rows: lane gl of group g stores its vectors c = v * LPR + gl of N = sizeof(V) / 4 elements (columns c * N ..
// < width) into the group's row of the [G][width] partials p.
template <int LPR, int VPL, typename V>
__device__ __forceinline__ void put_partials(float* p, int width, int g, int gl, const V (&x)[VPL]) {
  constexpr int N = sizeof(V) / sizeof(float);
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    const int col = (v * LPR + gl) * N;
    if (col < width)
#pragma unroll
      for (int e = 0; e < N; ++e) p[g * width + col + e] = vec_elem(x[v], e);
  }
}

// x = the G groups' partials summed in group order, 0 + p_0 + p_1 + ...: for the lanes of group 0, after a barrier that
// follows every group's put_partials.
template <int G, int LPR, int VPL, typename V>
__device__ __forceinline__ void sum_partials(const float* p, int width, int gl, V (&x)[VPL]) {
  constexpr int N = sizeof(V) / sizeof(float);
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    const int col = (v * LPR + gl) * N;
    if (col >= width) continue;
#pragma unroll
    for (int e = 0; e < N; ++e) vec_elem(x[v], e) = 0.f;
#pragma unroll 1
    for (int q = 0; q < G; ++q)
#pragma unroll
      for (int e = 0; e < N; ++e) vec_elem(x[v], e) += p[q * width + col + e];
  }
}

// One CTA per G rows of [a.r0, a.r1) with group_floats floats of dynamic shared memory per group; nothing for an empty
// range.
template <int LPR, typename Args>
void launch_full_rows(void (*kernel)(Args), const Args& a, size_t group_floats, cudaStream_t s) {
  constexpr int G = kFullRowThreads / LPR;
  if (a.r1 <= a.r0) return;
  const int64_t blocks = (a.r1 - a.r0 + G - 1) / G;
  const size_t smem = sizeof(float) * G * group_floats;
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  launch_k(kernel, dim3(static_cast<unsigned>(blocks)), dim3(kFullRowThreads), smem, s, a);
}

}  // namespace glt
