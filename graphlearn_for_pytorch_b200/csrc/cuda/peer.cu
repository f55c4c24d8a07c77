// Collectives over NVLink peer memory, written as ordinary kernels so that they are CUDA-graph
// nodes of the training step (no NCCL call, no host involvement):
//
//   k_peer_barrier   cross-GPU barrier: every rank stamps an epoch into its slot of every peer's
//                    flag array (st.release.sys over NVLink) and spins on its own array.
//   k_adam_peer      one-shot all-reduce FUSED with the optimizer: each rank reads the gradient
//                    shards of all peers straight from their HBM, sums them in rank order (bitwise
//                    identical on every rank) and applies Adam -- the reduced gradient is never
//                    written anywhere.
//
// The reference leaves gradient synchronisation to torch DDP/NCCL in its example scripts
// (examples/multi_gpu/train_sage_ogbn_papers100m.py:55); the model here is ~1.3 MB of fp32
// gradients, far below the size where NCCL's launch + protocol latency amortises.
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

__device__ __forceinline__ void st_release_sys(int32_t* p, int32_t v) {
  asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ int32_t ld_acquire_sys(const int32_t* p) {
  int32_t v;
  asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// one block, >= world threads
__global__ void k_peer_barrier(PeerPtrs p, int which, int32_t* epoch_dev, int32_t* err) {
  pdl_enter();
  __shared__ int s_epoch;
  const int r = threadIdx.x;
  if (r == 0) s_epoch = epoch_dev[which] + 1;
  __syncthreads();
  const int e = s_epoch;
  __threadfence_system();  // everything this GPU wrote before the barrier is visible to peers
  if (r < p.world) {
    st_release_sys(p.flags[r] + which * p.world + p.rank, e);
    const int32_t* mine = p.flags[p.rank] + which * p.world + r;
    const long long t0 = clock64();
    while (ld_acquire_sys(mine) < e) {
      if (clock64() - t0 > 8000000000LL) {  // ~4 s: a peer died; do not hang the GPU
        if (err) atomicExch(err, 1 + r);
        break;
      }
    }
  }
  __syncthreads();
  if (r == 0) epoch_dev[which] = e;
}

__device__ __forceinline__ float4 ld_cv4(const float* p) {
  float4 v;
  asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

__global__ void __launch_bounds__(256) k_adam_peer(PeerPtrs p, float* param, float* m, float* v,
                                                   __nv_bfloat16* pb, int64_t n, float lr, float b1, float b2,
                                                   float eps, float wd, int32_t* step_dev, float gscale,
                                                   const int32_t* err) {
  pdl_enter();
  // a barrier of this step timed out (a peer died or stalled): the gradients are incomplete, so the update is
  // skipped on every rank that saw the timeout; the host raises at its next health check (models/sage.py)
  if (err && *reinterpret_cast<const volatile int32_t*>(err) != 0) return;
  // t = steps so far + 1; the last block to finish publishes it (see k_adam)
  const int t = *reinterpret_cast<volatile int32_t*>(step_dev) + 1;
  // bias corrections in double, as k_sparse_adam: 1 - b2^t cancels most of b2^t's bits at small t, which left the
  // error of __powf's approximate log2 in the update at dozens of times its fp32 rounding error
  const float c1 = static_cast<float>(1.0 - pow(static_cast<double>(b1), t));
  const float c2 = static_cast<float>(1.0 - pow(static_cast<double>(b2), t));
  const int64_t n4 = n >> 2;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    // local optimizer state first: these loads are in flight while the peer gradients cross NVLink
    const float4 pp = reinterpret_cast<const float4*>(param)[i];
    const float4 mm = reinterpret_cast<const float4*>(m)[i];
    const float4 vv = reinterpret_cast<const float4*>(v)[i];
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    // all peer loads of a batch of 8 ranks are issued before the first add: one NVLink round trip per batch
    // instead of one per rank (the adds keep rank order: identical result on every rank)
#pragma unroll 1
    for (int r0 = 0; r0 < p.world; r0 += 8) {
      float4 x[8];
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (r0 + q < p.world) x[q] = ld_cv4(p.g[r0 + q] + i * 4);
#pragma unroll
      for (int q = 0; q < 8; ++q)
        if (r0 + q < p.world) { g.x += x[q].x; g.y += x[q].y; g.z += x[q].z; g.w += x[q].w; }
    }
    float gi[4] = {g.x, g.y, g.z, g.w};
    float pa[4] = {pp.x, pp.y, pp.z, pp.w}, ma[4] = {mm.x, mm.y, mm.z, mm.w}, va[4] = {vv.x, vv.y, vv.z, vv.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float gq = gi[q] * gscale + wd * pa[q];
      ma[q] = b1 * ma[q] + (1.f - b1) * gq;
      va[q] = b2 * va[q] + (1.f - b2) * gq * gq;
      pa[q] -= lr * (ma[q] / c1) / (sqrtf(va[q] / c2) + eps);
    }
    reinterpret_cast<float4*>(param)[i] = make_float4(pa[0], pa[1], pa[2], pa[3]);
    reinterpret_cast<float4*>(m)[i] = make_float4(ma[0], ma[1], ma[2], ma[3]);
    reinterpret_cast<float4*>(v)[i] = make_float4(va[0], va[1], va[2], va[3]);
    if (pb) {
      __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(pb + i * 4);
      o[0] = __floats2bfloat162_rn(pa[0], pa[1]);
      o[1] = __floats2bfloat162_rn(pa[2], pa[3]);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(step_dev + 1, 1) == static_cast<int>(gridDim.x) - 1) {
      step_dev[1] = 0;
      step_dev[0] += 1;
    }
  }
}

}  // namespace

void launch_peer_barrier(const PeerPtrs& p, int which, int32_t* epoch_dev, int32_t* err, cudaStream_t s) {
  launch_k(k_peer_barrier, dim3(1), dim3(32), 0, s, p, which, epoch_dev, err);
}

void launch_adam_peer(const PeerPtrs& p, float* param, float* m, float* v, void* p_bf16, int64_t n, float lr,
                      float b1, float b2, float eps, float wd, int32_t* step_dev, float gscale,
                      cudaStream_t s, const int32_t* err) {
  int64_t blocks = ((n >> 2) + 255) / 256;
  if (blocks > 132 * 4) blocks = 132 * 4;
  if (blocks < 1) blocks = 1;
  launch_k(k_adam_peer, dim3(static_cast<int>(blocks)), dim3(256), 0, s, p, param, m, v,
           reinterpret_cast<__nv_bfloat16*>(p_bf16), n, lr, b1, b2, eps, wd, step_dev, gscale, err);
}

}  // namespace glt
