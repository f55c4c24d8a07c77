// TMA-fed wgmma GEMMs of the GraphSAGE engine (sm_90a): every dense contraction of the training step that
// is not already inside the fused layer-1 kernel runs here instead of in cuBLAS --
//
//   forward  layers 2..L : Z  = act([mean | self] . W^T + b)            A K-major, B K-major, bf16 out
//   backward dA          : dA = dPre . W                                 A K-major, B MN-major, bf16 out
//   backward dW          : dW += dPre^T . A   (split-K over the batch)   A MN-major, B MN-major, fp32 red-add
//
// The extents that depend on the sampled batch (rows of A for forward / dA, the contraction length for dW) are
// read from the sampler's device counters, so the launch is static and CUDA-graph capturable.
//
// One persistent CTA per SM, three warpgroups:
//   warpgroup 0 (one lane)  TMA producer: cp.async.bulk.tensor.2d boxes (SWIZZLE_128B) into a 4-stage smem ring
//   warpgroups 1, 2         consumers: rows [0, 64) / [64, 128) of the 128-row tile; wgmma.m64n64k16 per 64 columns
//                           of the tile (N <= 256: up to 128 fp32 accumulator registers per thread), then the
//                           epilogue: bias/ReLU -> bf16 -> swizzled smem staging -> TMA store, or fp32
//                           red.global.add.v2 for the split-K weight gradients
// Up to two independent problems share one launch (dW and dA of a layer both consume dPre): their work items form
// one combined item space.  The producer claims items from a per-plan ticket (atomicAdd), so a CTA that starts late
// -- its SM still held by a kernel of another stream (the sampler runs beside the training step) -- takes whatever
// is left instead of holding up the whole GEMM on items dealt to it in advance.  It publishes each item id to the
// consumers through a shared slot of the ring stage that carries the item's first k-block (written before the
// stage's arrive, which releases it; the consumers' wait acquires it), and a stop sentinel (-1, a plain arrive with
// no bytes) when the ticket runs past the end.
//
// The reference has no counterpart (its examples call PyG / cuBLAS through autograd).
#include <cuda.h>

#include <cstdio>
#include <cstring>
#include <mutex>

#include "launch_utils.h"
#include "tc_utils.cuh"

namespace glt {

namespace {

using namespace tc;

constexpr int kBM = 128;              // tile rows (two wgmma M = 64 halves)
constexpr int kBK = 64;               // k-block: 64 bf16 = 128 B = one swizzle row
constexpr int kStages = 4;
constexpr int kABytes = kBM * 128;    // 16 KB
constexpr int kBBytes = 256 * 128;    // 32 KB (BN <= 256)
constexpr int kStageBytes = kABytes + kBBytes;
constexpr int kStoreBytes = kBM * 128;   // one 128 x 64 bf16 staging tile for the TMA store
constexpr int kGemmThreads = 3 * 128;
constexpr int kEpiThreads = 2 * 128;
constexpr size_t kGemmSmem = static_cast<size_t>(kStages) * kStageBytes + 2 * kStoreBytes + 1024 + 256;

struct Derived {   // per-problem quantities every role derives identically from device-side state
  int m_tiles, n_tiles, kb_total, splits, kb_per, items;
};

__device__ __forceinline__ Derived derive(const TcProblem& p, int grid_share) {
  Derived d;
  int dyn = p.dyn ? min(p.dyn[p.dyn_idx], p.dyn_cap) : p.dyn_cap;
  if (dyn < 0) dyn = 0;
  const int m_ext = p.dyn_is_k ? p.m : dyn;
  const int k_ext = p.dyn_is_k ? dyn : p.k;
  d.m_tiles = (m_ext + kBM - 1) / kBM;
  d.n_tiles = p.n / p.bn;
  d.kb_total = (k_ext + kBK - 1) / kBK;
  const int tiles = d.m_tiles * d.n_tiles;
  int splits = 1;
  if (p.epi == 1 && tiles > 0) {
    splits = grid_share / tiles;
    if (splits < 1) splits = 1;
    if (splits > d.kb_total) splits = d.kb_total;
    if (splits < 1) splits = 1;
  }
  d.kb_per = (d.kb_total + splits - 1) / splits;
  d.splits = d.kb_per > 0 ? (d.kb_total + d.kb_per - 1) / d.kb_per : 0;   // no empty split
  d.items = (d.kb_total > 0) ? tiles * d.splits : 0;
  return d;
}

struct Item { int prob, m_tile, n_tile, kb0, kb1; };

__device__ __forceinline__ Item decode(int item, const Derived& d0, const Derived& d1) {
  Item it;
  it.prob = item < d0.items ? 0 : 1;
  const Derived& d = it.prob ? d1 : d0;
  int r = it.prob ? item - d0.items : item;
  const int split = r % d.splits;
  r /= d.splits;
  it.n_tile = r % d.n_tiles;
  it.m_tile = r / d.n_tiles;
  it.kb0 = split * d.kb_per;
  it.kb1 = min(it.kb0 + d.kb_per, d.kb_total);
  return it;
}

// One k-block (64 deep) of a consumer warpgroup: 4 k16 steps x NSL 64-column slabs.  Both layouts put 64 rows
// (K-major) or 64 columns (MN-major) of an operand into 8 KB, so the warpgroup's half of A and every slab of B start
// 8 KB apart; a k16 step advances 32 B (K-major) or 16 rows of 128 B (MN-major).
template <int TA, int TB, int NSL>
__device__ __forceinline__ void mma_kblock(float (&acc)[4][32], uint32_t sa, uint32_t sb) {
  constexpr uint32_t ka = TA ? 2048u : 32u, kb = TB ? 2048u : 32u;
  wgmma_fence();
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    const uint64_t da = make_sw128_desc_lbo(sa + k4 * ka, TA ? 8192 : 16, 1024);
#pragma unroll
    for (int j = 0; j < NSL; ++j)
      wgmma_m64n64k16_bf16<TA, TB>(acc[j], da, make_sw128_desc_lbo(sb + j * 8192 + k4 * kb, TB ? 8192 : 16, 1024), 1u);
  }
}

__global__ void __launch_bounds__(kGemmThreads, 1)
k_tc_gemm(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmB0,
          const __grid_constant__ CUtensorMap tmC0, const __grid_constant__ CUtensorMap tmA1,
          const __grid_constant__ CUtensorMap tmB1, const __grid_constant__ CUtensorMap tmC1,
          const TcGemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* stage0 = smem;                                     // kStages x [A 16 KB | B 32 KB]
  uint8_t* store0 = smem + kStages * kStageBytes;             // 2 x 16 KB staging tiles
  uint64_t* bars = reinterpret_cast<uint64_t*>(store0 + 2 * kStoreBytes);
  const uint32_t bar_full0 = smem_u32(bars + 0);               // + 8 * stage
  const uint32_t bar_empty0 = smem_u32(bars + kStages);        // + 8 * stage
  volatile int* item_slot = reinterpret_cast<volatile int*>(bars + 2 * kStages);   // [kStages] item id or -1

  const int wg = threadIdx.x >> 7;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(bar_full0 + 8 * s, 1);
      mbar_init(bar_empty0 + 8 * s, 8);             // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    prefetch_tmap(&tmA0); prefetch_tmap(&tmB0);
    if (g.p[0].epi == 0) prefetch_tmap(&tmC0);
    if (g.n_prob > 1) {
      prefetch_tmap(&tmA1); prefetch_tmap(&tmB1);
      if (g.p[1].epi == 0) prefetch_tmap(&tmC1);
    }
  }
  __syncthreads();
  // everything above (barrier init, tensor-map prefetch) overlapped with the tail of the previous kernel; from here
  // on the predecessor's results (counters, operands) are read
  pdl_wait();
  pdl_trigger();

  // identical on every thread: work decomposition from the device counters
  const int share = g.n_prob > 1 ? max(1, static_cast<int>(gridDim.x) / 2) : static_cast<int>(gridDim.x);
  const Derived d0 = derive(g.p[0], share);
  Derived d1; d1.m_tiles = d1.n_tiles = d1.kb_total = d1.splits = d1.kb_per = d1.items = 0;
  if (g.n_prob > 1) d1 = derive(g.p[1], share);
  const int total_items = d0.items + d1.items;

  if (wg == 0) {
    // ------------------------------ TMA producer ------------------------------
    if (threadIdx.x == 0) {
      int fill = 0;   // k-blocks produced so far (ring position)
      for (;;) {
        const int item = atomicAdd(g.tickets, 1);
        if (item >= total_items) break;
        const Item it = decode(item, d0, d1);
        const TcProblem& p = g.p[it.prob];
        const CUtensorMap* ta = it.prob ? &tmA1 : &tmA0;
        const CUtensorMap* tb = it.prob ? &tmB1 : &tmB0;
        const uint32_t bytes = kABytes + static_cast<uint32_t>(p.bn) * 128u;
        for (int kb = it.kb0; kb < it.kb1; ++kb, ++fill) {
          const int s = fill % kStages;
          const uint32_t ph = (fill / kStages) & 1;
          mbar_wait(bar_empty0 + 8 * s, ph ^ 1);
          const uint32_t full = bar_full0 + 8 * s;
          if (kb == it.kb0) item_slot[s] = item;
          mbar_expect_tx(full, bytes);
          const uint32_t sa = smem_u32(stage0 + s * kStageBytes);
          const uint32_t sb = sa + kABytes;
          if (!p.a_mn) {
            tma_load_2d(sa, ta, kb * kBK, it.m_tile * kBM, full);              // box {64 k, 128 rows}
          } else {
            tma_load_2d(sa, ta, it.m_tile * kBM, kb * kBK, full);              // box {64 m, 64 k-rows}
            tma_load_2d(sa + 8192, ta, it.m_tile * kBM + 64, kb * kBK, full);
          }
          if (!p.b_mn) {
            tma_load_2d(sb, tb, kb * kBK, it.n_tile * p.bn, full);             // box {64 k, bn rows}
          } else {
            for (int j = 0; j < p.bn / 64; ++j)                                // boxes {64 n, 64 k-rows}
              tma_load_2d(sb + j * 8192, tb, it.n_tile * p.bn + j * 64, kb * kBK, full);
          }
        }
      }
      // stop sentinel in the next ring position: a plain arrive completes the stage's phase with no bytes
      const int s = fill % kStages;
      mbar_wait(bar_empty0 + 8 * s, ((fill / kStages) & 1) ^ 1);
      item_slot[s] = -1;
      mbar_arrive(bar_full0 + 8 * s);
      // every CTA has made its last claim once all have counted themselves out: the last one resets the ticket
      __threadfence();
      if (atomicAdd(g.tickets + 1, 1) == static_cast<int>(gridDim.x) - 1) {
        g.tickets[0] = 0;
        g.tickets[1] = 0;
      }
    }
  } else {
    // ------------------------------ consumers: wgmma + epilogue ------------------------------
    const int half = wg - 1;
    const int wq = warp & 3;                           // warp inside the warpgroup: rows 16 wq .. 16 wq + 15
    const int et = threadIdx.x - 128;                  // 0..255 inside the consumer group
    const bool issuer = (et == 0);
    int drain = 0;
    int chunk_ctr = 0;                                 // staging double buffer position
    for (;;) {
      // the item's first k-block stage carries its id (the k-block loop below waits on the same phase again)
      mbar_wait(bar_full0 + 8 * (drain % kStages), (drain / kStages) & 1);
      const int item = item_slot[drain % kStages];
      if (item < 0) break;
      const Item it = decode(item, d0, d1);
      const TcProblem& p = g.p[it.prob];
      const CUtensorMap* tcm = it.prob ? &tmC1 : &tmC0;
      const int nsl = p.bn / 64;
      // (a_mn, b_mn) is (0, 0) forward, (0, 1) dA or (1, 1) dW
      const int sel = (p.a_mn * 2 + p.b_mn) * 3 + (nsl == 4 ? 2 : nsl - 1);
      float acc[4][32];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[j][i] = 0.f;
      int prev_s = -1;
      for (int kb = it.kb0; kb < it.kb1; ++kb, ++drain) {
        const int s = drain % kStages;
        mbar_wait(bar_full0 + 8 * s, (drain / kStages) & 1);
        const uint32_t sa = smem_u32(stage0 + s * kStageBytes) + half * 8192;
        const uint32_t sb = smem_u32(stage0 + s * kStageBytes) + kABytes;
        // operand layouts and tile width are fixed per problem: one straight-line wgmma sequence per combination
        switch (sel) {
          case 0: mma_kblock<0, 0, 1>(acc, sa, sb); break;
          case 1: mma_kblock<0, 0, 2>(acc, sa, sb); break;
          case 2: mma_kblock<0, 0, 4>(acc, sa, sb); break;
          case 3: mma_kblock<0, 1, 1>(acc, sa, sb); break;
          case 4: mma_kblock<0, 1, 2>(acc, sa, sb); break;
          case 5: mma_kblock<0, 1, 4>(acc, sa, sb); break;
          case 9: mma_kblock<1, 1, 1>(acc, sa, sb); break;
          case 10: mma_kblock<1, 1, 2>(acc, sa, sb); break;
          default: mma_kblock<1, 1, 4>(acc, sa, sb); break;
        }
        wgmma_commit();
        // one k-block stays in flight: the MMAs of the previous one have completed, so its stage is reusable
        wgmma_wait<1>();
        if (prev_s >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_empty0 + 8 * prev_s);
        }
        prev_s = s;
      }
      wgmma_wait<0>();
      if (prev_s >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty0 + 8 * prev_s);
      }
      const int rl = half * 64 + wq * 16 + (lane >> 2);  // tile row of fragment rows h = 0; h = 1 is 8 further
      const int cl = 2 * (lane & 3);                     // first of this thread's two columns inside 8
      if (p.epi == 0) {
        const __nv_bfloat16* bias = reinterpret_cast<const __nv_bfloat16*>(p.bias);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (j >= nsl) break;
          uint8_t* stg = store0 + (chunk_ctr & 1) * kStoreBytes;
          // the TMA store issued two chunks ago must have finished READING this staging tile
          if (issuer) tma_wait_group_read<1>();
          named_bar_sync(1, kEpiThreads);
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            float b0 = 0.f, b1 = 0.f;
            if (bias) {
              const float2 bf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(
                  bias + it.n_tile * p.bn + j * 64 + jj * 8 + cl));
              b0 = bf.x; b1 = bf.y;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float x0 = acc[j][4 * jj + 2 * h] + b0, x1 = acc[j][4 * jj + 2 * h + 1] + b1;
              if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
              const __nv_bfloat162 o = __floats2bfloat162_rn(x0, x1);
              const int r = rl + 8 * h;
              sts32(smem_u32(stg) + r * 128 + ((jj ^ (r & 7)) << 4) + cl * 2, *reinterpret_cast<const int32_t*>(&o));
            }
          }
          fence_proxy_async();                         // generic-proxy smem writes -> visible to the TMA engine
          named_bar_sync(1, kEpiThreads);
          if (issuer) {
            tma_store_2d(tcm, it.n_tile * p.bn + j * 64, it.m_tile * kBM, smem_u32(stg));
            tma_commit_group();
          }
          ++chunk_ctr;
        }
      } else {
        // split-K partial sums: fp32 vector reductions straight into the gradient buffer
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = it.m_tile * kBM + rl + 8 * h;
          if (row < p.m_valid) {
            float* orow = p.out32 + static_cast<int64_t>(row) * p.ld32 + it.n_tile * p.bn + cl;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (j < nsl) {
#pragma unroll
                for (int jj = 0; jj < 8; ++jj)
                  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(orow + j * 64 + jj * 8),
                               "f"(acc[j][4 * jj + 2 * h]), "f"(acc[j][4 * jj + 2 * h + 1])
                               : "memory");
              }
            }
          }
        }
      }
    }
    if (issuer) tma_wait_group<0>();                   // all stores retired before the CTA exits
  }
}

// ---------------------------------------------------------------------------------------------------
// host side: tensor maps through the driver entry point (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

}  // namespace

// 2-D bf16 row-major tensor [rows, cols] (cols contiguous, row pitch `ld` elements), box {box_cols, box_rows},
// SWIZZLE_128B (box_cols * 2 bytes must be 128), zero fill out of bounds.
int make_tmap_bf16_2d(void* out_map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols,
                      int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return 1;
  cuuint64_t dims[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t strides[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(reinterpret_cast<CUtensorMap*>(out_map), CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2,
                        const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 2;
}

size_t tc_gemm_smem_bytes() { return kGemmSmem; }

void launch_tc_gemm(const TcGemmLaunch& L, int num_sms, cudaStream_t s) {
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFuncSetAttribute(k_tc_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kGemmSmem));
  });
  // per-device attribute: cheap to repeat, required on every device the kernel runs on
  cudaFuncSetAttribute(k_tc_gemm, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kGemmSmem));
  int grid = num_sms;
  if (L.max_items > 0 && L.max_items < grid) grid = L.max_items;
  const CUtensorMap* m = reinterpret_cast<const CUtensorMap*>(L.maps);
  launch_k(k_tc_gemm, dim3(grid), dim3(kGemmThreads), kGemmSmem, s, m[0], m[1], m[2], m[3], m[4], m[5], L.args);
}

}  // namespace glt
