// Exact top-K link retrieval (models/link_rank.py: link_topk): for every query q of a call, the k candidates c of
// [lo, hi) with the largest <emb[q], emb[c]>, ordered by (score desc, id asc), never returning q itself or an id of
// q's exclusion row.
//
// k_link_topk: grid (query tiles of 64 rows) x (candidate splits); one CTA sweeps its split's candidate tiles of 64
// rows in ascending id order.  160 threads:
//   warp 4 (one lane)   TMA producer: the query tile (all of d, once) into resident smem, then one 64 x 64 bf16
//                       k-block of candidates per ring stage (SWIZZLE_128B; columns past d and rows past hi read 0)
//   warpgroup 0         wgmma.m64n64k16 over the k-blocks of a tile (fp32 accumulators), then selection:
//                       a score below its row's current k-th value, or at an excluded column, is dropped in
//                       registers; the rest go to the row's queue (128 slots).  When a row's queue holds more than
//                       64 entries after a tile, every row's queue is merged into its sorted list (one warp per row,
//                       by rank: each element's position is the number of elements of list and queue above it).
// Threads 0..63 own the exclusion cursor of rows 0..63: the sorted row is entered by binary search at the split's
// first id and only moves forward, so a hub row costs its degree once per CTA, and each tile gets a 64-bit mask of the
// columns to drop (exclusion ids, the query itself, ids >= hi).
//
// Selection compares 64-bit keys: the order-preserving bits of the (sign-canonical) fp32 score above the complemented
// id, so a larger key is a better (score desc, id asc) candidate and all keys of one query are distinct.  Every score
// is computed by the same instruction sequence whatever the split, so the result is bitwise identical for any split
// count; k_link_topk_merge merges the splits' sorted lists the same way and decodes (id, score).
#include <cuda.h>

#include <cstdint>

#include "launch_utils.h"
#include "tc_utils.cuh"

namespace glt {

namespace {

using namespace tc;

constexpr int kTileQ = 64;                 // query rows per CTA
constexpr int kTileC = 64;                 // candidate rows per tile
constexpr int kBlockBytes = 64 * 128;      // one 64-row x 64-column bf16 k-block
constexpr int kQueue = 128;                // queue slots per row: at most kTileC arrive per tile
constexpr int kMergeAt = kQueue - kTileC;  // merge once a row holds more than this after a tile
constexpr int kThreads = 160;
constexpr int kConsumers = 128;

__device__ __forceinline__ uint64_t make_key(float s, int64_t id) {
  uint32_t u = __float_as_uint(s + 0.f);   // -0 -> +0
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return (static_cast<uint64_t>(u) << 32) | static_cast<uint32_t>(~static_cast<uint32_t>(id));
}
__device__ __forceinline__ float key_score(uint64_t key) {
  const uint32_t u = static_cast<uint32_t>(key >> 32);
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7FFFFFFFu) : ~u);
}
__device__ __forceinline__ int64_t key_id(uint64_t key) {
  return static_cast<int64_t>(~static_cast<uint32_t>(key));
}

// entries of the descending list l[0, n) greater than x
__device__ __forceinline__ int count_above(const uint64_t* l, int n, uint64_t x) {
  int a = 0, b = n;
  while (a < b) {
    const int m = (a + b) >> 1;
    if (l[m] > x) a = m + 1; else b = m;
  }
  return a;
}

struct Smem {   // carve-up of the dynamic shared memory (A and the ring 1024-aligned for SWIZZLE_128B)
  uint8_t* a;          // kb x 8 KB query k-blocks
  uint8_t* ring;       // stages x 8 KB candidate k-blocks
  uint64_t* list;      // [64][k] sorted keys, 0 = empty
  uint64_t* queue;     // [64][kQueue]
  uint64_t* mask;      // [64] dropped columns of the current tile
  int* cnt;            // [64] queue fill
  float* thr;          // [64] score of the k-th list entry (-inf while the list is not full)
  int* flag;           // [2] a queue passed kMergeAt, by tile parity
  uint64_t* bars;      // bar_a, full[stages], empty[stages]
};

__host__ __device__ inline size_t smem_layout(int kb, int stages, int k, uintptr_t base, Smem* s) {
  uintptr_t p = (base + 1023) & ~uintptr_t(1023);
  const uintptr_t p0 = base;
  if (s) s->a = reinterpret_cast<uint8_t*>(p);
  p += static_cast<size_t>(kb) * kBlockBytes;
  if (s) s->ring = reinterpret_cast<uint8_t*>(p);
  p += static_cast<size_t>(stages) * kBlockBytes;
  if (s) s->list = reinterpret_cast<uint64_t*>(p);
  p += static_cast<size_t>(kTileQ) * k * 8;
  if (s) s->queue = reinterpret_cast<uint64_t*>(p);
  p += static_cast<size_t>(kTileQ) * kQueue * 8;
  if (s) s->mask = reinterpret_cast<uint64_t*>(p);
  p += kTileQ * 8;
  if (s) s->bars = reinterpret_cast<uint64_t*>(p);
  p += (1 + 2 * stages) * 8;
  if (s) s->cnt = reinterpret_cast<int*>(p);
  p += kTileQ * 4;
  if (s) s->thr = reinterpret_cast<float*>(p);
  p += kTileQ * 4;
  if (s) s->flag = reinterpret_cast<int*>(p);
  p += 2 * 4;
  return static_cast<size_t>(p - p0) + (base == 0 ? 1023 : 0);   // worst-case alignment slack when sizing
}

// Merge row r's queue into its list (one warp).  Old list entries keep their order and shift down by the queue
// entries above them; a queue entry lands at (list entries above it) + (queue entries above it).  Keys in list and
// queue are distinct (empties, key 0, sit only at the list's tail), so the positions are distinct.
__device__ void merge_row(const Smem& sm, int r, int k, int lane) {
  const int c = sm.cnt[r];
  if (c == 0) return;
  uint64_t* l = sm.list + static_cast<size_t>(r) * k;
  const uint64_t* q = sm.queue + static_cast<size_t>(r) * kQueue;
  uint64_t lk[4], qk[4];
  int lr[4], qr[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int li = lane + 32 * i, qi = lane + 32 * i;
    lk[i] = li < k ? l[li] : 0;
    qk[i] = qi < c ? q[qi] : 0;
    lr[i] = qr[i] = 0;
  }
  for (int j = 0; j < c; ++j) {   // all lanes read the same q[j]: a broadcast
    const uint64_t x = q[j];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      lr[i] += x > lk[i];
      qr[i] += x > qk[i];
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    lr[i] += lane + 32 * i;
    if (lane + 32 * i < c) qr[i] += count_above(l, k, qk[i]);
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    if (lane + 32 * i < k && lr[i] < k) l[lr[i]] = lk[i];
    if (lane + 32 * i < c && qr[i] < k) l[qr[i]] = qk[i];
  }
  __syncwarp();
  if (lane == 0) {
    sm.cnt[r] = 0;
    const uint64_t last = l[k - 1];
    sm.thr[r] = last ? key_score(last) : -INFINITY;
  }
}

__global__ void __launch_bounds__(kThreads, 1)
k_link_topk(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmC, const LinkTopkArgs a,
            int kb, int stages, int tiles_per_split) {
  extern __shared__ uint8_t smem_raw[];
  Smem sm;
  smem_layout(kb, stages, a.k, reinterpret_cast<uintptr_t>(smem_raw), &sm);
  const int k = a.k;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, split = blockIdx.y;
  const int64_t n_cand = a.hi - a.lo;
  const int64_t n_tiles = (n_cand + kTileC - 1) / kTileC;
  const int64_t t0 = static_cast<int64_t>(split) * tiles_per_split;
  const int64_t t1 = min(n_tiles, t0 + tiles_per_split);
  const uint32_t bar_a = smem_u32(sm.bars);
  const uint32_t full0 = bar_a + 8, empty0 = bar_a + 8 + 8 * stages;

  if (threadIdx.x == 0) {
    mbar_init(bar_a, 1);
    for (int s = 0; s < stages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 4);   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    prefetch_tmap(&tmQ);
    prefetch_tmap(&tmC);
  }
  for (int i = threadIdx.x; i < kTileQ * k; i += kThreads) sm.list[i] = 0;
  if (threadIdx.x < kTileQ) {
    sm.cnt[threadIdx.x] = 0;
    sm.thr[threadIdx.x] = -INFINITY;
  }
  if (threadIdx.x < 2) sm.flag[threadIdx.x] = 0;
  __syncthreads();
  pdl_wait();

  if (warp == 4) {
    if (lane == 0) {
      mbar_expect_tx(bar_a, static_cast<uint32_t>(kb) * kBlockBytes);
      for (int b = 0; b < kb; ++b) tma_load_2d(smem_u32(sm.a) + b * kBlockBytes, &tmQ, b * 64, qt * kTileQ, bar_a);
      int fill = 0;
      for (int64_t t = t0; t < t1; ++t) {
        for (int b = 0; b < kb; ++b, ++fill) {
          const int s = fill % stages;
          mbar_wait(empty0 + 8 * s, ((fill / stages) & 1) ^ 1);
          mbar_expect_tx(full0 + 8 * s, kBlockBytes);
          tma_load_2d(smem_u32(sm.ring) + s * kBlockBytes, &tmC, b * 64, static_cast<int>(t * kTileC), full0 + 8 * s);
        }
      }
    }
    return;
  }

  // ---- consumers ----
  const int tid = threadIdx.x;
  // exclusion cursor of row tid (threads 0..63)
  int64_t qid = -1, pos = 0, end = 0, nxt = INT64_MAX;
  int part = 0;
  if (tid < kTileQ) {
    const int64_t row = static_cast<int64_t>(qt) * kTileQ + tid;
    if (row < a.n) {
      qid = a.queries[row];
      {
        const RowRef rr = load_row(a.g, qid);   // no shards, or qid past the graph's rows: nothing excluded
        if (rr.deg > 0) {
          part = rr.part;
          pos = rr.start;
          end = rr.start + rr.deg;
          const int64_t first = a.lo + t0 * kTileC;   // enter at the split's first id
          int64_t lo = pos, hi = end;
          while (lo < hi) {
            const int64_t m = (lo + hi) >> 1;
            if (load_col(a.g, part, m) < first) lo = m + 1; else hi = m;
          }
          pos = lo;
          nxt = pos < end ? load_col(a.g, part, pos) : INT64_MAX;
        }
      }
    }
  }
  const int r0 = 16 * warp + (lane >> 2);   // accumulator rows r0, r0 + 8; columns 8 j + 2 (lane % 4) + e
  const int cl = 2 * (lane & 3);
  mbar_wait(bar_a, 0);

  int drain = 0;
  for (int64_t t = t0; t < t1; ++t) {
    const int64_t g0 = a.lo + t * kTileC;
    if (tid < kTileQ) {
      uint64_t m = 0;
      if (qid < 0) {
        m = ~0ull;
      } else {
        while (nxt < g0 + kTileC) {
          if (nxt >= g0) m |= 1ull << (nxt - g0);
          ++pos;
          nxt = pos < end ? load_col(a.g, part, pos) : INT64_MAX;
        }
        if (qid >= g0 && qid < g0 + kTileC) m |= 1ull << (qid - g0);
        if (g0 + kTileC > a.hi) m |= ~0ull << (a.hi - g0);
      }
      sm.mask[tid] = m;
    }
    __syncwarp();                                // the wgmma instructions below are warp-aligned

    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    int prev_s = -1;
    for (int b = 0; b < kb; ++b, ++drain) {
      const int s = drain % stages;
      mbar_wait(full0 + 8 * s, (drain / stages) & 1);
      const uint32_t sa = smem_u32(sm.a) + b * kBlockBytes;
      const uint32_t sb = smem_u32(sm.ring) + s * kBlockBytes;
      wgmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4)
        wgmma_m64n64k16_bf16<0, 0>(acc, make_sw128_desc_lbo(sa + 32 * k4, 16, 1024),
                                   make_sw128_desc_lbo(sb + 32 * k4, 16, 1024), 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_s >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * prev_s);
      }
      prev_s = s;
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * prev_s);

    named_bar_sync(1, kConsumers);              // masks of this tile, thresholds of the last merge
    if (tid == 0) sm.flag[(t + 1) & 1] = 0;     // read for tile t - 1 by every thread before this barrier
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = r0 + 8 * h;
      const float thr = sm.thr[r];
      const uint64_t m = sm.mask[r];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = 8 * j + cl + e;
          const float sc = acc[4 * j + 2 * h + e];
          if (sc >= thr && !((m >> c) & 1)) {
            const int slot = atomicAdd(sm.cnt + r, 1);
            sm.queue[r * kQueue + slot] = make_key(sc, g0 + c);
            if (slot == kMergeAt) sm.flag[t & 1] = 1;
          }
        }
      }
    }
    named_bar_sync(1, kConsumers);
    if (sm.flag[t & 1] || t + 1 == t1) {
      for (int r = warp; r < kTileQ; r += 4) merge_row(sm, r, k, lane);
      named_bar_sync(1, kConsumers);
    }
  }

  // partial list of this split: keys [split][row][k]
  for (int i = tid; i < kTileQ * k; i += kConsumers) {
    const int64_t row = static_cast<int64_t>(qt) * kTileQ + i / k;
    if (row < a.n) a.part_keys[(static_cast<int64_t>(split) * a.n + row) * k + i % k] = sm.list[i];
  }
}

// One warp per query row: the union of the splits' sorted lists, by rank; slots past the number of entries read
// (id -1, -inf).
__global__ void __launch_bounds__(256) k_link_topk_merge(const uint64_t* part_keys, int64_t n, int k, int splits,
                                                         int64_t* ids, float* scores) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  for (int64_t row = (blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x) >> 5; row < n;
       row += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    int valid = 0;
    for (int s = 0; s < splits; ++s) valid += count_above(part_keys + (s * n + row) * k, k, 0);
    for (int s = 0; s < splits; ++s) {
      const uint64_t* l = part_keys + (s * n + row) * k;
      for (int i = lane; i < k; i += 32) {
        const uint64_t x = l[i];
        if (x == 0) continue;
        int rank = i;
        for (int o = 0; o < splits && rank < k; ++o)
          if (o != s) rank += count_above(part_keys + (o * n + row) * k, k, x);
        if (rank < k) {
          ids[row * k + rank] = key_id(x);
          scores[row * k + rank] = key_score(x);
        }
      }
    }
    for (int i = min(valid, k) + lane; i < k; i += 32) {
      ids[row * k + i] = -1;
      scores[row * k + i] = -INFINITY;
    }
  }
}

}  // namespace

int link_topk_stages(int d, int k, size_t smem_limit) {
  const int kb = (d + 63) / 64;
  for (int stages = 8; stages >= 2; --stages)
    if (smem_layout(kb, stages, k, 0, nullptr) <= smem_limit) return stages;
  return 0;
}

size_t link_topk_smem_bytes(int d, int k, int stages) { return smem_layout((d + 63) / 64, stages, k, 0, nullptr); }

int link_topk_ctas_per_sm(int d, int k, int stages) {
  const size_t smem = link_topk_smem_bytes(d, k, stages);
  cudaFuncSetAttribute(k_link_topk, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  int ctas = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, k_link_topk, kThreads, smem) != cudaSuccess) ctas = 1;
  return ctas < 1 ? 1 : ctas;
}

void launch_link_topk(const LinkTopkLaunch& L, cudaStream_t s) {
  const LinkTopkArgs& a = L.args;
  const int kb = (a.d + 63) / 64;
  const size_t smem = link_topk_smem_bytes(a.d, a.k, L.stages);
  cudaFuncSetAttribute(k_link_topk, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  const int64_t q_tiles = (a.n + kTileQ - 1) / kTileQ;
  const CUtensorMap* m = reinterpret_cast<const CUtensorMap*>(L.maps);
  launch_k(k_link_topk, dim3(static_cast<unsigned>(q_tiles), L.splits), dim3(kThreads), smem, s, m[0], m[1], a, kb,
           L.stages, L.tiles_per_split);
  launch_k(k_link_topk_merge, dim3(grid_for(a.n * 32, 256)), dim3(256), 0, s,
           reinterpret_cast<const uint64_t*>(a.part_keys), a.n, a.k, L.splits, a.ids, a.scores);
}

}  // namespace glt
