// Transposed per-batch adjacency and the atomics-free backward of the mean aggregation.
//
// The GraphSAGE engine's backward of the aggregation.  It replaced a zero fill, an fp32-atomic scatter over the edges
// and a ReLU/cast kernel: on an H100 (products shape, bench.py) the step took 0.297 ms with it and 0.409 ms with
// that scatter formulation.
//
//   build (sampling stream, overlapped with the training of the previous batch):
//     k_tr_count   in-degree histogram of the local source ids, one histogram per hop
//     k_tr_scan*   exclusive scan over sources (3-phase, fixed grids, sizes read from the device)
//     k_tr_fill    targets appended per source, hop 0 first, so a layer that uses hops 0..h reads
//                  the first cnt_upto[h][s] entries of the segment
//   use (training stream):
//     k_sage_gather_bwd  one lane group per SOURCE row: self gradient + sum of the incoming mean
//                  gradients scaled by 1/deg(target), ReLU mask, bf16 cast, fused bias column sums.
//
// The reference has no counterpart (PyG autograd scatter on the host-built COO).
#include "device_utils.cuh"
#include "launch_utils.h"

#ifndef GLT_GATHER_U
#define GLT_GATHER_U 2     // rows per lane group in flight (U = 4: spills at 128 registers, 56 us vs 42 us)
#endif
#ifndef GLT_GATHER_HB
#define GLT_GATHER_HB 8    // row loads in flight in the > 2 in-edges loop
#endif

namespace glt {

namespace {

constexpr int kScanBlock = 256;
constexpr int kScanItems = 4;  // elements per thread -> 1024 per block

__global__ void k_tr_count(TransposeArgs a, int hop) {
  const int f_begin = a.cum[hop];
  const int n_rows = min(a.cum[hop + 1] - f_begin, a.cap_rows[hop]);
  const int k = a.k[hop];
  const int64_t n = static_cast<int64_t>(n_rows) * k;
  int32_t* cnt = a.cnt + static_cast<int64_t>(hop) * a.cap_nodes;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / k), j = static_cast<int>(i % k);
    if (j >= a.deg[f_begin + r]) continue;
    const int32_t s = a.ell[hop][i];
    if (s >= 0 && s < a.cap_nodes) atomicAdd(cnt + s, 1);
  }
}

// phase 1: per-block exclusive scan of total[s] = sum_h cnt[h][s]; cnt becomes cumulative over hops
__global__ void __launch_bounds__(kScanBlock) k_tr_scan1(TransposeArgs a) {
  __shared__ int s_warp[kScanBlock / 32];
  const int base = (blockIdx.x * kScanBlock + threadIdx.x) * kScanItems;
  int v[kScanItems];
  int local = 0;
#pragma unroll
  for (int q = 0; q < kScanItems; ++q) {
    const int s = base + q;
    int tot = 0;
    if (s < a.cap_nodes) {
      for (int h = 0; h < a.n_hops; ++h) {
        int32_t* c = a.cnt + static_cast<int64_t>(h) * a.cap_nodes + s;
        tot += *c;
        *c = tot;  // cumulative over hops 0..h
      }
    }
    v[q] = local;  // exclusive inside the thread
    local += tot;
  }
  // block-wide exclusive scan of `local`
  int x = local;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) s_warp[w] = x;
  __syncthreads();
  if (w == 0) {
    int t = lane < kScanBlock / 32 ? s_warp[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, t, o);
      if (lane >= o) t += y;
    }
    if (lane < kScanBlock / 32) s_warp[lane] = t;  // inclusive warp totals
  }
  __syncthreads();
  const int warp_off = w > 0 ? s_warp[w - 1] : 0;
  const int thread_excl = warp_off + x - local;
#pragma unroll
  for (int q = 0; q < kScanItems; ++q) {
    const int s = base + q;
    if (s < a.cap_nodes) a.off[s] = thread_excl + v[q];
  }
  if (threadIdx.x == kScanBlock - 1) a.block_sums[blockIdx.x] = warp_off + x;  // block total
}

// phase 2: one block turns the block totals into exclusive block offsets (in place) + grand total
__global__ void __launch_bounds__(1024) k_tr_scan2(TransposeArgs a, int n_blocks) {
  __shared__ int s_warp[32];
  __shared__ int s_carry;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int base = 0; base < n_blocks; base += 1024) {
    const int i = base + threadIdx.x;
    const int val = i < n_blocks ? a.block_sums[i] : 0;
    int x = val;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[w] = x;
    __syncthreads();
    if (w == 0) {
      int t = s_warp[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, t, o);
        if (lane >= o) t += y;
      }
      s_warp[lane] = t;
    }
    __syncthreads();
    const int incl = (w > 0 ? s_warp[w - 1] : 0) + x;
    const int carry = s_carry;
    if (i < n_blocks) a.block_sums[i] = carry + incl - val;  // exclusive
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = carry + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) a.off[a.cap_nodes] = s_carry;  // total number of transposed edges
}

// phase 3: add the block offsets
__global__ void __launch_bounds__(kScanBlock) k_tr_scan3(TransposeArgs a) {
  const int add = a.block_sums[blockIdx.x];
  const int base = (blockIdx.x * kScanBlock + threadIdx.x) * kScanItems;
#pragma unroll
  for (int q = 0; q < kScanItems; ++q)
    if (base + q < a.cap_nodes) a.off[base + q] += add;
}

__global__ void k_tr_fill(TransposeArgs a, int hop) {
  const int f_begin = a.cum[hop];
  const int n_rows = min(a.cum[hop + 1] - f_begin, a.cap_rows[hop]);
  const int k = a.k[hop];
  const int64_t n = static_cast<int64_t>(n_rows) * k;
  // entries of hop h start after the entries of the earlier hops: offset by the cumulative count
  const int32_t* before = hop > 0 ? a.cnt + static_cast<int64_t>(hop - 1) * a.cap_nodes : nullptr;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / k), j = static_cast<int>(i % k);
    if (j >= a.deg[f_begin + r]) continue;
    const int32_t s = a.ell[hop][i];
    if (s < 0 || s >= a.cap_nodes) continue;
    const int pos = a.off[s] + (before ? before[s] : 0) + atomicAdd(a.cursor + static_cast<int64_t>(hop) * a.cap_nodes + s, 1);
    if (pos < a.cap_edges) a.tgt[pos] = f_begin + r;
  }
}

// one record per source for the backward gather: {segment start, first two in-neighbours, total in-edges} + their 1/deg
__global__ void k_tr_meta(TransposeArgs a) {
  const int n_nodes = min(a.cum[a.n_hops + 1], a.cap_nodes);
  const int32_t* total = a.cnt + static_cast<int64_t>(a.n_hops - 1) * a.cap_nodes;   // cumulative over all hops
  for (int s = blockIdx.x * blockDim.x + threadIdx.x; s < a.cap_nodes; s += gridDim.x * blockDim.x) {
    int4 m = make_int4(0, -1, -1, 0);
    float2 iv = make_float2(0.f, 0.f);
    if (s < n_nodes) {
      m.x = a.off[s];
      m.w = total[s];
      if (m.w > 0 && m.x < a.cap_edges) {
        m.y = a.tgt[m.x];
        const int dg = (m.y >= 0 && m.y < a.cap_nodes) ? a.deg[m.y] : 0;
        iv.x = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
      }
      if (m.w > 1 && m.x + 1 < a.cap_edges) {
        m.z = a.tgt[m.x + 1];
        const int dg = (m.z >= 0 && m.z < a.cap_nodes) ? a.deg[m.z] : 0;
        iv.y = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
      }
    }
    reinterpret_cast<int4*>(a.meta)[s] = m;
    reinterpret_cast<float2*>(a.meta_inv)[s] = iv;
  }
}

// ------------------------------------------------------------------------------------------
// Gather-style backward of the mean aggregation:
//   dPre[s] = relu'(Z[s]) * gscale * (dA_self[s] + sum_{t in in(s)} dA_mean[t] / deg[t])       (+ bias column sums)
//   (without Z there is no mask, but gscale -- the dropout rescale -- still applies)
//   * 32 consecutive source rows form a chunk served by a TEAM of warps; every warp of the team reads the chunk's
//     records ({count, segment start, first two in-neighbours, their 1/deg}: built by k_tr_meta on the sampling
//     stream, prefetched one chunk ahead) and takes every TEAM-th row;
//   * per row the ReLU-mask row, the "self" gradient row and the first two incoming "mean" gradient rows are issued
//     for U rows before the first add (in-batch in-degrees at products shape: mean 1.4, p90 2, p99 7, max ~160);
//   * further in-edges are fetched HB rows at a time; rows with more than kHeavy in-edges (RMAT hubs) are split over
//     the TEAM warps and combined through shared memory, so no warp is left walking a hub after the grid has drained;
//   * bias gradient: per-lane running column sums -> one shared slice per warp -> one red.global.add.v4.f32 per four
//     columns per CTA.
// Earlier variants were slower: one row per warp with dependent loads and same-address atomics for the column sums,
// and staging all rows through shared memory with cp.async (128 KB / CTA).  In situ on an H100 (products shape,
// bench.py --kernel-times) this kernel takes 58 us for layer 2 (44 k source rows x 256) and 15 us for layer 3.
template <int LPR, int VPL>
__global__ void __launch_bounds__(256, 2) k_sage_gather_bwd(SageGatherBwdArgs a) {
  pdl_enter();
  extern __shared__ float s_col[];  // [warps per block][d]
  constexpr int RPW = 32 / LPR;     // rows a warp works on concurrently (one per lane group)
  constexpr int U = (VPL == 1) ? GLT_GATHER_U : 1;
  constexpr int TEAM = (LPR == 32) ? 4 : (LPR == 16 ? 2 : 1);
  constexpr int Q = 32 / (TEAM * RPW);   // rows per lane group per chunk
  constexpr int kHeavy = 24;
  constexpr bool kSplitHeavy = (TEAM > 1 && LPR == 32);
  constexpr int HB = (VPL == 1) ? GLT_GATHER_HB : (VPL == 2 ? 4 : 2);
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int S = min(a.cum[a.n_hops_targets + 1], a.cap_src);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.d >> 3;
  const float gscale = a.gscale;
  float csum[VPL][8];
#pragma unroll
  for (int v = 0; v < VPL; ++v)
#pragma unroll
    for (int i = 0; i < 8; ++i) csum[v][i] = 0.f;
  const uint8_t* dA = reinterpret_cast<const uint8_t*>(a.dA);
  const uint8_t* Zb = reinterpret_cast<const uint8_t*>(a.Z);
  const int64_t a_row = static_cast<int64_t>(a.d) * 4;  // bytes of one [mean | self] row
  const int64_t z_row = static_cast<int64_t>(a.d) * 2;
  const uint4 zero4 = make_uint4(0, 0, 0, 0);
  const int n_teams = gridDim.x * wpb / TEAM;
  const int member = warp % TEAM;
  int pf_n = 0;
  int4 pf_m = make_int4(0, -1, -1, 0);
  float2 pf_i = make_float2(0.f, 0.f);
  {
    const int s0 = ((blockIdx.x * wpb + warp) / TEAM) * 32 + lane;
    if (s0 < S) {
      pf_n = a.cnt_upto[s0];
      pf_m = reinterpret_cast<const int4*>(a.meta)[s0];
      pf_i = reinterpret_cast<const float2*>(a.meta_inv)[s0];
    }
  }
  for (int base = ((blockIdx.x * wpb + warp) / TEAM) * 32; base < a.cap_src; base += n_teams * 32) {
    // ---- records of the chunk (lane i <-> row base + i); the next chunk's are requested right away
    int m_n = 0, m_e0 = 0, m_t0 = -1, m_t1 = -1;
    float m_i0 = 0.f, m_i1 = 0.f;
    {
      if (base + lane < S) {
        m_n = pf_n;
        m_e0 = pf_m.x;
        // the record lists the first two in-neighbours over ALL hops; this layer uses the first m_n of the segment
        if (m_n > 0 && pf_m.y >= 0 && pf_m.y < T) { m_t0 = pf_m.y; m_i0 = pf_i.x; }
        if (m_n > 1 && pf_m.z >= 0 && pf_m.z < T) { m_t1 = pf_m.z; m_i1 = pf_i.y; }
      }
      const int sn = base + n_teams * 32 + lane;
      if (sn < S) {
        pf_n = a.cnt_upto[sn];
        pf_m = reinterpret_cast<const int4*>(a.meta)[sn];
        pf_i = reinterpret_cast<const float2*>(a.meta_inv)[sn];
      }
    }
    const unsigned heavy_mask = kSplitHeavy ? __ballot_sync(0xffffffffu, m_n > kHeavy) : 0u;  // same in the whole team
#pragma unroll 1
    for (int q0 = 0; q0 < Q; q0 += U) {
      int s_[U], n_[U], e0_[U], t0_[U], t1_[U];
      float i0_[U], i1_[U];
      uint4 vz[U][VPL], vs[U][VPL], v0[U][VPL], v1[U][VPL];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int q = q0 + u;
        const int rr = min(((q * RPW + gw) * TEAM + member), 31);
        s_[u] = (q < Q && !((heavy_mask >> rr) & 1u)) ? base + rr : a.cap_src;   // no such row / done by the team
        n_[u] = __shfl_sync(0xffffffffu, m_n, rr);
        e0_[u] = __shfl_sync(0xffffffffu, m_e0, rr);
        t0_[u] = __shfl_sync(0xffffffffu, m_t0, rr);
        t1_[u] = __shfl_sync(0xffffffffu, m_t1, rr);
        i0_[u] = __shfl_sync(0xffffffffu, m_i0, rr);
        i1_[u] = __shfl_sync(0xffffffffu, m_i1, rr);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s_[u];
        const bool live = s < S;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          const bool ok = live && c < nvec;
          vz[u][v] = (ok && Zb) ? ld_nc_v4(Zb + s * z_row + c * 16) : zero4;
          vs[u][v] = (ok && s < T) ? ld_nc_v4(dA + s * a_row + z_row + c * 16) : zero4;
          v0[u][v] = (ok && t0_[u] >= 0) ? ld_nc_v4(dA + t0_[u] * a_row + c * 16) : zero4;
          v1[u][v] = (ok && t1_[u] >= 0) ? ld_nc_v4(dA + t1_[u] * a_row + c * 16) : zero4;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int s = s_[u];
        if (s >= a.cap_src) continue;
        uint8_t* o = reinterpret_cast<uint8_t*>(a.dPre) + s * z_row;
        float acc[VPL][8];
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          float tmp[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) { acc[v][i] = 0.f; tmp[i] = 0.f; }
          bf16x8_accum(vs[u][v], acc[v]);
          bf16x8_accum(v0[u][v], tmp);
#pragma unroll
          for (int i = 0; i < 8; ++i) { acc[v][i] += tmp[i] * i0_[u]; tmp[i] = 0.f; }
          bf16x8_accum(v1[u][v], tmp);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[v][i] += tmp[i] * i1_[u];
        }
        // rows with more than two in-edges: LPR in-neighbours resolved at a time, HB row loads in flight
        for (int j0 = 2; j0 < n_[u]; j0 += LPR) {
          int my_t = -1;
          float my_inv = 0.f;
          if (j0 + gl < n_[u]) {
            const int t = a.tgt[e0_[u] + j0 + gl];
            if (t >= 0 && t < T) {
              const int dg = a.deg[t];
              my_t = t;
              my_inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
            }
          }
          const int cnt = min(LPR, n_[u] - j0);
          for (int jb = 0; jb < cnt; jb += HB) {
            uint4 hv[HB][VPL];
            float hi[HB];
#pragma unroll
            for (int h = 0; h < HB; ++h) {
              const int jj = min(jb + h, LPR - 1);
              const int t = __shfl_sync(gmask, my_t, jj, LPR);
              const float inv = __shfl_sync(gmask, my_inv, jj, LPR);
              const bool ok = (jb + h < cnt) && t >= 0;
              hi[h] = ok ? inv : 0.f;
#pragma unroll
              for (int v = 0; v < VPL; ++v) {
                const int c = v * LPR + gl;
                hv[h][v] = (ok && c < nvec) ? ld_nc_v4(dA + t * a_row + c * 16) : zero4;
              }
            }
#pragma unroll
            for (int h = 0; h < HB; ++h)
#pragma unroll
              for (int v = 0; v < VPL; ++v) {
                float tmp[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) tmp[i] = 0.f;
                bf16x8_accum(hv[h][v], tmp);
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[v][i] += tmp[i] * hi[h];
              }
          }
        }
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c >= nvec) continue;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[v][i] *= gscale;
          if (Zb) {
            float z[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) z[i] = 0.f;
            bf16x8_accum(vz[u][v], z);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[v][i] = z[i] > 0.f ? acc[v][i] : 0.f;
          }
          const uint4 packed = pack_bf16x8(acc[v], 1.f);   // rows in [S, cap_src) come out as zeros
          reinterpret_cast<uint4*>(o)[c] = packed;
          if (a.colsum) {  // sum exactly what the GEMMs will see (bf16-rounded)
            float r[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) r[i] = 0.f;
            bf16x8_accum(packed, r);
#pragma unroll
            for (int i = 0; i < 8; ++i) csum[v][i] += r[i];
          }
        }
      }
    }
    if constexpr (kSplitHeavy) {
      // ---- hub rows of the chunk: the TEAM warps split the in-edges, the row's owner combines the partial sums
      const int bar_id = 1 + warp / TEAM;
      unsigned hm = heavy_mask;
      while (hm) {
        const int rr = __ffs(hm) - 1;
        hm &= hm - 1;
        const int s = base + rr;
        const int n = __shfl_sync(0xffffffffu, m_n, rr);
        const int e0 = __shfl_sync(0xffffffffu, m_e0, rr);
        float acc[VPL][8];
#pragma unroll
        for (int v = 0; v < VPL; ++v)
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[v][i] = 0.f;
        for (int j0 = member * 32; j0 < n; j0 += TEAM * 32) {   // this warp's share: every TEAM-th block of 32
          int my_t = -1;
          float my_inv = 0.f;
          if (j0 + lane < n) {
            const int t = a.tgt[e0 + j0 + lane];
            if (t >= 0 && t < T) {
              const int dg = a.deg[t];
              my_t = t;
              my_inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
            }
          }
          const int cnt = min(32, n - j0);
          for (int jb = 0; jb < cnt; jb += HB) {
            uint4 hv[HB][VPL];
            float hi[HB];
#pragma unroll
            for (int h = 0; h < HB; ++h) {
              const int jj = min(jb + h, 31);
              const int t = __shfl_sync(0xffffffffu, my_t, jj);
              const float inv = __shfl_sync(0xffffffffu, my_inv, jj);
              const bool ok = (jb + h < cnt) && t >= 0;
              hi[h] = ok ? inv : 0.f;
#pragma unroll
              for (int v = 0; v < VPL; ++v) {
                const int c = v * 32 + lane;
                hv[h][v] = (ok && c < nvec) ? ld_nc_v4(dA + t * a_row + c * 16) : zero4;
              }
            }
#pragma unroll
            for (int h = 0; h < HB; ++h)
#pragma unroll
              for (int v = 0; v < VPL; ++v) {
                float tmp[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) tmp[i] = 0.f;
                bf16x8_accum(hv[h][v], tmp);
#pragma unroll
                for (int i = 0; i < 8; ++i) acc[v][i] += tmp[i] * hi[h];
              }
          }
        }
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * 32 + lane;
          if (c < nvec) {
#pragma unroll
            for (int i = 0; i < 8; ++i) s_col[warp * a.d + c * 8 + i] = acc[v][i];
          }
        }
        asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(TEAM * 32) : "memory");
        if (member == rr % TEAM) {
          uint8_t* o = reinterpret_cast<uint8_t*>(a.dPre) + s * z_row;
          const int w0 = warp - member;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int c = v * 32 + lane;
            if (c >= nvec) continue;
            float tot[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) tot[i] = 0.f;
            if (s < T) bf16x8_accum(ld_nc_v4(dA + s * a_row + z_row + c * 16), tot);
            for (int w = 0; w < TEAM; ++w)
#pragma unroll
              for (int i = 0; i < 8; ++i) tot[i] += s_col[(w0 + w) * a.d + c * 8 + i];
#pragma unroll
            for (int i = 0; i < 8; ++i) tot[i] *= gscale;
            if (Zb) {
              float z[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) z[i] = 0.f;
              bf16x8_accum(ld_nc_v4(Zb + s * z_row + c * 16), z);
#pragma unroll
              for (int i = 0; i < 8; ++i) tot[i] = z[i] > 0.f ? tot[i] : 0.f;
            }
            const uint4 packed = pack_bf16x8(tot, 1.f);
            reinterpret_cast<uint4*>(o)[c] = packed;
            if (a.colsum) {
              float r[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) r[i] = 0.f;
              bf16x8_accum(packed, r);
#pragma unroll
              for (int i = 0; i < 8; ++i) csum[v][i] += r[i];
            }
          }
        }
        asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(TEAM * 32) : "memory");   // slices may be reused
      }
    }
  }
  __syncthreads();   // the per-warp slices change their role
  if (a.colsum) {
    // lane groups of a warp hold the same columns: fold them, then one slice per warp, then one red.v4 per 4 columns
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) csum[v][i] += __shfl_xor_sync(0xffffffffu, csum[v][i], o);
    if (gw == 0) {
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec) {
#pragma unroll
          for (int i = 0; i < 8; ++i) s_col[warp * a.d + c * 8 + i] = csum[v][i];
        }
      }
    }
    __syncthreads();
    for (int c4 = threadIdx.x; c4 < a.d / 4; c4 += blockDim.x) {
      float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int w = 0; w < wpb; ++w) {
        const float4 x = *reinterpret_cast<const float4*>(s_col + w * a.d + c4 * 4);
        t.x += x.x; t.y += x.y; t.z += x.z; t.w += x.w;
      }
      if (t.x != 0.f || t.y != 0.f || t.z != 0.f || t.w != 0.f)
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a.colsum + c4 * 4), "f"(t.x), "f"(t.y),
                     "f"(t.z), "f"(t.w) : "memory");
    }
  }
}

}  // namespace

void launch_build_transpose(const TransposeArgs& a, cudaStream_t s) {
  cudaMemsetAsync(a.cnt, 0, sizeof(int32_t) * static_cast<size_t>(a.n_hops) * a.cap_nodes, s);
  cudaMemsetAsync(a.cursor, 0, sizeof(int32_t) * static_cast<size_t>(a.n_hops) * a.cap_nodes, s);
  for (int h = 0; h < a.n_hops; ++h)
    k_tr_count<<<grid_for(static_cast<int64_t>(a.cap_rows[h]) * a.k[h], 256 * 4), 256, 0, s>>>(a, h);
  const int per_block = kScanBlock * kScanItems;
  const int n_blocks = (a.cap_nodes + per_block - 1) / per_block;
  k_tr_scan1<<<n_blocks, kScanBlock, 0, s>>>(a);
  k_tr_scan2<<<1, 1024, 0, s>>>(a, n_blocks);
  k_tr_scan3<<<n_blocks, kScanBlock, 0, s>>>(a);
  for (int h = 0; h < a.n_hops; ++h)
    k_tr_fill<<<grid_for(static_cast<int64_t>(a.cap_rows[h]) * a.k[h], 256 * 4), 256, 0, s>>>(a, h);
  if (a.meta) k_tr_meta<<<grid_for(a.cap_nodes, 256, 132 * 4), 256, 0, s>>>(a);
}

void launch_sage_gather_bwd(const SageGatherBwdArgs& a, cudaStream_t s) {
  if (a.colsum && !a.colsum_prezeroed) cudaMemsetAsync(a.colsum, 0, sizeof(float) * a.d, s);
  dispatch_lanes<4, 4>(a.d / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    constexpr int TEAM = (LPR == 32) ? 4 : (LPR == 16 ? 2 : 1);
    launch_k(k_sage_gather_bwd<LPR, VPL>, dim3(grid_for(a.cap_src, 8 * 32 / TEAM, 132 * 8)), dim3(256),
             sizeof(float) * a.d * 8, s, a);
  });
}

}  // namespace glt
