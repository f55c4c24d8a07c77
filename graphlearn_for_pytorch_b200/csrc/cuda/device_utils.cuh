// Device-side helpers shared by the sm_90a kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <cstdint>

#include "../philox.h"
#include "glt_cuda.h"

namespace glt {

constexpr int64_t kEmptyKey = -1;

// Programmatic dependent launch (PDL).  The kernels of a training step form one long dependency chain of short
// launches; with the launch attribute set (launch_utils.h) the NEXT kernel's CTAs are scheduled as soon as every
// CTA of the current grid has called pdl_trigger(), and block in pdl_wait() until the current grid has completed
// and flushed its memory -- so launch latency, scheduling and any prologue placed before pdl_wait() overlap with
// the tail of the predecessor.  Without the attribute both instructions are no-ops.  Rule: nothing that a
// predecessor kernel may have written is read before pdl_wait().
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_enter() { pdl_wait(); pdl_trigger(); }

__device__ __forceinline__ uint32_t hash_slot(int64_t key, uint32_t mask) {
  uint64_t x = static_cast<uint64_t>(key) * 0x9E3779B97F4A7C15ULL;
  return static_cast<uint32_t>(x >> 29) & mask;
}

constexpr uint32_t kTableFull = 0xFFFFFFFFu;

// Insert `key`; returns the slot and whether this thread claimed it.  The probe sequence is bounded
// by the table size: a full table (a batch with far more unique nodes than the calibrated arena
// was sized for) yields kTableFull instead of spinning forever; callers drop that neighbour and
// count it as overflow.
__device__ __forceinline__ uint32_t table_insert(const HashTable& t, int64_t key, bool* is_new) {
  uint32_t s = hash_slot(key, t.mask);
  *is_new = false;
  for (uint32_t probes = 0; probes <= t.mask; ++probes) {
    unsigned long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(t.keys + s),
                                        static_cast<unsigned long long>(kEmptyKey),
                                        static_cast<unsigned long long>(key));
    if (prev == static_cast<unsigned long long>(kEmptyKey)) { *is_new = true; return s; }
    if (prev == static_cast<unsigned long long>(key)) return s;
    s = (s + 1) & t.mask;
  }
  return kTableFull;
}

__device__ __forceinline__ int32_t table_find_slot(const HashTable& t, int64_t key) {
  uint32_t s = hash_slot(key, t.mask);
  for (uint32_t probes = 0; probes <= t.mask; ++probes) {
    int64_t k = t.keys[s];
    if (k == key) return static_cast<int32_t>(s);
    if (k == kEmptyKey) return -1;
    s = (s + 1) & t.mask;
  }
  return -1;
}

struct RowRef {
  int64_t start;  // offset into the owning shard's indices
  int32_t deg;
  int32_t part;
};

// Owner lookup + row extent.  The shard may be peer HBM: these are plain
// ld.global on NVLink-mapped addresses, no RPC, no host staging.
__device__ __forceinline__ RowRef load_row(const GraphTable& g, int64_t v) {
  RowRef r;
  r.start = 0; r.deg = 0; r.part = -1;
#pragma unroll 1
  for (int p = 0; p < g.num_parts; ++p) {
    const int64_t b = g.parts[p].row_begin, e = g.parts[p].row_end;
    if (v >= b && v < e) {
      const int64_t* ip = g.parts[p].indptr + (v - b);
      const int64_t s0 = __ldg(ip), s1 = __ldg(ip + 1);
      r.start = s0; r.deg = static_cast<int32_t>(s1 - s0); r.part = p;
      break;
    }
  }
  return r;
}

__device__ __forceinline__ int64_t load_col(const GraphTable& g, int part, int64_t pos) {
  if (g.idx_bytes == 4) return __ldg(reinterpret_cast<const int32_t*>(g.parts[part].indices) + pos);
  return __ldg(reinterpret_cast<const int64_t*>(g.parts[part].indices) + pos);
}

// Is c in the (column-sorted) row already located by load_row?  Binary search.
__device__ __forceinline__ bool row_has_col(const GraphTable& g, const RowRef& row, int64_t c) {
  int64_t lo = 0, hi = row.deg;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int64_t x = load_col(g, row.part, row.start + mid);
    if (x == c) return true;
    if (x < c) lo = mid + 1; else hi = mid;
  }
  return false;
}

// Strict edge test: is c a neighbour of r?  Binary search of r's row (rows are column-sorted, Topology guarantees it).
__device__ __forceinline__ bool edge_exists(const GraphTable& g, int64_t r, int64_t c) {
  return row_has_col(g, load_row(g, r), c);
}

__device__ __forceinline__ unsigned lanemask_lt() {
  unsigned m;
  asm volatile("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// 16-byte streaming load that bypasses L1 allocation (feature rows are touched
// once per batch; peer rows are not L2-cached locally anyway).
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t ld_nc_u32(const void* p) {
  uint32_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
  return r;
}

// MXFP8 (OCP microscaling: e4m3 elements, one UE8M0 power-of-two scale per 32 elements; a scale byte b is 2^(b - 127)).
// acc[0..16) += the 16 consecutive elements in `v` times their block's scale s.
__device__ __forceinline__ void mxfp8x16_accum_scaled(const uint4& v, float s, float* acc) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const __half2_raw hr = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>((w[i] >> (16 * h)) & 0xFFFFu),
                                                        __NV_E4M3);
      const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&hr));
      acc[i * 4 + h * 2] += f2.x * s;
      acc[i * 4 + h * 2 + 1] += f2.y * s;
    }
  }
}

// d = 128 rows: `v` holds the elements starting at element gl * 16, `scales` the row's four block-scale bytes; the
// block of this lane's elements is gl >> 1.
__device__ __forceinline__ void mxfp8x16_accum(const uint4& v, uint32_t scales, int gl, float* acc) {
  mxfp8x16_accum_scaled(v, __uint_as_float(((scales >> (8 * (gl >> 1))) & 0xFFu) << 23), acc);
}

// Rows of any width d (a multiple of 32): `row` points at an MXFP8 row, c is the 16-element vector
// index (elements [16c, 16c + 16), block c >> 1).  The block's scale byte sits at row + d + (c >> 1) and is fetched
// once per vector.  mxfp8_scale_at and mxfp8x16_accum_scaled are the two halves, for callers that issue the loads
// of several rows before they accumulate.
__device__ __forceinline__ float mxfp8_scale_at(const uint8_t* row, int d, int c) {
  uint32_t b;
  asm volatile("ld.global.nc.L1::no_allocate.u8 %0, [%1];" : "=r"(b) : "l"(row + d + (c >> 1)));
  return __uint_as_float(b << 23);
}

__device__ __forceinline__ void mxfp8x16_accum_at(const uint8_t* row, int d, int c, float* acc) {
  mxfp8x16_accum_scaled(ld_nc_v4(row + c * 16), mxfp8_scale_at(row, d, c), acc);
}

__device__ __forceinline__ void bf16x8_accum(const uint4& v, float* acc) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 f = __bfloat1622float2(h[i]);
    acc[2 * i] += f.x;
    acc[2 * i + 1] += f.y;
  }
}

__device__ __forceinline__ uint4 pack_bf16x8(const float* a, float scale) {
  uint4 r;
  __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2bfloat162_rn(a[2 * i] * scale, a[2 * i + 1] * scale);
  return r;
}

// Row pointer of a RowTable by (already remapped) row index.
__device__ __forceinline__ const uint8_t* row_ptr(const RowTable& t, int64_t row) {
#pragma unroll 1
  for (int p = 0; p < t.num_parts; ++p) {
    if (row >= t.row_begin[p] && row < t.row_begin[p + 1])
      return reinterpret_cast<const uint8_t*>(t.base[p]) + (row - t.row_begin[p]) * t.row_bytes;
  }
  return nullptr;
}

// Target row t of a sampled batch -> (hop, row inside that hop's ELL block), from the cumulative per-hop counters
// cum[0..n_hops].
struct HopLoc { int hop; int row; };

__device__ __forceinline__ HopLoc locate_hop(const int32_t* cum, int n_hops, int t) {
  HopLoc l; l.hop = 0; l.row = t;
#pragma unroll 1
  for (int h = 0; h < n_hops; ++h) {
    const int b = cum[h], e = cum[h + 1];
    if (t >= b && t < e) { l.hop = h; l.row = t - b; break; }
  }
  return l;
}

// Source row s of a GraphSAGE aggregation: the dense bf16 activation of the previous layer, or the feature table row of
// batch node s (layer 1).
__device__ __forceinline__ const uint8_t* src_row(const SageAggArgs& a, int s) {
  if (a.src_local) return reinterpret_cast<const uint8_t*>(a.src_local) + static_cast<int64_t>(s) * a.d * 2;
  return row_ptr(a.feat, a.nodes[s]);
}

// dst[0..8) += v[0..8) as two 16-byte vector atomics (red.global.add.v4.f32; dst 16-byte aligned).
__device__ __forceinline__ void red_add8(float* dst, const float* v) {
  atomicAdd(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3]));
  atomicAdd(reinterpret_cast<float4*>(dst + 4), make_float4(v[4], v[5], v[6], v[7]));
}

__device__ __forceinline__ float leaky(float x, float slope) { return x > 0.f ? x : x * slope; }

// Random bits of 16-byte vector i (8 bf16 elements) of a dropout mask: a pure function of (seed, layer, optimizer
// step, i), so a replayed step draws the same mask and a backward can regenerate it.  Element q is kept when 16-bit
// half (q & 1) of word q >> 1 is >= the caller's threshold.
__device__ __forceinline__ U4 dropout_bits(uint64_t seed, int layer, uint32_t step, int64_t i) {
  U4 c;
  c.x = static_cast<uint32_t>(i);
  c.y = static_cast<uint32_t>(i >> 32);
  c.z = step;
  c.w = 0xD509u + static_cast<uint32_t>(layer);
  return philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), c);
}

}  // namespace glt
