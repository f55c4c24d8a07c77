// Multi-source row gather (UnifiedTensor / Feature lookup).
//
// out[i,:] = part(owner(idx[i]))[idx[i] - begin(owner)], where a part is local
// HBM, a peer GPU's HBM mapped over NVLink (CUDA IPC) or pinned host memory.
// Capability parity with the reference's GatherTensorKernel
// (csrc/cuda/unified_tensor.cu:47-81: warp per row, scalar T loads); here rows
// move as 16-byte vectors with L1::no_allocate, several rows share a warp when
// rows are narrow, every lane keeps up to four loads in flight, and the row
// count can stay on the device (n_dev) so the launch is CUDA-graph capturable.
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// LPR lanes cooperate on one row; every group keeps R independent rows in flight: the id ->
// (id2index) -> owner-shard pointer chase and the 16-byte row loads of R rows are issued back to
// back before anything is stored.  Rows in peer HBM cost ~2 us per dependent step over NVLink, so
// the kernel is a latency x parallelism product: R = 4 quadruples the bytes in flight per SM for
// the common 256/512-byte rows.
template <int LPR, int R>
__global__ void __launch_bounds__(256) k_gather_vec(RowTable t, const int64_t* idx,
                                                    const int64_t* id2index, int64_t n,
                                                    const int32_t* n_dev, uint8_t* out,
                                                    int64_t out_row_bytes, int64_t map_len) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int64_t n_valid = n_dev ? min(static_cast<int64_t>(*n_dev), n) : n;
  const int nvec = static_cast<int>(t.row_bytes >> 4);
  const int64_t wpb = blockDim.x >> 5;
  for (int64_t base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * (RPW * R); base < n;
       base += static_cast<int64_t>(gridDim.x) * wpb * (RPW * R)) {
    int64_t row[R];
#pragma unroll
    for (int k = 0; k < R; ++k) {
      const int64_t r = base + k * RPW + gw;
      row[k] = (r < n_valid) ? idx[r] : -1;
    }
    if (id2index) {
#pragma unroll
      for (int k = 0; k < R; ++k)
        if (row[k] >= 0) row[k] = (map_len <= 0 || row[k] < map_len) ? id2index[row[k]] : -1;
    }
    const uint4* src[R];
#pragma unroll
    for (int k = 0; k < R; ++k)
      src[k] = row[k] >= 0 ? reinterpret_cast<const uint4*>(row_ptr(t, row[k])) : nullptr;
    for (int c = gl; c < nvec; c += LPR) {
      uint4 v[R];
#pragma unroll
      for (int k = 0; k < R; ++k) v[k] = src[k] ? ld_nc_v4(src[k] + c) : make_uint4(0, 0, 0, 0);
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int64_t r = base + k * RPW + gw;
        if (r < n) reinterpret_cast<uint4*>(out + r * out_row_bytes)[c] = v[k];
      }
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256) k_gather_scalar(RowTable t, const int64_t* idx,
                                                       const int64_t* id2index, int64_t n,
                                                       const int32_t* n_dev, uint8_t* out,
                                                       int64_t out_row_bytes, int64_t map_len) {
  const int lane = threadIdx.x & 31;
  const int64_t n_valid = n_dev ? min(static_cast<int64_t>(*n_dev), n) : n;
  const int nel = static_cast<int>(t.row_bytes / sizeof(T));
  const int64_t wpb = blockDim.x >> 5;
  for (int64_t r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n;
       r += static_cast<int64_t>(gridDim.x) * wpb) {
    const uint8_t* src = nullptr;
    if (r < n_valid) {
      int64_t row = idx[r];
      if (row >= 0 && id2index) row = (map_len <= 0 || row < map_len) ? id2index[row] : -1;
      if (row >= 0) src = row_ptr(t, row);
    }
    T* dst = reinterpret_cast<T*>(out + r * out_row_bytes);
    const T* s = reinterpret_cast<const T*>(src);
    for (int c = lane; c < nel; c += 32) dst[c] = src ? s[c] : T(0);
  }
}

// 8 lanes per row, 16 e4m3 elements per lane and iteration (d multiple of 128 keeps every lane busy)
__global__ void __launch_bounds__(256) k_gather_mxfp8(RowTable t, const int64_t* idx, int64_t n, int d,
                                                      __nv_bfloat16* out) {
  const int lane = threadIdx.x & 31;
  const int gl = lane & 7, gw = lane >> 3;
  const int64_t wpb = blockDim.x >> 5;
  for (int64_t base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * 4; base < n;
       base += static_cast<int64_t>(gridDim.x) * wpb * 4) {
    const int64_t r = base + gw;
    if (r >= n) continue;
    const int64_t row = idx[r];
    const uint8_t* p = row >= 0 ? row_ptr(t, row) : nullptr;
    for (int e0 = gl * 16; e0 < d; e0 += 128) {
      float x[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) x[i] = 0.f;
      if (p) {
        // scale bytes of this 128-element span: 4 consecutive bytes at d + e0 / 32 (e0 / 32 is a multiple of 4
        // for the span start; the lane picks its block inside mxfp8x16_accum from gl)
        const uint32_t sc = ld_nc_u32(p + d + ((e0 - gl * 16) >> 5));
        mxfp8x16_accum(ld_nc_v4(p + e0), sc, gl, x);
      }
      __nv_bfloat16* o = out + r * d + e0;
      *reinterpret_cast<uint4*>(o) = pack_bf16x8(x, 1.f);
      *reinterpret_cast<uint4*>(o + 8) = pack_bf16x8(x + 8, 1.f);
    }
  }
}

// k_gather_vec for MXFP8 rows of d elements (d / 16 vectors of 16 e4m3 elements): the same id -> (id2index) -> shard
// pointer chase with R rows in flight per lane group, but every 16-byte load comes with its block's scale byte and
// is stored as two 16-byte vectors of bf16.  Rows past the device count and negative ids are written as zeros.
template <int LPR, int R>
__global__ void __launch_bounds__(256) k_gather_mxfp8_vec(RowTable t, const int64_t* idx, const int64_t* id2index,
                                                          int64_t n, const int32_t* n_dev, int d, uint8_t* out,
                                                          int64_t out_row_bytes, int64_t map_len) {
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int64_t n_valid = n_dev ? min(static_cast<int64_t>(*n_dev), n) : n;
  const int nvec = d >> 4;
  const int64_t wpb = blockDim.x >> 5;
  for (int64_t base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * (RPW * R); base < n;
       base += static_cast<int64_t>(gridDim.x) * wpb * (RPW * R)) {
    int64_t row[R];
#pragma unroll
    for (int k = 0; k < R; ++k) {
      const int64_t r = base + k * RPW + gw;
      row[k] = (r < n_valid) ? idx[r] : -1;
    }
    if (id2index) {
#pragma unroll
      for (int k = 0; k < R; ++k)
        if (row[k] >= 0) row[k] = (map_len <= 0 || row[k] < map_len) ? id2index[row[k]] : -1;
    }
    const uint8_t* src[R];
#pragma unroll
    for (int k = 0; k < R; ++k) src[k] = row[k] >= 0 ? row_ptr(t, row[k]) : nullptr;
    for (int c = gl; c < nvec; c += LPR) {
      uint4 v[R];
      float sc[R];
#pragma unroll
      for (int k = 0; k < R; ++k) {
        v[k] = src[k] ? ld_nc_v4(src[k] + c * 16) : make_uint4(0, 0, 0, 0);
        sc[k] = src[k] ? mxfp8_scale_at(src[k], d, c) : 0.f;
      }
#pragma unroll
      for (int k = 0; k < R; ++k) {
        const int64_t r = base + k * RPW + gw;
        if (r >= n) continue;
        float x[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) x[i] = 0.f;
        mxfp8x16_accum_scaled(v[k], sc[k], x);
        uint4* o = reinterpret_cast<uint4*>(out + r * out_row_bytes) + 2 * c;
        o[0] = pack_bf16x8(x, 1.f);
        o[1] = pack_bf16x8(x + 8, 1.f);
      }
    }
  }
}

}  // namespace

void launch_gather_rows(RowTable t, const int64_t* idx, const int64_t* id2index, int64_t n,
                        const int32_t* n_dev, void* out, int64_t out_row_bytes, cudaStream_t s,
                        int64_t id2index_len) {
  if (n <= 0) return;
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  bool aligned = (t.row_bytes % 16 == 0) && (out_row_bytes % 16 == 0) &&
                 (reinterpret_cast<uintptr_t>(out) % 16 == 0);
  for (int p = 0; p < t.num_parts; ++p) aligned &= (reinterpret_cast<uintptr_t>(t.base[p]) % 16 == 0);
  if (aligned) {
    // small lookups spread one row per group over as many SMs as possible; large ones keep four rows
    // in flight per group
    dispatch_lanes<1, 1>(static_cast<int>(t.row_bytes / 16), [&](auto lpr, auto) {
      constexpr int LPR = decltype(lpr)::value;
      if (n >= static_cast<int64_t>(132) * 2 * 8 * (32 / LPR) * 4)
        k_gather_vec<LPR, 4><<<grid_for(n, 8 * (32 / LPR) * 4), 256, 0, s>>>(t, idx, id2index, n, n_dev, o,
                                                                              out_row_bytes, id2index_len);
      else
        k_gather_vec<LPR, 1><<<grid_for(n, 8 * (32 / LPR)), 256, 0, s>>>(t, idx, id2index, n, n_dev, o,
                                                                          out_row_bytes, id2index_len);
    });
    return;
  }
  const int g = grid_for(n, 8);
  if (t.row_bytes % 4 == 0 && out_row_bytes % 4 == 0)
    k_gather_scalar<uint32_t><<<g, 256, 0, s>>>(t, idx, id2index, n, n_dev, o, out_row_bytes, id2index_len);
  else if (t.row_bytes % 2 == 0 && out_row_bytes % 2 == 0)
    k_gather_scalar<uint16_t><<<g, 256, 0, s>>>(t, idx, id2index, n, n_dev, o, out_row_bytes, id2index_len);
  else
    k_gather_scalar<uint8_t><<<g, 256, 0, s>>>(t, idx, id2index, n, n_dev, o, out_row_bytes, id2index_len);
}

// NVSwitch multicast store: one write lands in the replica of every GPU bound to the
// multicast object (hot-cache fill).  `mc_dst` is a multicast virtual address.
__global__ void k_multimem_copy(const uint4* __restrict__ src, uint4* mc_dst, int64_t n16) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n16;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const uint4 v = src[i];
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(mc_dst + i),
                 "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                 "f"(__uint_as_float(v.w))
                 : "memory");
  }
}

void launch_multimem_copy(const void* src, void* mc_dst, int64_t nbytes, cudaStream_t s) {
  const int64_t n16 = nbytes / 16;
  if (n16 <= 0) return;
  int64_t blocks = (n16 + 255) / 256;
  if (blocks > 132 * 8) blocks = 132 * 8;
  k_multimem_copy<<<static_cast<int>(blocks), 256, 0, s>>>(reinterpret_cast<const uint4*>(src),
                                                           reinterpret_cast<uint4*>(mc_dst), n16);
}

void launch_gather_mxfp8(RowTable t, const int64_t* idx, int64_t n, int d, void* out, cudaStream_t s) {
  if (n <= 0) return;
  int64_t blocks = (n + 31) / 32;
  if (blocks > 132 * 16) blocks = 132 * 16;
  k_gather_mxfp8<<<static_cast<int>(blocks), 256, 0, s>>>(t, idx, n, d, reinterpret_cast<__nv_bfloat16*>(out));
}

void launch_gather_mxfp8_rows(RowTable t, const int64_t* idx, const int64_t* id2index, int64_t n, const int32_t* n_dev,
                              int d, void* out, int64_t out_row_bytes, cudaStream_t s, int64_t id2index_len) {
  if (n <= 0) return;
  uint8_t* o = reinterpret_cast<uint8_t*>(out);
  // launch shapes as in launch_gather_rows: small lookups one row per group, large ones four rows in flight
  dispatch_lanes<2, 1>(d / 16, [&](auto lpr, auto) {
    constexpr int LPR = decltype(lpr)::value;
    if (n >= static_cast<int64_t>(132) * 2 * 8 * (32 / LPR) * 4)
      k_gather_mxfp8_vec<LPR, 4><<<grid_for(n, 8 * (32 / LPR) * 4), 256, 0, s>>>(t, idx, id2index, n, n_dev, d, o,
                                                                                  out_row_bytes, id2index_len);
    else
      k_gather_mxfp8_vec<LPR, 1><<<grid_for(n, 8 * (32 / LPR)), 256, 0, s>>>(t, idx, id2index, n, n_dev, d, o,
                                                                              out_row_bytes, id2index_len);
  });
}

}  // namespace glt
