// Exact layer-wise GraphSAGE inference: the neighbour mean over a node's FULL CSR row (the `fanout >= degree` limit of
// the sampler, which takes every neighbour of a row with d <= k), for a chunk [r0, r1) of global node ids.
//
// Rows are reduced in a fixed order with fp32 accumulators and rounded once (the row schedule of full_rows.cuh: hub rows
// are split over the CTA and their partial sums added in group order), so the result is bitwise identical from call to
// call and for any chunking.
#include "full_rows.cuh"

namespace glt {

namespace {

// Source row of global node u: the dense bf16 table at column src_col, or the feature table (layer 1).
__device__ __forceinline__ const uint8_t* full_src_row(const SageFullAggArgs& a, int64_t u) {
  if (a.src) {
    if (u < 0 || u >= a.n_src) return nullptr;
    return reinterpret_cast<const uint8_t*>(a.src) + (u * a.src_ld + a.src_col) * 2;
  }
  return row_ptr(a.feat, u);
}

// LPR lanes per row; each lane owns VPL vectors of EPV elements (8 bf16 or 16 e4m3 = 16 bytes).
template <int LPR, int VPL, bool FP8>
struct FullAgg {
  static constexpr int EPV = FP8 ? 16 : 8;
  static constexpr int R = LPR < 8 ? LPR : 8;   // LPR and R are powers of two: jj + u < LPR

  // acc += x_u for neighbours j = first, first + stride, ... < deg of the row (part, start), in increasing j order.
  __device__ static void accumulate(const SageFullAggArgs& a, int part, int64_t start, int deg, int first, int stride,
                                    int gl, unsigned gmask, float (&acc)[VPL][EPV]) {
    const int n = first < deg ? (deg - first + stride - 1) / stride : 0;
    const int nvec = a.d / EPV;
    for (int i0 = 0; i0 < n; i0 += LPR) {
      const uint8_t* mine = nullptr;
      if (i0 + gl < n)
        mine = full_src_row(a, load_col(a.g, part, start + first + static_cast<int64_t>(i0 + gl) * stride));
      const int cnt = min(LPR, n - i0);
      // R rows in flight per lane group, accumulated in neighbour order
      for (int jj = 0; jj < cnt; jj += R) {
        const uint8_t* p[R];
        uint4 raw[R][VPL];
        float sc[R][VPL];   // FP8: the block scale of each vector
#pragma unroll
        for (int u = 0; u < R; ++u) {
          p[u] = reinterpret_cast<const uint8_t*>(
              __shfl_sync(gmask, reinterpret_cast<unsigned long long>(mine), jj + u, LPR));
          if (jj + u >= cnt) p[u] = nullptr;
#pragma unroll
          for (int v = 0; v < VPL; ++v) { raw[u][v] = make_uint4(0, 0, 0, 0); sc[u][v] = 0.f; }
        }
#pragma unroll
        for (int u = 0; u < R; ++u) {
          if (p[u] == nullptr) continue;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int c = v * LPR + gl;
            if (c >= nvec) continue;
            raw[u][v] = ld_nc_v4(p[u] + c * 16);
            if (FP8) sc[u][v] = mxfp8_scale_at(p[u], a.d, c);   // MXFP8 rows: d e4m3 bytes, then d/32 UE8M0 scales
          }
        }
#pragma unroll
        for (int u = 0; u < R; ++u) {
          if (p[u] == nullptr) continue;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            if (FP8) mxfp8x16_accum_scaled(raw[u][v], sc[u][v], acc[v]);
            else bf16x8_accum(raw[u][v], acc[v]);
          }
        }
      }
    }
  }

  // concat: out = bf16([mean | self]) (mean only: bf16(mean));  combine: out = act(mean + src[r, self_col:] + b)
  __device__ static void epilogue(const SageFullAggArgs& a, int64_t r, int deg, int gl, const float (&acc)[VPL][EPV]) {
    const float inv = deg > 0 ? 1.f / static_cast<float>(deg) : 0.f;
    uint8_t* o = reinterpret_cast<uint8_t*>(a.out) + (r - a.r0) * a.out_ld * 2;
    if (FP8) {
      const uint8_t* sp = a.mean_only ? nullptr : row_ptr(a.feat, r);
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c >= a.d / EPV) continue;
        reinterpret_cast<uint4*>(o)[c * 2] = pack_bf16x8(acc[v], inv);
        reinterpret_cast<uint4*>(o)[c * 2 + 1] = pack_bf16x8(acc[v] + 8, inv);
        if (a.mean_only) continue;
        float self[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) self[i] = 0.f;
        if (sp) mxfp8x16_accum_at(sp, a.d, c, self);
        reinterpret_cast<uint4*>(o + a.d * 2)[c * 2] = pack_bf16x8(self, 1.f);
        reinterpret_cast<uint4*>(o + a.d * 2)[c * 2 + 1] = pack_bf16x8(self + 8, 1.f);
      }
      return;
    }
    const int nvec = a.d >> 3;
    const uint8_t* sp;
    if (a.mean_only)
      sp = nullptr;
    else if (a.src)
      sp = reinterpret_cast<const uint8_t*>(a.src) + (r * a.src_ld + a.self_col) * 2;
    else
      sp = row_ptr(a.feat, r);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      const uint4 sv = sp ? ld_nc_v4(sp + c * 16) : make_uint4(0, 0, 0, 0);
      if (!a.combine) {
        reinterpret_cast<uint4*>(o)[c] = pack_bf16x8(acc[v], inv);
        if (!a.mean_only) reinterpret_cast<uint4*>(o + a.d * 2)[c] = sv;
      } else {
        float z[8], b[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) z[i] = b[i] = 0.f;
        bf16x8_accum(sv, z);
        if (a.bias) bf16x8_accum(reinterpret_cast<const uint4*>(a.bias)[c], b);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          z[i] += acc[v][i] * inv + b[i];
          if (a.relu) z[i] = fmaxf(z[i], 0.f);
        }
        reinterpret_cast<uint4*>(o)[c] = pack_bf16x8(z, 1.f);
      }
    }
  }
};

// One row per lane group (G = 256 / LPR rows per CTA); hub rows are reduced by the whole CTA.
template <int LPR, int VPL, bool FP8>
__global__ void __launch_bounds__(kFullRowThreads) k_sage_full_aggregate(SageFullAggArgs a) {
  using K = FullAgg<LPR, VPL, FP8>;
  constexpr int G = kFullRowThreads / LPR;
  extern __shared__ float s_part[];    // [G][d] partial sums of a hub row
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int g = threadIdx.x / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << ((lane / LPR) * LPR));
  float acc[VPL][K::EPV];
  auto zero = [&]() {
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int i = 0; i < K::EPV; ++i) acc[v][i] = 0.f;
  };
  RowRef rr;
  zero();
  full_rows<G>(
      a.r0, a.r1, g, gl, [&](int64_t r) { rr = load_row(a.g, r); return rr.deg; },
      [&](int64_t r) {
        if (rr.deg > 0) K::accumulate(a, rr.part, rr.start, rr.deg, 0, 1, gl, gmask, acc);
        K::epilogue(a, r, rr.deg, gl, acc);
      },
      [&](int64_t hr) {
        const RowRef hb = load_row(a.g, hr);
        zero();
        K::accumulate(a, hb.part, hb.start, hb.deg, g, G, gl, gmask, acc);
        put_partials<LPR>(s_part, a.d, g, gl, acc);
        __syncthreads();
        if (g == 0) {
          sum_partials<G, LPR>(s_part, a.d, gl, acc);
          K::epilogue(a, hr, hb.deg, gl, acc);
        }
      });
}

template <int LPR, int VPL, bool FP8>
void launch_full(const SageFullAggArgs& a, cudaStream_t s) {
  launch_full_rows<LPR>(k_sage_full_aggregate<LPR, VPL, FP8>, a, a.d, s);
}

}  // namespace

void launch_sage_full_aggregate(const SageFullAggArgs& a, cudaStream_t s) {
  if (a.feat_fp8) {   // d / 16 vectors of 16 e4m3 elements; d = 128 is <8, 1, true>
    dispatch_lanes<2, 2>(a.d / 16, [&](auto lpr, auto vpl) {
      launch_full<decltype(lpr)::value, decltype(vpl)::value, true>(a, s);
    });
    return;
  }
  dispatch_lanes<4, 4>(a.d / 8, [&](auto lpr, auto vpl) {
    launch_full<decltype(lpr)::value, decltype(vpl)::value, false>(a, s);
  });
}

}  // namespace glt
