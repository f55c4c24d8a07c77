// Full-neighbourhood attention of the heterogeneous engines' layer-wise inference (HeteroGatEngine.inference,
// HeteroHgtEngine.inference): the softmax of a target spans its COMPLETE CSR rows (the `fanout >= degree` limit of the
// sampled kernels in gat.cu / hgt.cu), for a chunk [r0, r1) of global target ids.
//
// Lane-group layout of the sampled siblings: LPR lanes per row, a lane owns VPL 16-byte vectors (columns c * 8 ..
// c * 8 + 7, c = v * LPR + lane) of an H-wide row.  Rows follow the schedule of full_rows.cuh (hub rows split over the
// CTA, partials merged in group order), so every row has one fixed reduction order: results are bitwise identical from
// call to call and for any chunking.  No exp is ever taken of a score that is not shifted by the maximum it is
// normalised against.
#include <cmath>

#include "full_rows.cuh"

namespace glt {

namespace {

// ------------------------------------------------------------------------------------------------------ R-GAT
// Scores are per node (as, ad), so both passes over a row read scalars; only pass 2 reads the projection rows.
//   pass 1  m = max_j e_ij,h                       (order-free: a max is exact)
//   pass 2  s = sum_j exp(e_ij,h - m),  acc = sum_j exp(e_ij,h - m) P[j]      then out = acc / s
// Each lane keeps the statistics of the head of each of its vectors (lanes sharing a head compute identical values).
template <int LPR, int VPL>
struct GatFull {
  __device__ __forceinline__ static void adh(const GatFullAggArgs& a, int64_t r, int gl, float (&ad)[VPL]) {
    const int nvec = a.H >> 3, cv = nvec / a.heads;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      ad[v] = c < nvec ? a.ad[r * a.heads + c / cv] : 0.f;
    }
  }

  __device__ __forceinline__ static void max_pass(const GatFullAggArgs& a, const RowRef& rr, int first, int stride, int gl,
                                  const float (&ad)[VPL], float (&m)[VPL]) {
    const int nvec = a.H >> 3, cv = nvec / a.heads;
    for (int j = first; j < rr.deg; j += stride) {
      const int64_t u = load_col(a.g, rr.part, rr.start + j);
      if (u < 0 || u >= a.n_src) continue;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec) m[v] = fmaxf(m[v], leaky(a.as[u * a.heads + c / cv] + ad[v], 0.2f));
      }
    }
  }

  __device__ __forceinline__ static void sum_pass(const GatFullAggArgs& a, const RowRef& rr, int first, int stride, int gl,
                                  const float (&ad)[VPL], const float (&m)[VPL], float (&s)[VPL],
                                  float (&acc)[VPL][8]) {
    const int nvec = a.H >> 3, cv = nvec / a.heads;
    for (int j = first; j < rr.deg; j += stride) {
      const int64_t u = load_col(a.g, rr.part, rr.start + j);
      if (u < 0 || u >= a.n_src) continue;
      const uint8_t* p = reinterpret_cast<const uint8_t*>(a.P) + u * a.H * 2;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec) {
          const float w = expf(leaky(a.as[u * a.heads + c / cv] + ad[v], 0.2f) - m[v]);
          s[v] += w;
          float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          bf16x8_accum(ld_nc_v4(p + c * 16), x);
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[v][q] = fmaf(w, x[q], acc[v][q]);
        }
      }
    }
  }

  // out = acc / s, then the relation sum / bias / activation of the sampled kernel's epilogue
  __device__ __forceinline__ static void epilogue(const GatFullAggArgs& a, int64_t r, int gl, const float (&s)[VPL],
                                  const float (&acc)[VPL][8]) {
    const int nvec = a.H >> 3;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      const float inv = s[v] > 0.f ? __fdividef(1.f, s[v]) : 0.f;
      const int64_t e = (r - a.r0) * a.H + c * 8;
      float o[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) o[q] = acc[v][q] * inv;
      if (!a.first) {
        const float4 p0 = reinterpret_cast<const float4*>(a.acc + e)[0], p1 = reinterpret_cast<const float4*>(a.acc + e)[1];
        const float prev[8] = {p0.x, p0.y, p0.z, p0.w, p1.x, p1.y, p1.z, p1.w};
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = prev[q] + o[q];
      }
      if (!a.last) {
        reinterpret_cast<float4*>(a.acc + e)[0] = make_float4(o[0], o[1], o[2], o[3]);
        reinterpret_cast<float4*>(a.acc + e)[1] = make_float4(o[4], o[5], o[6], o[7]);
        continue;
      }
      for (int b = 0; b < a.n_bias; ++b)
        bf16x8_accum(reinterpret_cast<const uint4*>(a.bias)[(b * a.H + c * 8) >> 3], o);
      if (a.act) {
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = leaky(o[q], 0.01f);
      }
      reinterpret_cast<uint4*>(a.z)[e >> 3] = pack_bf16x8(o, 1.f);
    }
  }
};

// One row per lane group (G = 256 / LPR rows per CTA); hub rows are reduced by the whole CTA.
// Shared memory: [G][H] partial sums and [G][nvec] partial statistics of a hub row.
template <int LPR, int VPL>
__global__ void __launch_bounds__(kFullRowThreads, 2) k_gat_full_aggregate(GatFullAggArgs a) {
  using K = GatFull<LPR, VPL>;
  constexpr int G = kFullRowThreads / LPR;
  extern __shared__ float smem[];
  float* s_part = smem;                         // [G][H]
  float* s_stat = smem + G * a.H;               // [G][nvec]
  pdl_enter();
  const int gl = (threadIdx.x & 31) % LPR;
  const int g = threadIdx.x / LPR;
  const int nvec = a.H >> 3;
  float ad[VPL], m[VPL], s[VPL], acc[VPL][8];
  auto reset = [&]() {
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      m[v] = -INFINITY; s[v] = 0.f;
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[v][q] = 0.f;
    }
  };
  RowRef rr;
  full_rows<G>(
      a.r0, a.r1, g, gl, [&](int64_t r) { rr = load_row(a.g, r); return rr.deg; },
      [&](int64_t r) {
        reset();
        K::adh(a, r, gl, ad);
        K::max_pass(a, rr, 0, 1, gl, ad, m);
        K::sum_pass(a, rr, 0, 1, gl, ad, m, s, acc);
        K::epilogue(a, r, gl, s, acc);
      },
      [&](int64_t hr) {
        const RowRef hb = load_row(a.g, hr);
        reset();
        K::adh(a, hr, gl, ad);
        K::max_pass(a, hb, g, G, gl, ad, m);
        put_partials<LPR>(s_stat, nvec, g, gl, m);
        __syncthreads();
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec)
#pragma unroll 1
            for (int q = 0; q < G; ++q) m[v] = fmaxf(m[v], s_stat[q * nvec + c]);
        }
        __syncthreads();
        K::sum_pass(a, hb, g, G, gl, ad, m, s, acc);
        put_partials<LPR>(s_stat, nvec, g, gl, s);
        put_partials<LPR>(s_part, a.H, g, gl, acc);
        __syncthreads();
        if (g == 0) {
          sum_partials<G, LPR>(s_stat, nvec, gl, s);
          sum_partials<G, LPR>(s_part, a.H, gl, acc);
          K::epilogue(a, hr, gl, s, acc);
        }
      });
}

// ------------------------------------------------------------------------------------------------------ HGT
// Per target row, over the rows of all its relations (heads gl, gl + LPR, ... are owned by lane gl; a head's dot
// product goes through the group's shared-memory row `part`, as in k_hgt_attention):
//   pass 1 (reads K)      online softmax statistics per head: running max m and sum s of exp(score - m), rescaled by
//                         exp(m_old - m_new) <= 1 whenever the max grows
//   pass 2 (reads K, V)   per relation: alpha = exp(score - m) / s, u_r = sum_j alpha v_j; the alphas of one slot reach
//                         the lanes of its columns through the group's `al` row
template <int LPR, int VPL>
struct HgtFull {
  struct Ctx {
    float* part;                // [LPR * VPL] per-vector partial dots of this group
    float* al;                  // [heads] alphas of the current slot
    int gl;
    unsigned gmask;
  };

  __device__ __forceinline__ static void load_q(const HgtFullAttnArgs& a, int64_t row, int r, int gl, float (&qv)[VPL][8]) {
    const int nvec = a.H >> 3;
    const uint4* q = reinterpret_cast<const uint4*>(a.qq) + (((row - a.r0) * a.n_rel + r) * a.H >> 3);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
#pragma unroll
      for (int e = 0; e < 8; ++e) qv[v][e] = 0.f;
      const int c = v * LPR + gl;
      if (c < nvec) bf16x8_accum(q[c], qv[v]);
    }
  }

  // part[c] = <qv_c, K_u c-vector>; returns the K row (nullptr: skipped id)
  __device__ __forceinline__ static const uint8_t* dots(const HgtFullAttnArgs& a, int r, int64_t u, const Ctx& x,
                                        const float (&qv)[VPL][8]) {
    const int nvec = a.H >> 3;
    if (u < 0 || u >= a.n_src[r]) return nullptr;
    const uint8_t* p = reinterpret_cast<const uint8_t*>(a.kv[r]) + u * a.kv_ld * 2;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + x.gl;
      if (c < nvec) {
        float k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        bf16x8_accum(ld_nc_v4(p + c * 16), k);
        float d = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) d = fmaf(qv[v][e], k[e], d);
        x.part[c] = d;
      }
    }
    return p;
  }

  __device__ __forceinline__ static float head_score(const HgtFullAttnArgs& a, int h, const Ctx& x, float ps) {
    const int cv = (a.H >> 3) / a.heads;
    float d = 0.f;
    for (int c = h * cv; c < (h + 1) * cv; ++c) d += x.part[c];
    return d * ps;
  }

  __device__ __forceinline__ static void stats_pass(const HgtFullAttnArgs& a, int64_t row, int first, int stride, const Ctx& x,
                                    float (&m)[VPL], float (&s)[VPL]) {
    float qv[VPL][8];
#pragma unroll 1
    for (int r = 0; r < a.n_rel; ++r) {
      const RowRef rr = load_row(a.g[r], row);
      load_q(a, row, r, x.gl, qv);
      float ps[VPL];
#pragma unroll
      for (int q = 0; q < VPL; ++q) {
        const int h = x.gl + q * LPR;
        ps[q] = h < a.heads ? a.prior[r][h] * a.scale : 0.f;
      }
      for (int j = first; j < rr.deg; j += stride) {
        const int64_t u = load_col(a.g[r], rr.part, rr.start + j);
        const bool ok = dots(a, r, u, x, qv) != nullptr;
        __syncwarp(x.gmask);
        if (ok) {
#pragma unroll
          for (int q = 0; q < VPL; ++q) {
            const int h = x.gl + q * LPR;
            if (h < a.heads) {
              const float sc = head_score(a, h, x, ps[q]);
              if (sc > m[q]) { s[q] = s[q] * expf(m[q] - sc) + 1.f; m[q] = sc; }
              else s[q] += expf(sc - m[q]);
            }
          }
        }
        __syncwarp(x.gmask);
      }
    }
  }

  // acc = sum over relation r's slots j = first, first + stride, ... of alpha v_j (inv = 1 / s)
  __device__ __forceinline__ static void value_pass(const HgtFullAttnArgs& a, int r, int64_t row, int first, int stride, const Ctx& x,
                                    const float (&m)[VPL], const float (&inv)[VPL], float (&acc)[VPL][8]) {
    const int nvec = a.H >> 3, cv = nvec / a.heads;
    float qv[VPL][8];
    load_q(a, row, r, x.gl, qv);
    float ps[VPL];
#pragma unroll
    for (int q = 0; q < VPL; ++q) {
      const int h = x.gl + q * LPR;
      ps[q] = h < a.heads ? a.prior[r][h] * a.scale : 0.f;
    }
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[v][e] = 0.f;
    const RowRef rr = load_row(a.g[r], row);
    for (int j = first; j < rr.deg; j += stride) {
      const int64_t u = load_col(a.g[r], rr.part, rr.start + j);
      const uint8_t* p = dots(a, r, u, x, qv);
      __syncwarp(x.gmask);
      if (p != nullptr) {
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
          const int h = x.gl + q * LPR;
          if (h < a.heads) x.al[h] = expf(head_score(a, h, x, ps[q]) - m[q]) * inv[q];
        }
      }
      __syncwarp(x.gmask);
      if (p != nullptr) {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + x.gl;
          if (c < nvec) {
            const float w = x.al[c / cv];
            float val[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            bf16x8_accum(ld_nc_v4(p + (a.v_off + c * 8) * 2), val);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[v][e] = fmaf(w, val[e], acc[v][e]);
          }
        }
      }
      __syncwarp(x.gmask);
    }
  }

  __device__ __forceinline__ static void store_u(const HgtFullAttnArgs& a, int r, int64_t row, int gl, const float (&acc)[VPL][8]) {
    const int nvec = a.H >> 3;
    uint4* o = reinterpret_cast<uint4*>(a.u) + (((row - a.r0) * a.n_rel + r) * a.H >> 3);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c < nvec) o[c] = pack_bf16x8(acc[v], 1.f);
    }
  }
};

// Shared memory: per group a dot row [LPR * VPL] and an alpha row [heads]; for hub rows [G][2 heads] statistics and
// [G][H] partial sums.
template <int LPR, int VPL>
__global__ void __launch_bounds__(kFullRowThreads, 2) k_hgt_full_attention(HgtFullAttnArgs a) {
  using K = HgtFull<LPR, VPL>;
  constexpr int G = kFullRowThreads / LPR;
  extern __shared__ float smem[];
  const int heads = a.heads;
  float* s_dot = smem;                                  // [G][LPR * VPL]
  float* s_al = s_dot + G * LPR * VPL;                  // [G][heads]
  float* s_stat = s_al + G * heads;                     // [G][2 heads]
  float* s_part = s_stat + G * 2 * heads;               // [G][H]
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int g = threadIdx.x / LPR;
  typename K::Ctx x;
  x.part = s_dot + g * LPR * VPL;
  x.al = s_al + g * heads;
  x.gl = gl;
  x.gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << ((lane / LPR) * LPR));
  float m[VPL], s[VPL], inv[VPL], acc[VPL][8];
#pragma unroll
  for (int q = 0; q < VPL; ++q) { m[q] = -INFINITY; s[q] = 0.f; }
  full_rows<G>(
      a.r0, a.r1, g, gl,
      [&](int64_t row) {   // the row's neighbours over all its relations
        int total = 0;
#pragma unroll 1
        for (int r = 0; r < a.n_rel; ++r) total += load_row(a.g[r], row).deg;
        return total;
      },
      [&](int64_t row) {
        K::stats_pass(a, row, 0, 1, x, m, s);
#pragma unroll
        for (int q = 0; q < VPL; ++q) inv[q] = s[q] > 0.f ? __fdividef(1.f, s[q]) : 0.f;
#pragma unroll 1
        for (int r = 0; r < a.n_rel; ++r) {
          K::value_pass(a, r, row, 0, 1, x, m, inv, acc);
          K::store_u(a, r, row, gl, acc);
        }
      },
      [&](int64_t hr) {
#pragma unroll
        for (int q = 0; q < VPL; ++q) { m[q] = -INFINITY; s[q] = 0.f; }
        K::stats_pass(a, hr, g, G, x, m, s);
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
          const int h = gl + q * LPR;
          if (h < heads) { s_stat[(g * heads + h) * 2] = m[q]; s_stat[(g * heads + h) * 2 + 1] = s[q]; }
        }
        __syncthreads();
        // merge the groups' (max, sum) in group order; every group computes the same result
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
          const int h = gl + q * LPR;
          float M = -INFINITY, S = 0.f;
          if (h < heads) {
#pragma unroll 1
            for (int p = 0; p < G; ++p) {
              const float mq = s_stat[(p * heads + h) * 2], sq = s_stat[(p * heads + h) * 2 + 1];
              if (!(sq > 0.f)) continue;
              if (mq > M) { S = S * expf(M - mq) + sq; M = mq; }
              else S += sq * expf(mq - M);
            }
          }
          m[q] = M;
          inv[q] = S > 0.f ? __fdividef(1.f, S) : 0.f;
        }
#pragma unroll 1
        for (int r = 0; r < a.n_rel; ++r) {
          if (r > 0) __syncthreads();   // group 0 has summed the previous relation's partials
          K::value_pass(a, r, hr, g, G, x, m, inv, acc);
          put_partials<LPR>(s_part, a.H, g, gl, acc);
          __syncthreads();
          if (g == 0) {
            sum_partials<G, LPR>(s_part, a.H, gl, acc);
            K::store_u(a, r, hr, gl, acc);
          }
        }
      });
}

}  // namespace

// lane-group shape from the row width H (a multiple of 64 in [64, 1024]: 8 .. 128 vectors)
void launch_gat_full_aggregate(const GatFullAggArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value;
    launch_full_rows<LPR>(k_gat_full_aggregate<LPR, decltype(vpl)::value>, a, a.H + a.H / 8, s);
  });
}

void launch_hgt_full_attention(const HgtFullAttnArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    // up to 48 KB (H = 1024, D = 8)
    launch_full_rows<LPR>(k_hgt_full_attention<LPR, VPL>, a, LPR * VPL + 3 * a.heads + a.H, s);
  });
}

}  // namespace glt
