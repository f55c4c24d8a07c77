// Label propagation over the full graph (models/label_prop.py: LabelPropagation, CorrectAndSmooth): one launch per
// iteration, for every row i of [0, n)
//   out_i = post(alpha * s_i * sum_{j in row(i)} t_j x_j + (1 - alpha) * base_i)
// with post = clamp to [lo, hi], then out_i = base_i where fixed[i].  fp32 rows of pitch cp (a multiple of 4 floats);
// columns >= c are written as 0.
//
// Rows take the schedule of full_rows.cuh (hub rows reduced by the whole CTA, partials merged in group order) and no
// floating-point atomics are used, so every row has one fixed summation order: results are bitwise identical from call
// to call.
#include "full_rows.cuh"

namespace glt {

namespace {

__device__ __forceinline__ float4 ld_nc_f4(const float* p) {
  const uint4 u = ld_nc_v4(p);
  return make_float4(__uint_as_float(u.x), __uint_as_float(u.y), __uint_as_float(u.z), __uint_as_float(u.w));
}

// s = t = deg^-1/2 ('sym'), or s = 1 / deg ('row', t unused); a factor of a row of degree 0 is 0.
__global__ void __launch_bounds__(256) k_label_prop_factors(GraphTable g, int64_t n, int sym, float* s, float* t) {
  pdl_enter();
  for (int64_t v = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; v < n;
       v += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float deg = static_cast<float>(load_row(g, v).deg);
    if (sym) {
      const float d = deg > 0.f ? 1.f / sqrtf(deg) : 0.f;
      s[v] = d;
      t[v] = d;
    } else {
      s[v] = deg > 0.f ? 1.f / deg : 0.f;
    }
  }
}

// LPR lanes per row; each lane owns VPL vectors of 4 floats (vector c = v * LPR + gl).
template <int LPR, int VPL>
struct LabelProp {
  static constexpr int R = LPR < 8 ? LPR : 8;   // rows in flight per lane group; LPR and R are powers of two

  // acc += t_u x_u for neighbours j = first, first + stride, ... < deg of the row (part, start), in increasing j order.
  __device__ static void accumulate(const LabelPropArgs& a, int part, int64_t start, int deg, int first, int stride,
                                    int gl, unsigned gmask, float (&acc)[VPL][4]) {
    const int n = first < deg ? (deg - first + stride - 1) / stride : 0;
    const int nvec = a.cp >> 2;
    for (int i0 = 0; i0 < n; i0 += LPR) {
      const float* mine = nullptr;
      float wt = 0.f;
      if (i0 + gl < n) {
        const int64_t u = load_col(a.g, part, start + first + static_cast<int64_t>(i0 + gl) * stride);
        if (u >= 0 && u < a.n) {   // columns outside [0, n) read as zero rows
          mine = a.x + u * a.cp;
          wt = a.t ? __ldg(a.t + u) : 1.f;
        }
      }
      const int cnt = min(LPR, n - i0);
      for (int jj = 0; jj < cnt; jj += R) {
        const float* p[R];
        float w[R];
        float4 raw[R][VPL];
#pragma unroll
        for (int u = 0; u < R; ++u) {
          p[u] = reinterpret_cast<const float*>(
              __shfl_sync(gmask, reinterpret_cast<unsigned long long>(mine), jj + u, LPR));
          w[u] = __shfl_sync(gmask, wt, jj + u, LPR);
          if (jj + u >= cnt) p[u] = nullptr;
#pragma unroll
          for (int v = 0; v < VPL; ++v) raw[u][v] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < R; ++u) {
          if (p[u] == nullptr) continue;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            const int c = v * LPR + gl;
            if (c < nvec) raw[u][v] = ld_nc_f4(p[u] + c * 4);
          }
        }
#pragma unroll
        for (int u = 0; u < R; ++u) {
          if (p[u] == nullptr) continue;
#pragma unroll
          for (int v = 0; v < VPL; ++v) {
            acc[v][0] = fmaf(w[u], raw[u][v].x, acc[v][0]);
            acc[v][1] = fmaf(w[u], raw[u][v].y, acc[v][1]);
            acc[v][2] = fmaf(w[u], raw[u][v].z, acc[v][2]);
            acc[v][3] = fmaf(w[u], raw[u][v].w, acc[v][3]);
          }
        }
      }
    }
  }

  __device__ static void epilogue(const LabelPropArgs& a, int64_t r, int gl, const float (&acc)[VPL][4]) {
    const int nvec = a.cp >> 2;
    const float sr = __ldg(a.s + r);
    const bool fix = a.fixed != nullptr && a.fixed[r] != 0;
    const float* b = a.base + r * a.cp;
    float4* o = reinterpret_cast<float4*>(a.out + r * a.cp);
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      const float4 bv = ld_nc_f4(b + c * 4);
      const float bs[4] = {bv.x, bv.y, bv.z, bv.w};
      float z[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        z[e] = fix ? bs[e] : fminf(fmaxf(fmaf(a.alpha, sr * acc[v][e], a.beta * bs[e]), a.lo), a.hi);
        if (c * 4 + e >= a.c) z[e] = 0.f;
      }
      o[c] = make_float4(z[0], z[1], z[2], z[3]);
    }
  }
};

// One row per lane group (G = 256 / LPR rows per CTA); hub rows are reduced by the whole CTA.
template <int LPR, int VPL>
__global__ void __launch_bounds__(kFullRowThreads) k_label_prop(LabelPropArgs a) {
  using K = LabelProp<LPR, VPL>;
  constexpr int G = kFullRowThreads / LPR;
  extern __shared__ float s_part[];    // [G][cp] partial sums of a hub row
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int g = threadIdx.x / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << ((lane / LPR) * LPR));
  float acc[VPL][4];
  auto zero = [&]() {
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[v][e] = 0.f;
  };
  RowRef rr;
  zero();
  full_rows<G>(
      a.r0, a.r1, g, gl, [&](int64_t r) { rr = load_row(a.g, r); return rr.deg; },
      [&](int64_t r) {
        if (rr.deg > 0) K::accumulate(a, rr.part, rr.start, rr.deg, 0, 1, gl, gmask, acc);
        K::epilogue(a, r, gl, acc);
      },
      [&](int64_t hr) {
        const RowRef hb = load_row(a.g, hr);
        zero();
        K::accumulate(a, hb.part, hb.start, hb.deg, g, G, gl, gmask, acc);
        put_partials<LPR>(s_part, a.cp, g, gl, acc);
        __syncthreads();
        if (g == 0) {
          sum_partials<G, LPR>(s_part, a.cp, gl, acc);
          K::epilogue(a, hr, gl, acc);
        }
      });
}

}  // namespace

void launch_label_prop_factors(const GraphTable& g, int64_t n, bool sym, float* s, float* t, cudaStream_t st) {
  launch_k(k_label_prop_factors, dim3(grid_for(n, 256)), dim3(256), 0, st, g, n, sym ? 1 : 0, s, t);
}

void launch_label_prop(const LabelPropArgs& args, cudaStream_t s) {
  LabelPropArgs a = args;
  a.r0 = 0;
  a.r1 = a.n;
  // cp / 4 vectors of 4 floats: cp = 48 (47 classes) is <16, 1>, cp = 512 is <32, 4>
  dispatch_lanes<1, 4>(a.cp / 4, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_full_rows<LPR>(k_label_prop<LPR, VPL>, a, a.cp, s);
  });
}

}  // namespace glt
