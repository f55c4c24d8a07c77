// Knowledge-graph embedding kernels of KgeEngine (models/kge.py): TransE, DistMult, ComplEx and RotatE.  One training
// step is
//   k_m2v_begin        advance the device step counters (skipgram.cu; [next step, Adam step, current step])
//   k_kge_negatives    thread per (positive, draw): the corrupted head or tail id
//   k_kge_loss_grad    lane group per positive: its K negatives share the positive's rows; loss, red.add gradients,
//                      touched flags; relation gradients pre-reduced per CTA in shared memory
//   k_sparse_adam      twice (skipgram.cu): entity and relation tables, on the rows flagged touched
// and reads nothing back to the host, so the step is captured into one CUDA graph.  Evaluation:
//   k_kge_score        lane group per triple: the forward score
//   k_kge_den          warp per entity: TransE's normalisation denominator max(||e||_p, 1e-12), for ranking
//   k_kge_query        warp per query: the query vector (h∘r, n(h) + r, ...)
//   k_kge_rank         (query tiles) x (candidate splits): candidate rows staged by cp.async, double-buffered, scored
//                      against the tile's query vectors; integer counts of better and tied candidates
//
// Tables: entity rows are [D] (TransE, DistMult) or [re | im] of width 2D (ComplEx, RotatE); relation rows are [D]
// (TransE, DistMult, RotatE's phase) or [re | im] (ComplEx).
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

constexpr uint32_t kKgeNegStream = 0x4B47454Eu;
constexpr float kNormEps = 1e-12f;   // F.normalize's eps
constexpr int kRelSlots = 8;         // relation rows pre-reduced per CTA in k_kge_loss_grad

template <int M> struct Kge {
  static constexpr bool complex_ = M == kKgeComplEx || M == kKgeRotatE;
  static constexpr int PE = complex_ ? 2 : 1;              // entity parts
  static constexpr int PR = complex_ ? 2 : 1;              // relation parts in registers (RotatE: cos, sin)
  static constexpr int PRS = M == kKgeComplEx ? 2 : 1;     // relation parts stored (and of its gradient)
  static constexpr bool margin_loss = M == kKgeTransE || M == kKgeDistMult;
};

// Lane gl of a group of LPR lanes owns the 8-column vectors gl + v * LPR (v < VPL) of every part of a row.
template <int P, int LPR, int VPL>
__device__ __forceinline__ void load_parts(const float* row, int D, int gl, float (&x)[P][VPL * 8]) {
  const int nvec = D >> 3;
#pragma unroll
  for (int p = 0; p < P; ++p)
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = gl + v * LPR;
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
      if (c < nvec) {
        const float4* q = reinterpret_cast<const float4*>(row + p * D + c * 8);
        a = q[0];
        b = q[1];
      }
      float* o = &x[p][v * 8];
      o[0] = a.x; o[1] = a.y; o[2] = a.z; o[3] = a.w; o[4] = b.x; o[5] = b.y; o[6] = b.z; o[7] = b.w;
    }
}

template <int P, int LPR, int VPL>
__device__ __forceinline__ void red_parts(float* row, int D, int gl, const float (&g)[P][VPL * 8]) {
  const int nvec = D >> 3;
#pragma unroll
  for (int p = 0; p < P; ++p)
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = gl + v * LPR;
      if (c < nvec) red_add8(row + p * D + c * 8, &g[p][v * 8]);
    }
}

template <int LPR>
__device__ __forceinline__ float gsum(float x, unsigned gmask) {
#pragma unroll
  for (int off = LPR / 2; off > 0; off >>= 1) x += __shfl_xor_sync(gmask, x, off);
  return x;
}

// TransE: x <- x / max(||x||_p, eps) over the group's row; returns the denominator.
template <int LPR, int NC>
__device__ __forceinline__ float normalize_row(float (&x)[1][NC], int p, unsigned gmask) {
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NC; ++j) s = p == 1 ? s + fabsf(x[0][j]) : fmaf(x[0][j], x[0][j], s);
  s = gsum<LPR>(s, gmask);
  const float den = fmaxf(p == 1 ? s : sqrtf(s), kNormEps);
#pragma unroll
  for (int j = 0; j < NC; ++j) x[0][j] = __fdiv_rn(x[0][j], den);
  return den;
}

// g <- J^T g for n = e / max(||e||_p, eps), given n and the denominator: (g - s(n) (n . g)) / den with s(n) = sign(n)
// (p = 1) or n (p = 2), or g / eps when the norm was clamped (the norm's gradient is masked).
template <int LPR, int NC>
__device__ __forceinline__ void normalize_bwd(float (&g)[1][NC], const float (&n)[1][NC], float den, int p,
                                              unsigned gmask) {
  const bool clamped = den <= kNormEps;
  float ng = 0.f;
#pragma unroll
  for (int j = 0; j < NC; ++j) ng = fmaf(n[0][j], g[0][j], ng);
  ng = clamped ? 0.f : gsum<LPR>(ng, gmask);
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const float sn = p == 1 ? (n[0][j] > 0.f ? 1.f : (n[0][j] < 0.f ? -1.f : 0.f)) : n[0][j];
    g[0][j] = (g[0][j] - sn * ng) / den;
  }
}

// Lane partial of the score sum of triple (h, r, t), where the fixed entity `es` is h when tail (tail corrupted) and
// t otherwise, and `ev` is the other one (tail is uniform over a lane group, so it is a template parameter).  TransE rows are already normalised.  Sum over the group, then kge_finish.
template <int M, bool tail, int NC>
__device__ __forceinline__ float tri_partial(const float (&es)[Kge<M>::PE][NC],
                                             const float (&rr)[Kge<M>::PR][NC], const float (&ev)[Kge<M>::PE][NC],
                                             int p) {
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    if constexpr (M == kKgeTransE) {
      const float h = tail ? es[0][j] : ev[0][j], t = tail ? ev[0][j] : es[0][j];
      const float x = h + rr[0][j] - t;
      s = p == 1 ? s + fabsf(x) : fmaf(x, x, s);
    } else if constexpr (M == kKgeDistMult) {
      s = fmaf(es[0][j] * rr[0][j], ev[0][j], s);
    } else if constexpr (M == kKgeComplEx) {
      const float hr = tail ? es[0][j] : ev[0][j], hi = tail ? es[1][j] : ev[1][j];
      const float tr = tail ? ev[0][j] : es[0][j], ti = tail ? ev[1][j] : es[1][j];
      s += hr * rr[0][j] * tr + hi * rr[0][j] * ti + hr * rr[1][j] * ti - hi * rr[1][j] * tr;
    } else {
      const float hr = tail ? es[0][j] : ev[0][j], hi = tail ? es[1][j] : ev[1][j];
      const float tr = tail ? ev[0][j] : es[0][j], ti = tail ? ev[1][j] : es[1][j];
      const float a = rr[0][j] * hr - rr[1][j] * hi - tr, b = rr[0][j] * hi + rr[1][j] * hr - ti;
      s = fmaf(a, a, fmaf(b, b, s));
    }
  }
  return s;
}

template <int M>
__device__ __forceinline__ float kge_finish(float S, int p, float margin) {
  if constexpr (M == kKgeTransE) return p == 1 ? -S : -sqrtf(S);
  else if constexpr (M == kKgeRotatE) return margin - sqrtf(S);
  else return S;
}

// c * d score / d rows of the triple of tri_partial (S: its group sum): added to the fixed entity's accumulator gs and
// the relation accumulator gr (RotatE: the phase).  The varying entity's gradient goes to gv for TransE (with respect
// to the normalised row; the caller applies normalize_bwd) and is red.added into the row gv_dst, one 8-column vector
// at a time, for the other models.
template <int M, bool tail, int LPR, int VPL>
__device__ __forceinline__ void tri_grad(const float (&es)[Kge<M>::PE][VPL * 8],
                                         const float (&rr)[Kge<M>::PR][VPL * 8],
                                         const float (&ev)[Kge<M>::PE][VPL * 8], int p, float S, float c,
                                         float (&gs)[Kge<M>::PE][VPL * 8], float (&gr)[Kge<M>::PRS][VPL * 8],
                                         float (&gv)[Kge<M>::PE][VPL * 8], float* gv_dst, int D, int gl) {
  float inv = 0.f;   // 1 / distance for the 2-norm scores, 0 at distance 0 (the norm's gradient at 0)
  if constexpr (M == kKgeTransE || M == kKgeRotatE)
    if ((M == kKgeRotatE || p == 2) && S > 0.f) inv = 1.f / sqrtf(S);
#pragma unroll
  for (int v = 0; v < VPL; ++v) {
    float gw[Kge<M>::PE][8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int j = v * 8 + e;
      if constexpr (M == kKgeTransE) {
        const float h = tail ? es[0][j] : ev[0][j], t = tail ? ev[0][j] : es[0][j];
        const float x = h + rr[0][j] - t;
        const float gx = p == 1 ? -c * (x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f)) : -c * x * inv;
        gr[0][j] += gx;                          // d/dh = gx, d/dr = gx, d/dt = -gx
        gs[0][j] += tail ? gx : -gx;
        gw[0][e] = tail ? -gx : gx;
      } else if constexpr (M == kKgeDistMult) {
        gs[0][j] += c * rr[0][j] * ev[0][j];
        gr[0][j] += c * es[0][j] * ev[0][j];
        gw[0][e] = c * es[0][j] * rr[0][j];
      } else if constexpr (M == kKgeComplEx) {
        const float hr = tail ? es[0][j] : ev[0][j], hi = tail ? es[1][j] : ev[1][j];
        const float tr = tail ? ev[0][j] : es[0][j], ti = tail ? ev[1][j] : es[1][j];
        const float rre = rr[0][j], rim = rr[1][j];
        const float dhr = c * (rre * tr + rim * ti), dhi = c * (rre * ti - rim * tr);   // conj(r) t
        const float dtr = c * (hr * rre - hi * rim), dti = c * (hi * rre + hr * rim);   // h r
        gr[0][j] += c * (hr * tr + hi * ti);                                            // conj(h) t
        gr[1][j] += c * (hr * ti - hi * tr);
        gs[0][j] += tail ? dhr : dtr;
        gs[1][j] += tail ? dhi : dti;
        gw[0][e] = tail ? dtr : dhr;
        gw[1][e] = tail ? dti : dhi;
      } else {
        const float hr = tail ? es[0][j] : ev[0][j], hi = tail ? es[1][j] : ev[1][j];
        const float tr = tail ? ev[0][j] : es[0][j], ti = tail ? ev[1][j] : es[1][j];
        const float cs = rr[0][j], sn = rr[1][j];
        const float a = cs * hr - sn * hi - tr, b = cs * hi + sn * hr - ti;
        const float ga = -c * a * inv, gb = -c * b * inv;
        const float dhr = ga * cs + gb * sn, dhi = gb * cs - ga * sn;
        gr[0][j] += ga * (-sn * hr - cs * hi) + gb * (cs * hr - sn * hi);
        gs[0][j] += tail ? dhr : -ga;
        gs[1][j] += tail ? dhi : -gb;
        gw[0][e] = tail ? -ga : dhr;
        gw[1][e] = tail ? -gb : dhi;
      }
    }
    if constexpr (M == kKgeTransE) {
#pragma unroll
      for (int e = 0; e < 8; ++e) gv[0][v * 8 + e] = gw[0][e];
    } else {
      const int cv = gl + v * LPR;
      if (cv < (D >> 3))
#pragma unroll
        for (int q = 0; q < Kge<M>::PE; ++q) red_add8(gv_dst + q * D + cv * 8, gw[q]);
    }
  }
}

// Relation row of the registers: RotatE's phase becomes (cos, sin).
template <int M, int LPR, int VPL>
__device__ __forceinline__ void load_rel(const float* row, int D, int gl, float (&rr)[Kge<M>::PR][VPL * 8]) {
  if constexpr (M == kKgeRotatE) {
    float th[1][VPL * 8];
    load_parts<1, LPR, VPL>(row, D, gl, th);
#pragma unroll
    for (int j = 0; j < VPL * 8; ++j) sincosf(th[0][j], &rr[1][j], &rr[0][j]);
  } else {
    load_parts<Kge<M>::PR, LPR, VPL>(row, D, gl, rr);
  }
}

__global__ void __launch_bounds__(256) k_kge_negatives(const int32_t* n_dev, int B, int K, int64_t N, uint64_t seed,
                                                       const int32_t* step_dev, int64_t* neg) {
  pdl_enter();
  const int n = min(*n_dev, B);
  const uint64_t step = static_cast<uint32_t>(*step_dev);
  const int64_t total = static_cast<int64_t>(n) * K;
  for (int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; q < total;
       q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t i = q / K;
    const int j = static_cast<int>(q - i * K);
    neg[q] = bounded(philox_draw(seed, kKgeNegStream, (step << 32) | static_cast<uint32_t>(i), j),
                     static_cast<uint32_t>(N));
  }
}

// Lane group per positive i < n (n = *n_dev): positive (h, r, t) = trip[0 / 1 / 2][i]; its K negatives replace the
// head (i < n / 2) or the tail with neg[i * K + j].  Margin models: loss += max(0, margin - s_i + s_ij) / (n K);
// BCE models: loss += (softplus(-s_i) + sum_j softplus(s_ij)) / (n + n K).  A triple or negative with an id out of
// range is skipped.  Relation gradients of the CTA's positives collect in kRelSlots shared rows (a relation without a
// slot goes straight to global memory) and are red.added once at the end.
template <int M, int LPR, int VPL>
__global__ void __launch_bounds__(256) k_kge_loss_grad(const int64_t* trip, int B, const int32_t* n_dev,
                                                       const int64_t* neg, int K, const float* ent, const float* rel,
                                                       int64_t N, int64_t R, int D, float margin, int p, float* gent,
                                                       float* grel, uint8_t* tent, uint8_t* trel, float* loss) {
  using T = Kge<M>;
  constexpr int NC = VPL * 8, GPW = 32 / LPR;
  extern __shared__ float4 s_dyn[];
  float* s_rel = reinterpret_cast<float*>(s_dyn);
  __shared__ int s_key[kRelSlots];
  const int WE = T::PE * D, WR = T::PRS * D;
  for (int i = threadIdx.x; i < kRelSlots * WR; i += blockDim.x) s_rel[i] = 0.f;
  if (threadIdx.x < kRelSlots) s_key[threadIdx.x] = -1;
  __syncthreads();
  pdl_enter();
  const int lane = threadIdx.x & 31, gl = lane % LPR, gw = lane / LPR;
  const unsigned gmask = 0xffffffffu >> (32 - LPR) << (gw * LPR);
  const int wpb = blockDim.x >> 5;
  const int n = min(*n_dev, B);
  const float inv_pairs = T::margin_loss ? 1.f / (static_cast<float>(n) * K) : 1.f / (static_cast<float>(n) * (K + 1));
  float l_acc = 0.f;
  for (int base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * GPW; base < n; base += gridDim.x * wpb * GPW) {
    const int i = base + gw;
    if (i >= n) continue;                            // no collectives below span lane groups
    const int64_t h = trip[i], r = trip[B + i], t = trip[2 * static_cast<int64_t>(B) + i];
    if (h < 0 || h >= N || t < 0 || t >= N || r < 0 || r >= R) continue;
    const bool tail = i >= n / 2;
    const int64_t es_id = tail ? h : t, ev_id = tail ? t : h;
    float es[T::PE][NC], ev[T::PE][NC], rr[T::PR][NC];
    float gs[T::PE][NC], gr[T::PRS][NC], gv[T::PE][NC];
    load_parts<T::PE, LPR, VPL>(ent + es_id * WE, D, gl, es);
    load_parts<T::PE, LPR, VPL>(ent + ev_id * WE, D, gl, ev);
    load_rel<M, LPR, VPL>(rel + r * WR, D, gl, rr);
#pragma unroll
    for (int j = 0; j < NC; ++j) {
#pragma unroll
      for (int q = 0; q < T::PE; ++q) gs[q][j] = 0.f;
#pragma unroll
      for (int q = 0; q < T::PRS; ++q) gr[q][j] = 0.f;
    }
    float den_s = 1.f, den_v = 1.f;
    if constexpr (M == kKgeTransE) {
      den_s = normalize_row<LPR>(es, p, gmask);
      den_v = normalize_row<LPR>(ev, p, gmask);
    }
    if (gl == 0) {
      tent[h] = 1;
      tent[t] = 1;
      trel[r] = 1;
    }
    // the triple's orientation is uniform over the group: one branch per call instead of a select per column
    auto partial = [&](const float (&x)[T::PE][NC]) {
      return gsum<LPR>(tail ? tri_partial<M, true>(es, rr, x, p) : tri_partial<M, false>(es, rr, x, p), gmask);
    };
    auto grad = [&](const float (&x)[T::PE][NC], float S, float c, float* dst) {
      if (tail) tri_grad<M, true, LPR, VPL>(es, rr, x, p, S, c, gs, gr, gv, dst, D, gl);
      else tri_grad<M, false, LPR, VPL>(es, rr, x, p, S, c, gs, gr, gv, dst, D, gl);
    };
    const float S_pos = partial(ev);
    const float s_pos = kge_finish<M>(S_pos, p, margin);
    // BCE: the positive's gradient is known now, and its varying row is not needed after it
    if constexpr (!T::margin_loss) {
      const float sp = fmaxf(-s_pos, 0.f) + log1pf(expf(-fabsf(s_pos)));
      l_acc += gl == 0 ? sp * inv_pairs : 0.f;
      const float c = -inv_pairs / (1.f + expf(s_pos));     // d softplus(-s) / ds = -sigmoid(-s)
      grad(ev, S_pos, c, gent + ev_id * WE);
    }
    int active = 0;
    for (int j = 0; j < K; ++j) {
      const int64_t x = neg[static_cast<int64_t>(i) * K + j];
      if (x < 0 || x >= N) continue;
      float nv[T::PE][NC];
      load_parts<T::PE, LPR, VPL>(ent + x * WE, D, gl, nv);
      float den_n = 1.f;
      if constexpr (M == kKgeTransE) den_n = normalize_row<LPR>(nv, p, gmask);
      if (gl == 0) tent[x] = 1;
      const float S = partial(nv);
      const float s = kge_finish<M>(S, p, margin);
      float c;
      if constexpr (T::margin_loss) {
        const float term = margin - s_pos + s;
        if (!(term > 0.f)) continue;
        l_acc += gl == 0 ? term * inv_pairs : 0.f;
        ++active;
        c = inv_pairs;
      } else {
        l_acc += gl == 0 ? (fmaxf(s, 0.f) + log1pf(expf(-fabsf(s)))) * inv_pairs : 0.f;
        c = inv_pairs / (1.f + expf(-s));                   // d softplus(s) / ds = sigmoid(s)
      }
      grad(nv, S, c, gent + x * WE);
      if constexpr (M == kKgeTransE) {
        normalize_bwd<LPR>(gv, nv, den_n, p, gmask);
        red_parts<T::PE, LPR, VPL>(gent + x * WE, D, gl, gv);
      }
    }
    if constexpr (T::margin_loss) {
      if (active > 0) {
        grad(ev, S_pos, -active * inv_pairs, gent + ev_id * WE);
        if constexpr (M == kKgeTransE) {
          normalize_bwd<LPR>(gv, ev, den_v, p, gmask);
          red_parts<T::PE, LPR, VPL>(gent + ev_id * WE, D, gl, gv);
        }
      }
    }
    if constexpr (M == kKgeTransE) normalize_bwd<LPR>(gs, es, den_s, p, gmask);
    red_parts<T::PE, LPR, VPL>(gent + es_id * WE, D, gl, gs);
    // relation gradient: into this CTA's shared row of relation r when it has (or can claim) one
    int slot = -1;
    if (gl == 0) {
      for (int k = 0; k < kRelSlots; ++k) {
        int key = reinterpret_cast<volatile int*>(s_key)[k];
        if (key == -1) key = atomicCAS(&s_key[k], -1, static_cast<int>(r));
        if (key == -1 || key == static_cast<int>(r)) {
          slot = k;
          break;
        }
      }
    }
    slot = __shfl_sync(gmask, slot, 0, LPR);
    if (slot < 0) {
      red_parts<T::PRS, LPR, VPL>(grel + r * WR, D, gl, gr);
    } else {
      float* srow = s_rel + slot * WR;
#pragma unroll
      for (int q = 0; q < T::PRS; ++q)
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = gl + v * LPR;
          if (c >= (D >> 3)) continue;
#pragma unroll
          for (int e = 0; e < 8; ++e) atomicAdd(srow + q * D + c * 8 + e, gr[q][v * 8 + e]);
        }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) l_acc += __shfl_xor_sync(0xffffffffu, l_acc, off);
  if (lane == 0 && l_acc != 0.f) atomicAdd(loss, l_acc);
  __syncthreads();
  for (int k = 0; k < kRelSlots; ++k) {
    const int key = s_key[k];
    if (key < 0) continue;
    const float4* src = reinterpret_cast<const float4*>(s_rel + k * WR);
    float4* dst = reinterpret_cast<float4*>(grel + static_cast<int64_t>(key) * WR);
    for (int c = threadIdx.x; c < WR / 4; c += blockDim.x) atomicAdd(dst + c, src[c]);
  }
}

// Lane group per triple i < n: out[i] = score(h[i], r[i], t[i]); ids are checked by the binding.
template <int M, int LPR, int VPL>
__global__ void __launch_bounds__(256) k_kge_score(const int64_t* hs, const int64_t* rs, const int64_t* ts, int64_t n,
                                                   const float* ent, const float* rel, int D, float margin, int p,
                                                   float* out) {
  using T = Kge<M>;
  constexpr int NC = VPL * 8, GPW = 32 / LPR;
  pdl_enter();
  const int lane = threadIdx.x & 31, gl = lane % LPR, gw = lane / LPR;
  const unsigned gmask = 0xffffffffu >> (32 - LPR) << (gw * LPR);
  const int wpb = blockDim.x >> 5;
  const int WE = T::PE * D, WR = T::PRS * D;
  for (int64_t base = (static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5)) * GPW; base < n;
       base += static_cast<int64_t>(gridDim.x) * wpb * GPW) {
    const int64_t i = base + gw;
    if (i >= n) continue;
    float hh[T::PE][NC], tt[T::PE][NC], rr[T::PR][NC];
    load_parts<T::PE, LPR, VPL>(ent + hs[i] * WE, D, gl, hh);
    load_parts<T::PE, LPR, VPL>(ent + ts[i] * WE, D, gl, tt);
    load_rel<M, LPR, VPL>(rel + rs[i] * WR, D, gl, rr);
    if constexpr (M == kKgeTransE) {
      normalize_row<LPR>(hh, p, gmask);
      normalize_row<LPR>(tt, p, gmask);
    }
    const float s = kge_finish<M>(gsum<LPR>(tri_partial<M, true>(hh, rr, tt, p), gmask), p, margin);
    if (gl == 0) out[i] = s;
  }
}

// ---- ranking ---------------------------------------------------------------------------------------------------------
// Every model scores a candidate entity row e against a query vector q of the same width W (the entity width):
//   DistMult, ComplEx   s = sum q e                     tail q = h∘r, head q = r∘t (ComplEx: conj(r) t) [re | im]
//   TransE              s = -||q - n(e)||_p              tail q = n(h) + r, head q = n(t) - r
//   RotatE              s = margin - ||q - e||_2         tail q = h∘e^{iθ}, head q = t∘e^{-iθ}
// rank_term / rank_finish are the one code path that scores a pair, for the candidates and for the true entity alike.
constexpr int kRankQ = 64;    // queries per CTA
constexpr int kRankC = 64;    // candidates per tile
constexpr int kRankK = 32;    // columns per pipeline step
constexpr int kRankLd = kRankK + 4;

template <int M>
__device__ __forceinline__ float rank_term(float acc, float q, float e, int p) {
  if constexpr (M == kKgeDistMult || M == kKgeComplEx) return fmaf(q, e, acc);
  const float d = __fsub_rn(q, e);
  if (M == kKgeTransE && p == 1) return __fadd_rn(acc, fabsf(d));
  return fmaf(d, d, acc);
}

template <int M>
__device__ __forceinline__ float rank_finish(float acc, int p, float margin) {
  if constexpr (M == kKgeDistMult || M == kKgeComplEx) return acc;
  else if constexpr (M == kKgeTransE) return p == 1 ? -acc : -sqrtf(acc);
  else return __fsub_rn(margin, sqrtf(acc));
}

__global__ void __launch_bounds__(256) k_kge_den(const float* ent, int64_t N, int D, int p, float* den) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  for (int64_t e = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; e < N;
       e += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    float s = 0.f;
    for (int c = lane; c < D; c += 32) {
      const float x = ent[e * D + c];
      s = p == 1 ? s + fabsf(x) : fmaf(x, x, s);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (lane == 0) den[e] = fmaxf(p == 1 ? s : sqrtf(s), kNormEps);
  }
}

// Warp per query i with fixed entity f = (tail ? h : t): q[i] = the query vector.
template <int M>
__global__ void __launch_bounds__(256) k_kge_query(const int64_t* hs, const int64_t* rs, const int64_t* ts, int64_t n,
                                                   bool tail, const float* ent, const float* rel, const float* den,
                                                   int D, float* q) {
  using T = Kge<M>;
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int WE = T::PE * D, WR = T::PRS * D;
  for (int64_t i = (static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5; i < n;
       i += (static_cast<int64_t>(gridDim.x) * blockDim.x) >> 5) {
    const int64_t f = tail ? hs[i] : ts[i];
    const float* fe = ent + f * WE;
    const float* rw = rel + rs[i] * WR;
    float* qo = q + i * WE;
    for (int c = lane; c < D; c += 32) {
      if constexpr (M == kKgeTransE) {
        const float x = __fdiv_rn(fe[c], den[f]);
        qo[c] = tail ? __fadd_rn(x, rw[c]) : __fsub_rn(x, rw[c]);
      } else if constexpr (M == kKgeDistMult) {
        qo[c] = __fmul_rn(fe[c], rw[c]);
      } else {
        float cr, ci;
        if constexpr (M == kKgeComplEx) {
          cr = rw[c];
          ci = rw[D + c];
        } else {
          sincosf(rw[c], &ci, &cr);
        }
        if (!tail) ci = -ci;                      // conj(r) (ComplEx), e^{-iθ} (RotatE)
        const float fr = fe[c], fi = fe[D + c];
        qo[c] = fr * cr - fi * ci;
        qo[D + c] = fi * cr + fr * ci;
      }
    }
  }
}

// first index of the sorted keys[0, n) that is >= x
__device__ __forceinline__ int64_t lower_bound_key(const int64_t* keys, int64_t n, int64_t x) {
  int64_t a = 0;
  while (a < n) {
    const int64_t m = (a + n) >> 1;
    if (keys[m] < x) a = m + 1; else n = m;
  }
  return a;
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// Grid (query tiles of 64, candidate splits); 256 threads as 16 x 16, thread (ty, tx) owns queries ty + 16 a and
// candidates tx + 16 b (a, b < 4).  The true entity's score comes first, by the same rank_term / rank_finish sequence
// in the same column order as the sweep, so it is bitwise the score the sweep gives it.  Split y sweeps candidate tiles [y per, (y + 1) per) of 64 ids; each tile is
// streamed in 32-column steps, query and candidate columns by cp.async into a two-stage ring (TransE divides the
// candidate columns by den[] in shared memory).  Thread i < 64 owns query i's filter cursor: entered by binary search
// at the split's first id, it only moves forward and gives each tile a 64-bit mask of filtered ids.  Candidate c of
// query i counts as better (s_c > s_t) or tied (s_c == s_t) unless c is the true id, filtered or >= N; the counts
// leave the CTA as one 64-bit atomic per query, (better << 32) + tied.
template <int M>
__global__ void __launch_bounds__(256) k_kge_rank(const float* q, const int64_t* hs, const int64_t* rs,
                                                  const int64_t* ts, bool tail, const int64_t* keys, int64_t n_keys,
                                                  const float* ent, const float* den, int64_t n, int64_t N, int64_t R,
                                                  int W, int p, float margin, int tiles_per_split,
                                                  unsigned long long* counts) {
  __shared__ __align__(16) float sq[2][kRankQ][kRankLd];
  __shared__ __align__(16) float sc[2][kRankC][kRankLd];
  __shared__ uint64_t s_mask[kRankQ];
  __shared__ float s_true[kRankQ];
  __shared__ int64_t s_truth[kRankQ];
  pdl_enter();
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t q0 = static_cast<int64_t>(blockIdx.x) * kRankQ;
  const int64_t c_tiles = (N + kRankC - 1) / kRankC;
  const int64_t t_begin = static_cast<int64_t>(blockIdx.y) * tiles_per_split;
  const int64_t t_end = min(c_tiles, t_begin + tiles_per_split);
  // query tid: true score (same pair code as the sweep), filter cursor
  int64_t cur = 0, fend = 0, kbase = 0;
  if (tid < kRankQ) {
    const int64_t i = q0 + tid;
    float s = 0.f;
    int64_t tr = -1;
    if (i < n) {
      tr = tail ? ts[i] : hs[i];
      const float* qi = q + i * W;
      const float* e = ent + tr * W;
      float acc = 0.f;
      for (int k = 0; k < W; ++k) {
        const float ev = M == kKgeTransE ? __fdiv_rn(e[k], den[tr]) : e[k];
        acc = rank_term<M>(acc, qi[k], ev, p);
      }
      s = rank_finish<M>(acc, p, margin);
      if (keys != nullptr) {
        kbase = ((tail ? hs[i] : ts[i]) * R + rs[i]) * N;
        cur = lower_bound_key(keys, n_keys, kbase + t_begin * kRankC);
        fend = lower_bound_key(keys, n_keys, kbase + N);
      }
    }
    s_true[tid] = s;
    s_truth[tid] = tr;
  }
  const int kc = (W + kRankK - 1) / kRankK;
  const int64_t steps = (t_end - t_begin) * kc;
  auto issue = [&](int64_t st) {
    const int buf = static_cast<int>(st & 1);
    const int64_t c0 = (t_begin + st / kc) * kRankC;
    const int k0 = static_cast<int>(st % kc) * kRankK;
#pragma unroll
    for (int u = 0; u < 2; ++u) {   // 512 float4s per operand, 2 per thread
      const int idx = tid + u * 256, row = idx >> 3, col = (idx & 7) * 4;
      const bool kin = k0 + col < W;
      const int64_t qi = q0 + row, ci = c0 + row;
      cp_async16(&sq[buf][row][col], q + (kin && qi < n ? qi * W + k0 + col : 0), kin && qi < n);
      cp_async16(&sc[buf][row][col], ent + (kin && ci < N ? ci * W + k0 + col : 0), kin && ci < N);
    }
    cp_async_commit();
  };
  uint32_t better[4] = {0, 0, 0, 0}, tied[4] = {0, 0, 0, 0};
  float acc[4][4];
  if (steps > 0) issue(0);
  for (int64_t st = 0; st < steps; ++st) {
    const int buf = static_cast<int>(st & 1);
    const int kk = static_cast<int>(st % kc);
    const int64_t c0 = (t_begin + st / kc) * kRankC;
    if (kk == 0) {
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
      if (tid < kRankQ) {
        uint64_t m = 0;
        while (cur < fend) {
          const int64_t id = keys[cur] - kbase;
          if (id >= c0 + kRankC) break;
          if (id >= c0) m |= uint64_t(1) << (id - c0);
          ++cur;
        }
        s_mask[tid] = m;
      }
    }
    if (st + 1 < steps) {
      issue(st + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    if constexpr (M == kKgeTransE) {
      for (int idx = tid; idx < kRankC * kRankK; idx += 256) {
        const int row = idx / kRankK, col = idx % kRankK;
        const int64_t ci = c0 + row;
        if (ci < N) sc[buf][row][col] = __fdiv_rn(sc[buf][row][col], den[ci]);
      }
      __syncthreads();
    }
#pragma unroll 2
    for (int k = 0; k < kRankK; k += 4) {
      float4 qv[4], cv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) qv[a] = *reinterpret_cast<const float4*>(&sq[buf][ty + 16 * a][k]);
#pragma unroll
      for (int b = 0; b < 4; ++b) cv[b] = *reinterpret_cast<const float4*>(&sc[buf][tx + 16 * b][k]);
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          float x = acc[a][b];
          x = rank_term<M>(x, qv[a].x, cv[b].x, p);
          x = rank_term<M>(x, qv[a].y, cv[b].y, p);
          x = rank_term<M>(x, qv[a].z, cv[b].z, p);
          x = rank_term<M>(x, qv[a].w, cv[b].w, p);
          acc[a][b] = x;
        }
    }
    if (kk == kc - 1) {
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const int qr = ty + 16 * a;
        const float st_true = s_true[qr];
        const int64_t tr = s_truth[qr];
        const uint64_t m = s_mask[qr];
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int cl = tx + 16 * b;
          const int64_t c = c0 + cl;
          if (c >= N || c == tr || ((m >> cl) & 1)) continue;
          const float s = rank_finish<M>(acc[a][b], p, margin);
          better[a] += s > st_true;
          tied[a] += s == st_true;
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    uint32_t bt = better[a], td = tied[a];
#pragma unroll
    for (int off = 8; off > 0; off >>= 1) {
      bt += __shfl_xor_sync(0xffffffffu, bt, off);
      td += __shfl_xor_sync(0xffffffffu, td, off);
    }
    const int64_t i = q0 + ty + 16 * a;
    if (tx == 0 && i < n) atomicAdd(counts + i, (static_cast<unsigned long long>(bt) << 32) + td);
  }
}

template <class F>
void dispatch_model(int model, F&& f) {
  switch (model) {
    case kKgeTransE: f(std::integral_constant<int, kKgeTransE>()); break;
    case kKgeDistMult: f(std::integral_constant<int, kKgeDistMult>()); break;
    case kKgeComplEx: f(std::integral_constant<int, kKgeComplEx>()); break;
    default: f(std::integral_constant<int, kKgeRotatE>()); break;
  }
}

}  // namespace

int kge_entity_parts(int model) { return model == kKgeComplEx || model == kKgeRotatE ? 2 : 1; }
int kge_relation_parts(int model) { return model == kKgeComplEx ? 2 : 1; }

void launch_kge_negatives(const int32_t* n_dev, int B, int K, int64_t N, uint64_t seed, const int32_t* step_dev,
                          int64_t* neg, cudaStream_t s) {
  launch_k(k_kge_negatives, dim3(grid_for(static_cast<int64_t>(B) * K, 256)), dim3(256), 0, s, n_dev, B, K, N, seed,
           step_dev, neg);
}

void launch_kge_loss_grad(int model, const int64_t* trip, int B, const int32_t* n_dev, const int64_t* neg, int K,
                          const float* ent, const float* rel, int64_t N, int64_t R, int D, float margin, int p,
                          float* gent, float* grel, uint8_t* tent, uint8_t* trel, float* loss, cudaStream_t s) {
  cudaMemsetAsync(loss, 0, sizeof(float), s);
  const size_t smem = static_cast<size_t>(kRelSlots) * kge_relation_parts(model) * D * sizeof(float);
  dispatch_model(model, [&](auto m) {
    constexpr int M = decltype(m)::value;
    dispatch_lanes<2, 2>(D / 8, [&](auto lpr, auto vpl) {
      constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
      launch_k(k_kge_loss_grad<M, LPR, VPL>, dim3(grid_for(B, 8 * (32 / LPR))), dim3(256), smem, s, trip, B, n_dev,
               neg, K, ent, rel, N, R, D, margin, p, gent, grel, tent, trel, loss);
    });
  });
}

void launch_kge_score(int model, const int64_t* h, const int64_t* r, const int64_t* t, int64_t n, const float* ent,
                      const float* rel, int D, float margin, int p, float* out, cudaStream_t s) {
  dispatch_model(model, [&](auto m) {
    constexpr int M = decltype(m)::value;
    dispatch_lanes<2, 2>(D / 8, [&](auto lpr, auto vpl) {
      constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
      launch_k(k_kge_score<M, LPR, VPL>, dim3(grid_for(n, 8 * (32 / LPR))), dim3(256), 0, s, h, r, t, n, ent, rel, D,
               margin, p, out);
    });
  });
}

void launch_kge_rank(const KgeRankArgs& a, cudaStream_t s) {
  const int W = kge_entity_parts(a.model) * a.D;
  if (a.model == kKgeTransE)
    launch_k(k_kge_den, dim3(grid_for(a.N, 8)), dim3(256), 0, s, a.ent, a.N, a.D, a.p, a.den);
  cudaMemsetAsync(a.counts, 0, a.n * sizeof(unsigned long long), s);
  dispatch_model(a.model, [&](auto m) {
    constexpr int M = decltype(m)::value;
    launch_k(k_kge_query<M>, dim3(grid_for(a.n, 8)), dim3(256), 0, s, a.h, a.r, a.t, a.n, a.tail, a.ent, a.rel,
             static_cast<const float*>(a.den), a.D, a.q);
    const int64_t q_tiles = (a.n + kRankQ - 1) / kRankQ;
    launch_k(k_kge_rank<M>, dim3(static_cast<unsigned>(q_tiles), static_cast<unsigned>(a.splits)), dim3(256), 0, s,
             static_cast<const float*>(a.q), a.h, a.r, a.t, a.tail, a.keys, a.n_keys, a.ent,
             static_cast<const float*>(a.den), a.n, a.N, a.R, W, a.p, a.margin, a.tiles_per_split, a.counts);
  });
}

}  // namespace glt
