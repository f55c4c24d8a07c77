// Relational GAT (R-GAT) engine kernels: the attention of one relation r = (s -> t) of a heterogeneous layer over the
// sampler's per-hop ELL blocks, its backward, and the activation backward of a GAT layer.  Same conventions as
// sage.cu: extents come from device counters, grids are worst case, every kernel enters the programmatic-launch chain.
//
// Per relation, with projections h_j = W_src x_s[j] and g_i = W_dst x_t[i] (bf16, [rows, H], H = heads * C) computed
// by the TcGemm GEMMs:
//   scores     as[j, h] = <att_src[h], h_j,h>,  ad[i, h] = <att_dst[h], g_i,h>           (k_gat_scores, per node)
//   aggregate  e_ij,h = leaky_relu(as[j, h] + ad[i, h], 0.2),  alpha = softmax_j(e),
//              out_i = concat_h sum_j alpha_ij,h h_j,h                                    (k_gat_aggregate, per target)
// The relation outputs of one destination type are summed in fp32 in relation order; the last relation adds the
// summed per-relation biases, the layer activation (leaky_relu 0.01, inverted dropout) and writes bf16 Z.
// The scores are per node, not per edge, so the aggregation reads each neighbour row exactly once and the softmax is
// exact in two scalar passes (max, then sum) before the row pass: no exp of an unshifted score anywhere.
#include <cmath>

#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// keep bits of the 8 elements of 16-byte vector i of a dropout mask, drawn from dropout_bits as in k_dropout_bf16
// (sage.cu), so a mask regenerated here equals the one `dropout_bf16` draws for the same (seed, layer, step) and row
// pitch
__device__ __forceinline__ unsigned dropout_keep8(uint64_t seed, int layer, uint32_t step, int64_t i,
                                                  uint32_t thresh16) {
  const U4 r = dropout_bits(seed, layer, step, i);
  const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
  unsigned m = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q)
    if (((rr[q >> 1] >> ((q & 1) * 16)) & 0xFFFFu) >= thresh16) m |= 1u << q;
  return m;
}

__device__ __forceinline__ void load_f32x8(const float* p, float* v) {
  const float4 a = reinterpret_cast<const float4*>(p)[0], b = reinterpret_cast<const float4*>(p)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

__device__ __forceinline__ void store_f32x8(float* p, const float* v) {
  reinterpret_cast<float4*>(p)[0] = make_float4(v[0], v[1], v[2], v[3]);
  reinterpret_cast<float4*>(p)[1] = make_float4(v[4], v[5], v[6], v[7]);
}

// ---------------------------------------------------------------------------------------------------------------
// one thread per (row, head): out[row, h] = <att[h], P[row, h*C : (h+1)*C]> over the valid rows of two row sets
// (source rows of the relation and its target rows).  zero (optional, [cap0, heads]) is cleared alongside the first
// set: it is the per-source score gradient that k_gat_backward accumulates with atomics later in the step.
__global__ void __launch_bounds__(256) k_gat_scores(GatScoreArgs a) {
  pdl_enter();
  const int C = a.H / a.heads;
  const int64_t n0 = static_cast<int64_t>(a.cap[0]) * a.heads;
  const int64_t n = n0 + static_cast<int64_t>(a.cap[1]) * a.heads;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const bool set = i >= n0;                   // (selects, not indexing: keeps the parameter arrays off the stack)
    const void* P = set ? a.P[1] : a.P[0];
    if (P == nullptr) continue;
    const int64_t li = set ? i - n0 : i;
    const int row = static_cast<int>(li / a.heads), h = static_cast<int>(li % a.heads);
    if (row >= (set ? min(a.cum[1][a.idx[1]], a.cap[1]) : min(a.cum[0][a.idx[0]], a.cap[0]))) continue;
    const uint4* p = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(P) +
                                                    static_cast<int64_t>(row) * a.H + h * C);
    const uint4* w = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(set ? a.att[1] : a.att[0]) +
                                                    h * C);
    float s = 0.f;
    for (int v = 0; v < C / 8; ++v) {
      float x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      bf16x8_accum(p[v], x);
      bf16x8_accum(w[v], y);
#pragma unroll
      for (int q = 0; q < 8; ++q) s = fmaf(x[q], y[q], s);
    }
    (set ? a.out[1] : a.out[0])[li] = s;
    if (!set && a.zero) a.zero[li] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// LPR lanes per target row, each lane owns VPL 16-byte vectors (columns c * 8 .. c * 8 + 7, c = v * LPR + lane) and
// the softmax statistics of heads lane, lane + LPR, ...  alpha is saved per (ELL slot, head) with the sign of the
// pre-activation score in its sign bit (alpha >= 0): the backward needs both and reads them back, nothing is recomputed.
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_gat_aggregate(GatAggArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.H >> 3, heads = a.heads, cv = nvec / heads;
  const uint32_t step = a.step_dev ? static_cast<uint32_t>(*a.step_dev) : 0u;
  for (int base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    if (t >= T) continue;                       // whole lane groups leave together
    const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
    const int dg = a.deg[t];
    const int k = a.k[l.hop];
    const int32_t* ell = a.ell[l.hop] + static_cast<int64_t>(l.row) * k;
    float* al = a.alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
    // softmax statistics per head: max, then sum, then the normalised alpha of every slot
    for (int h = gl; h < heads; h += LPR) {
      const float adh = a.ad[static_cast<int64_t>(t) * heads + h];
      float m = -INFINITY;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s >= 0) m = fmaxf(m, leaky(a.as[static_cast<int64_t>(s) * heads + h] + adh, 0.2f));
      }
      float sum = 0.f;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s >= 0) sum += expf(leaky(a.as[static_cast<int64_t>(s) * heads + h] + adh, 0.2f) - m);
      }
      const float inv = sum > 0.f ? 1.f / sum : 0.f;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        float w = -0.f;
        if (s >= 0) {
          const float raw = a.as[static_cast<int64_t>(s) * heads + h] + adh;
          w = expf(leaky(raw, 0.2f) - m) * inv;
          if (!(raw > 0.f)) w = -w;
        }
        al[j * heads + h] = w;
      }
    }
    __syncwarp(gmask);
    float acc[VPL][8];
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[v][q] = 0.f;
    for (int j = 0; j < dg; ++j) {
      const int s = ell[j];
      if (s < 0) continue;
      const uint8_t* p = reinterpret_cast<const uint8_t*>(a.P) + static_cast<int64_t>(s) * a.H * 2;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec) {
          const float w = fabsf(al[j * heads + c / cv]);
          float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          bf16x8_accum(ld_nc_v4(p + c * 16), x);
#pragma unroll
          for (int q = 0; q < 8; ++q) acc[v][q] = fmaf(w, x[q], acc[v][q]);
        }
      }
    }
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      const int64_t e = static_cast<int64_t>(t) * a.H + c * 8;
      float o[8];
      if (a.first) {
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = acc[v][q];
      } else {
        load_f32x8(a.acc + e, o);
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] += acc[v][q];
      }
      if (!a.last) { store_f32x8(a.acc + e, o); continue; }
      for (int b = 0; b < a.n_bias; ++b)
        bf16x8_accum(reinterpret_cast<const uint4*>(a.bias)[(b * a.H + c * 8) >> 3], o);
      if (a.act) {
        const unsigned keep = a.thresh16 ? dropout_keep8(a.seed, a.layer, step, e >> 3, a.thresh16) : 0xFFu;
#pragma unroll
        for (int q = 0; q < 8; ++q) o[q] = ((keep >> q) & 1u) ? leaky(o[q], 0.01f) * a.dscale : 0.f;
      }
      reinterpret_cast<uint4*>(a.z)[e >> 3] = pack_bf16x8(o, 1.f);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of one relation per target row i, given G_i (bf16 gradient of the type's layer output, pre-activation):
//   pass 1 (reads each neighbour row once)  dalpha_j,h = <G_i,h, h_j,h>   -> dal (alpha's layout)
//                                           dP[s_j] += alpha_j,h G_i,h     (vector red.add, fp32)
//   pass 2 (scalars)  ds_j,h = alpha_j,h (dalpha_j,h - sum_k alpha_k,h dalpha_k,h) * leaky'(score)
//                     da_src[s_j, h] += ds_j,h (atomic),  da_dst[i, h] = sum_j ds_j,h
// The per-head sums of pass 1 go through a per-group shared-memory row (heads need not align with lanes: C = 24, 48).
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_gat_backward(GatBwdArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  __shared__ float s_part[8][32 * VPL];         // per warp: RPW groups x (LPR * VPL) per-vector partial dots
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int warp = threadIdx.x >> 5;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  float* part = s_part[warp] + gw * LPR * VPL;
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.H >> 3, heads = a.heads, cv = nvec / heads;
  for (int base = (blockIdx.x * wpb + warp) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    if (t >= T) continue;
    const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
    const int dg = a.deg[t];
    const int k = a.k[l.hop];
    const int32_t* ell = a.ell[l.hop] + static_cast<int64_t>(l.row) * k;
    const float* al = a.alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
    float* dal = a.dal[l.hop] + static_cast<int64_t>(l.row) * k * heads;
    float g[VPL][8];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
#pragma unroll
      for (int q = 0; q < 8; ++q) g[v][q] = 0.f;
      const int c = v * LPR + gl;
      if (c < nvec) bf16x8_accum(reinterpret_cast<const uint4*>(a.G)[(static_cast<int64_t>(t) * a.H >> 3) + c], g[v]);
    }
    float ssum[VPL];                             // sum_j alpha dalpha of heads gl + q * LPR
#pragma unroll
    for (int q = 0; q < VPL; ++q) ssum[q] = 0.f;
    for (int j = 0; j < dg; ++j) {
      const int s = ell[j];
      if (s < 0) continue;
      const uint8_t* p = reinterpret_cast<const uint8_t*>(a.P) + static_cast<int64_t>(s) * a.H * 2;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec) {
          float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          bf16x8_accum(ld_nc_v4(p + c * 16), x);
          float d = 0.f;
#pragma unroll
          for (int q = 0; q < 8; ++q) d = fmaf(g[v][q], x[q], d);
          part[c] = d;
          const float w = fabsf(al[j * heads + c / cv]);
          float y[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) y[q] = w * g[v][q];
          red_add8(a.dP + static_cast<int64_t>(s) * a.H + c * 8, y);
        }
      }
      __syncwarp(gmask);
#pragma unroll
      for (int q = 0; q < VPL; ++q) {
        const int h = gl + q * LPR;
        if (h < heads) {
          float d = 0.f;
          for (int c = h * cv; c < (h + 1) * cv; ++c) d += part[c];
          dal[j * heads + h] = d;
          ssum[q] = fmaf(fabsf(al[j * heads + h]), d, ssum[q]);
        }
      }
      __syncwarp(gmask);
    }
#pragma unroll
    for (int q = 0; q < VPL; ++q) {
      const int h = gl + q * LPR;
      if (h >= heads) continue;
      float dd = 0.f;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s < 0) continue;
        const float w = al[j * heads + h];
        const float ds = fabsf(w) * (dal[j * heads + h] - ssum[q]) * (signbit(w) ? 0.2f : 1.f);
        atomicAdd(a.da_src + static_cast<int64_t>(s) * heads + h, ds);
        dd += ds;
      }
      a.da_dst[static_cast<int64_t>(t) * heads + h] = dd;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Closes the backward of one relation over the rows of its two projections (blockIdx.y = 0: source rows,
// 1: destination rows when they are a separate projection).  Each thread keeps one 8-column group, so the attention
// vector gradients are per-CTA column partials reduced in shared memory, one atomic per column per CTA.
//   source rows j < n_src:  dPb[j] = bf16(dP[j] + da_src[j, h] att_src[h] (+ da_dst[j, h] att_dst[h] if folded)),
//                           d att_src += da_src[j, h] P[j, h-block]  (d att_dst likewise); dP[j] is zeroed for the
//                           next use; rows [n_src, round_up(n_src, 128)) of dPb are written as zeros (wgrad tiles)
//   destination rows i < T: dPb[i] = bf16(da_dst[i, h] att_dst[h]),  d att_dst += da_dst[i, h] P[i, h-block]
__global__ void __launch_bounds__(256) k_gat_score_bwd(GatScoreBwdArgs a) {
  pdl_enter();
  __shared__ float s_acc[2][256][8];
  const int seg = blockIdx.y;
  const GatScoreBwdArgs::Seg& S = a.seg[seg];
  const int nvec = a.H >> 3, heads = a.heads, cv = nvec / heads;
  const int rpb = 256 / nvec;                      // rows per block iteration (nvec <= 128)
  const int cg = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  const int h = cg / cv;
  float acc0[8], acc1[8], att0[8], att1[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) acc0[q] = acc1[q] = att0[q] = att1[q] = 0.f;
  if (S.P != nullptr) {
    const int n = min(S.cum[S.idx], S.cap);
    const int zero_end = min(S.cap, (n + 127) / 128 * 128);
    if (S.att0) bf16x8_accum(reinterpret_cast<const uint4*>(S.att0)[cg], att0);
    if (S.att1) bf16x8_accum(reinterpret_cast<const uint4*>(S.att1)[cg], att1);
    const int n1 = S.da1 ? min(S.cum1[S.idx1], n) : 0;   // rows carrying the second (destination) term
    if (rl < rpb) {
      for (int r = blockIdx.x * rpb + rl; r < zero_end; r += gridDim.x * rpb) {
        const int64_t e = static_cast<int64_t>(r) * a.H + cg * 8;
        float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (r < n) {
          if (S.dP) {
            load_f32x8(S.dP + e, o);
            const float z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            store_f32x8(S.dP + e, z);
          }
          float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          bf16x8_accum(reinterpret_cast<const uint4*>(S.P)[e >> 3], x);
          const float d0 = S.da0[static_cast<int64_t>(r) * heads + h];
#pragma unroll
          for (int q = 0; q < 8; ++q) { o[q] = fmaf(d0, att0[q], o[q]); acc0[q] = fmaf(d0, x[q], acc0[q]); }
          if (r < n1) {
            const float d1 = S.da1[static_cast<int64_t>(r) * heads + h];
#pragma unroll
            for (int q = 0; q < 8; ++q) { o[q] = fmaf(d1, att1[q], o[q]); acc1[q] = fmaf(d1, x[q], acc1[q]); }
          }
        }
        reinterpret_cast<uint4*>(S.dPb)[e >> 3] = pack_bf16x8(o, 1.f);
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) { s_acc[0][threadIdx.x][q] = acc0[q]; s_acc[1][threadIdx.x][q] = acc1[q]; }
  __syncthreads();
  if (S.P == nullptr) return;
  for (int which = 0; which < 2; ++which) {
    float* out = which ? S.gatt1 : S.gatt0;
    if (out == nullptr) continue;
    for (int c = threadIdx.x; c < a.H; c += blockDim.x) {
      float v = 0.f;
      for (int t = c >> 3; t < rpb * nvec; t += nvec) v += s_acc[which][t][c & 7];
      if (v != 0.f) atomicAdd(out + c, v);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Activation backward of a GAT layer output plus the bias gradients of its relations.
//   dH != nullptr: dPre = bf16(dH * leaky'(Z) * keep / (1 - p)) for rows < T (Z > 0 <=> pre-activation > 0; the
//                  keep mask is regenerated from its Philox key, never inferred from Z == 0); rows [T, cap) = 0
//   dH == nullptr: dPre is only read (the last layer: its gradient comes straight from the head GEMM)
//   bias_g[b * d + c] += sum_{rows < T} dPre[:, c] for b < n_bias (every relation's bias sees the same gradient)
__global__ void __launch_bounds__(256) k_gat_act_bwd(GatActBwdArgs a) {
  pdl_enter();
  __shared__ float s_acc[256][8];
  const int nvec = a.d >> 3;
  const int T = min(a.cum[a.n_hops], a.cap);
  const uint32_t step = a.step_dev ? static_cast<uint32_t>(*a.step_dev) : 0u;
  const int rpb = 256 / nvec;
  const int cg = threadIdx.x % nvec, rl = threadIdx.x / nvec;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (rl < rpb) {
    const int end = a.dH ? a.cap : T;
    for (int r = blockIdx.x * rpb + rl; r < end; r += gridDim.x * rpb) {
      const int64_t e = static_cast<int64_t>(r) * a.d + cg * 8;
      uint4 o = make_uint4(0, 0, 0, 0);
      if (a.dH) {
        if (r < T) {
          float g[8], z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          load_f32x8(a.dH + e, g);
          bf16x8_accum(reinterpret_cast<const uint4*>(a.Z)[e >> 3], z);
          const unsigned keep = a.thresh16 ? dropout_keep8(a.seed, a.layer, step, e >> 3, a.thresh16) : 0xFFu;
#pragma unroll
          for (int q = 0; q < 8; ++q) g[q] = ((keep >> q) & 1u) ? g[q] * (z[q] > 0.f ? 1.f : a.slope) * a.dscale : 0.f;
          o = pack_bf16x8(g, 1.f);
        }
        reinterpret_cast<uint4*>(a.dPre)[e >> 3] = o;
      } else {
        o = reinterpret_cast<const uint4*>(a.dPre)[e >> 3];
      }
      if (r < T) bf16x8_accum(o, acc);            // sum exactly what the GEMMs see (bf16-rounded)
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) s_acc[threadIdx.x][q] = acc[q];
  __syncthreads();
  if (a.bias_g == nullptr) return;
  for (int c = threadIdx.x; c < a.d; c += blockDim.x) {
    float v = 0.f;
    for (int t = c >> 3; t < rpb * nvec; t += nvec) v += s_acc[t][c & 7];
    if (v != 0.f)
      for (int b = 0; b < a.n_bias; ++b) atomicAdd(a.bias_g + static_cast<int64_t>(b) * a.d + c, v);
  }
}

}  // namespace

void launch_gat_scores(const GatScoreArgs& a, cudaStream_t s) {
  const int64_t n = (static_cast<int64_t>(a.cap[0]) + a.cap[1]) * a.heads;
  launch_k(k_gat_scores, dim3(grid_for(n, 256)), dim3(256), 0, s, a);
}

// lane-group shape from the row width H (a multiple of 64 in [64, 1024]: 8 .. 128 vectors)
void launch_gat_aggregate(const GatAggArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_gat_aggregate<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

void launch_gat_backward(const GatBwdArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_gat_backward<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

void launch_gat_score_bwd(const GatScoreBwdArgs& a, cudaStream_t s) {
  const int rpb = 256 / (a.H / 8);
  int cap = a.seg[0].cap;
  if (a.seg[1].P) cap = cap > a.seg[1].cap ? cap : a.seg[1].cap;
  launch_k(k_gat_score_bwd, dim3(grid_for(cap, rpb * 4, 132 * 4), a.seg[1].P ? 2 : 1), dim3(256), 0, s, a);
}

void launch_gat_act_bwd(const GatActBwdArgs& a, cudaStream_t s) {
  const int rpb = 256 / (a.d / 8);
  launch_k(k_gat_act_bwd, dim3(grid_for(a.cap, rpb * 4, 132 * 4)), dim3(256), 0, s, a);
}

}  // namespace glt
