// Heterogeneous Graph Transformer (HGT) engine kernels: the cross-relation attention of one (layer, destination type)
// over the sampler's per-hop ELL blocks, its backward, and the small fused kernels around them (exact GELU, the gated
// skip connection, the block-diagonal relation images and their gradients, the K/Q/V gradient cast).  Same conventions
// as sage.cu / gat.cu: extents come from device counters, grids are worst case, every kernel enters the
// programmatic-launch chain.
//
// Both relation transforms act on the target side (they are linear):
//   <q_i, k_j W_att>  = <q_i W_att^T, k_j>           qq_r = Q W_att,r^T      one GEMM per type over all its relations
//   sum_j a_ij v_j W_msg = (sum_j a_ij v_j) W_msg     agg  = [u_r1 | u_r2 | ...] . [W_msg,r1; W_msg,r2; ...]
// so the attention kernel reads each source row's raw K and V (one bf16 row [K | Q | V] per node) once per slot:
//   s_ij,h  = <qq_r[i, h], k_j,h> * prior_r[h] / sqrt(D)          for every slot j of every relation r into the type
//   alpha   = softmax over ALL of them per (i, h): max, then the sum of exp(s - max), then the normalised weights
//   u_r[i, h] = sum_{j in r} alpha_ij,h v_j,h
#include <cmath>

#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ float gelu_grad(float x) {
  return 0.5f * (1.f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * expf(-0.5f * x * x);
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.f / (1.f + expf(-x)); }

// ---------------------------------------------------------------------------------------------------------------
// LPR lanes per target row; a lane owns VPL 16-byte vectors (columns c * 8 .. c * 8 + 7, c = v * LPR + lane) of an
// H-wide row and the softmax statistics of heads lane, lane + LPR, ...  Per-head dot products go through a per-group
// shared-memory row (a head need not align with the lanes: D = 24, 48).
//   pass 1 (reads K once per slot)   raw scores s into alpha, running max per head over every relation
//   pass 2 (scalars)                 sum of exp(s - max) over every relation, then alpha = exp(s - max) / sum
//   pass 3 (reads V once per slot)   u_r = sum_j alpha v_j, one bf16 row segment per relation
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_hgt_attention(HgtAttnArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  __shared__ float s_part[8][32 * VPL];
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int warp = threadIdx.x >> 5;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  float* part = s_part[warp] + gw * LPR * VPL;
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.H >> 3, heads = a.heads, cv = nvec / heads;
  const int64_t ldq = static_cast<int64_t>(a.n_rel) * a.H;
  for (int base = (blockIdx.x * wpb + warp) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    if (t >= T) continue;                       // whole lane groups leave together
    const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
    float mx[VPL];
#pragma unroll
    for (int q = 0; q < VPL; ++q) mx[q] = -INFINITY;
#pragma unroll 1
    for (int r = 0; r < a.n_rel; ++r) {
      const int dg = a.rel[r].deg[t];
      const int k = a.rel[r].k[l.hop];
      const int32_t* ell = a.rel[r].ell[l.hop] + static_cast<int64_t>(l.row) * k;
      float* al = a.rel[r].alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
      const uint8_t* kv = reinterpret_cast<const uint8_t*>(a.rel[r].kv);
      float ps[VPL];
#pragma unroll
      for (int q = 0; q < VPL; ++q) {
        const int h = gl + q * LPR;
        ps[q] = h < heads ? a.rel[r].prior[h] * a.scale : 0.f;
      }
      float qv[VPL][8];
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
#pragma unroll
        for (int e = 0; e < 8; ++e) qv[v][e] = 0.f;
        const int c = v * LPR + gl;
        if (c < nvec)
          bf16x8_accum(reinterpret_cast<const uint4*>(a.qq)[((t * ldq + static_cast<int64_t>(r) * a.H) >> 3) + c], qv[v]);
      }
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s < 0) continue;
        const uint8_t* p = kv + static_cast<int64_t>(s) * a.kv_ld * 2;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec) {
            float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            bf16x8_accum(ld_nc_v4(p + c * 16), x);
            float d = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) d = fmaf(qv[v][e], x[e], d);
            part[c] = d;
          }
        }
        __syncwarp(gmask);
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
          const int h = gl + q * LPR;
          if (h < heads) {
            float d = 0.f;
            for (int c = h * cv; c < (h + 1) * cv; ++c) d += part[c];
            const float sc = d * ps[q];
            al[j * heads + h] = sc;
            mx[q] = fmaxf(mx[q], sc);
          }
        }
        __syncwarp(gmask);
      }
    }
    // softmax over every relation's slots, per head
#pragma unroll
    for (int q = 0; q < VPL; ++q) {
      const int h = gl + q * LPR;
      if (h >= heads) continue;
      float sum = 0.f;
#pragma unroll 1
      for (int r = 0; r < a.n_rel; ++r) {
        const int dg = a.rel[r].deg[t];
        const int k = a.rel[r].k[l.hop];
        const int32_t* ell = a.rel[r].ell[l.hop] + static_cast<int64_t>(l.row) * k;
        const float* al = a.rel[r].alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
        for (int j = 0; j < dg; ++j)
          if (ell[j] >= 0) sum += expf(al[j * heads + h] - mx[q]);
      }
      const float inv = sum > 0.f ? 1.f / sum : 0.f;
#pragma unroll 1
      for (int r = 0; r < a.n_rel; ++r) {
        const int dg = a.rel[r].deg[t];
        const int k = a.rel[r].k[l.hop];
        const int32_t* ell = a.rel[r].ell[l.hop] + static_cast<int64_t>(l.row) * k;
        float* al = a.rel[r].alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
        for (int j = 0; j < dg; ++j)
          al[j * heads + h] = ell[j] >= 0 ? expf(al[j * heads + h] - mx[q]) * inv : 0.f;
      }
    }
    __syncwarp(gmask);
    // alpha-weighted sums of the raw V rows, one segment per relation
#pragma unroll 1
    for (int r = 0; r < a.n_rel; ++r) {
      const int dg = a.rel[r].deg[t];
      const int k = a.rel[r].k[l.hop];
      const int32_t* ell = a.rel[r].ell[l.hop] + static_cast<int64_t>(l.row) * k;
      const float* al = a.rel[r].alpha[l.hop] + static_cast<int64_t>(l.row) * k * heads;
      const uint8_t* kv = reinterpret_cast<const uint8_t*>(a.rel[r].kv) + a.v_off * 2;
      float acc[VPL][8];
#pragma unroll
      for (int v = 0; v < VPL; ++v)
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[v][e] = 0.f;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s < 0) continue;
        const uint8_t* p = kv + static_cast<int64_t>(s) * a.kv_ld * 2;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec) {
            const float w = al[j * heads + c / cv];
            float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            bf16x8_accum(ld_nc_v4(p + c * 16), x);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[v][e] = fmaf(w, x[e], acc[v][e]);
          }
        }
      }
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec)
          reinterpret_cast<uint4*>(a.u)[((t * ldq + static_cast<int64_t>(r) * a.H) >> 3) + c] = pack_bf16x8(acc[v], 1.f);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of k_hgt_attention per target row i, given dU = dL/du (bf16 [T, n_rel * H]):
//   pass A (reads K and V once per slot)  dalpha_j,h = <dU_r[i, h], v_j,h> and the raw dot c_j,h = <qq_r[i, h], k_j,h>
//                                         into dal (two floats per (slot, head)); dV[s_j] += alpha dU_r[i] (red.add)
//   pass B (scalars)  ds = alpha (dalpha - sum over ALL relations' slots of alpha dalpha);  dprior_r[h] += ds c / sqrt(D)
//                     (per-CTA partials in shared memory);  g = ds prior_r[h] / sqrt(D) replaces dalpha in dal
//   pass C (reads K once per slot)  dqq_r[i] = sum_j g k_j (bf16 row segment),  dK[s_j] += g qq_r[i] (red.add)
// Rows [T, round_up(T, 128)) of dqq are written as zeros (the weight-gradient GEMM reads whole tiles).
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_hgt_attention_bwd(HgtAttnBwdArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  __shared__ float s_part[2][8][32 * VPL];
  __shared__ float s_prior[kHgtMaxRel * 128];
  for (int i = threadIdx.x; i < a.n_rel * a.heads; i += blockDim.x) s_prior[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int warp = threadIdx.x >> 5;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  float* part0 = s_part[0][warp] + gw * LPR * VPL;
  float* part1 = s_part[1][warp] + gw * LPR * VPL;
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.H >> 3, heads = a.heads, cv = nvec / heads;
  const int64_t ldq = static_cast<int64_t>(a.n_rel) * a.H;
  const int64_t ldg = 2 * static_cast<int64_t>(a.H);   // fp32 gradient rows [dK | dV]
  for (int base = (blockIdx.x * wpb + warp) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    if (t >= T) continue;
    const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
    float ssum[VPL];
#pragma unroll
    for (int q = 0; q < VPL; ++q) ssum[q] = 0.f;
#pragma unroll 1
    for (int r = 0; r < a.n_rel; ++r) {
      const int dg = a.rel[r].deg[t];
      const int k = a.rel[r].k[l.hop];
      const int64_t slot0 = static_cast<int64_t>(l.row) * k;
      const int32_t* ell = a.rel[r].ell[l.hop] + slot0;
      const float* al = a.rel[r].alpha[l.hop] + slot0 * heads;
      float2* dal = reinterpret_cast<float2*>(a.rel[r].dal[l.hop]) + slot0 * heads;
      const uint8_t* kv = reinterpret_cast<const uint8_t*>(a.rel[r].kv);
      float* dkv = a.rel[r].dkv;
      float g[VPL][8], qv[VPL][8];
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { g[v][e] = 0.f; qv[v][e] = 0.f; }
        const int c = v * LPR + gl;
        if (c < nvec) {
          const int64_t o = ((t * ldq + static_cast<int64_t>(r) * a.H) >> 3) + c;
          bf16x8_accum(reinterpret_cast<const uint4*>(a.du)[o], g[v]);
          bf16x8_accum(reinterpret_cast<const uint4*>(a.qq)[o], qv[v]);
        }
      }
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s < 0) continue;
        const uint8_t* p = kv + static_cast<int64_t>(s) * a.kv_ld * 2;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec) {
            float x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            bf16x8_accum(ld_nc_v4(p + a.v_off * 2 + c * 16), x);
            bf16x8_accum(ld_nc_v4(p + c * 16), y);
            float d0 = 0.f, d1 = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) { d0 = fmaf(g[v][e], x[e], d0); d1 = fmaf(qv[v][e], y[e], d1); }
            part0[c] = d0;
            part1[c] = d1;
            const float w = al[j * heads + c / cv];
            float z[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) z[e] = w * g[v][e];
            red_add8(dkv + s * ldg + a.H + c * 8, z);
          }
        }
        __syncwarp(gmask);
#pragma unroll
        for (int q = 0; q < VPL; ++q) {
          const int h = gl + q * LPR;
          if (h < heads) {
            float d0 = 0.f, d1 = 0.f;
            for (int c = h * cv; c < (h + 1) * cv; ++c) { d0 += part0[c]; d1 += part1[c]; }
            dal[j * heads + h] = make_float2(d0, d1);
            ssum[q] = fmaf(al[j * heads + h], d0, ssum[q]);
          }
        }
        __syncwarp(gmask);
      }
    }
#pragma unroll
    for (int q = 0; q < VPL; ++q) {
      const int h = gl + q * LPR;
      if (h >= heads) continue;
#pragma unroll 1
      for (int r = 0; r < a.n_rel; ++r) {
        const int dg = a.rel[r].deg[t];
        const int k = a.rel[r].k[l.hop];
        const int64_t slot0 = static_cast<int64_t>(l.row) * k;
        const int32_t* ell = a.rel[r].ell[l.hop] + slot0;
        const float* al = a.rel[r].alpha[l.hop] + slot0 * heads;
        float2* dal = reinterpret_cast<float2*>(a.rel[r].dal[l.hop]) + slot0 * heads;
        const float pr = a.rel[r].prior[h] * a.scale;
        float dp = 0.f;
        for (int j = 0; j < dg; ++j) {
          if (ell[j] < 0) continue;
          const float2 dc = dal[j * heads + h];
          const float ds = al[j * heads + h] * (dc.x - ssum[q]);
          dp = fmaf(ds, dc.y, dp);
          dal[j * heads + h].x = ds * pr;
        }
        if (dp != 0.f) atomicAdd(&s_prior[r * heads + h], dp * a.scale);
      }
    }
    __syncwarp(gmask);
#pragma unroll 1
    for (int r = 0; r < a.n_rel; ++r) {
      const int dg = a.rel[r].deg[t];
      const int k = a.rel[r].k[l.hop];
      const int64_t slot0 = static_cast<int64_t>(l.row) * k;
      const int32_t* ell = a.rel[r].ell[l.hop] + slot0;
      const float2* dal = reinterpret_cast<const float2*>(a.rel[r].dal[l.hop]) + slot0 * heads;
      const uint8_t* kv = reinterpret_cast<const uint8_t*>(a.rel[r].kv);
      float* dkv = a.rel[r].dkv;
      float qv[VPL][8], acc[VPL][8];
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
#pragma unroll
        for (int e = 0; e < 8; ++e) { qv[v][e] = 0.f; acc[v][e] = 0.f; }
        const int c = v * LPR + gl;
        if (c < nvec)
          bf16x8_accum(reinterpret_cast<const uint4*>(a.qq)[((t * ldq + static_cast<int64_t>(r) * a.H) >> 3) + c], qv[v]);
      }
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s < 0) continue;
        const uint8_t* p = kv + static_cast<int64_t>(s) * a.kv_ld * 2;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec) {
            const float w = dal[j * heads + c / cv].x;
            float x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, z[8];
            bf16x8_accum(ld_nc_v4(p + c * 16), x);
#pragma unroll
            for (int e = 0; e < 8; ++e) { acc[v][e] = fmaf(w, x[e], acc[v][e]); z[e] = w * qv[v][e]; }
            red_add8(dkv + s * ldg + c * 8, z);
          }
        }
      }
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int c = v * LPR + gl;
        if (c < nvec)
          reinterpret_cast<uint4*>(a.dqq)[((t * ldq + static_cast<int64_t>(r) * a.H) >> 3) + c] = pack_bf16x8(acc[v], 1.f);
      }
    }
  }
  // zero rows past the targets up to the next 128-row tile
  const int zend = min(a.cap_targets, (T + 127) / 128 * 128);
  const int64_t nz = static_cast<int64_t>(zend - T) * (ldq >> 3);
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < nz;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    reinterpret_cast<uint4*>(a.dqq)[static_cast<int64_t>(T) * (ldq >> 3) + i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  for (int i = threadIdx.x; i < a.n_rel * a.heads; i += blockDim.x) {
    const float v = s_prior[i];
    if (v != 0.f) atomicAdd(a.rel[i / a.heads].dprior + i % a.heads, v);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Elementwise kernels over rows < T = min(cum[n_hops], cap) of [cap, d] bf16 rows, one 16-byte vector per thread.
//   gelu      Y = gelu(X) (exact erf form); X is kept for the backward
//   gelu_bwd  dX = bf16(dY gelu'(X)); rows [T, round_up(T, 128)) = 0
__global__ void __launch_bounds__(256) k_hgt_gelu(const __nv_bfloat16* X, __nv_bfloat16* Y, const int32_t* cum,
                                                  int n_hops, int cap, int d, const __nv_bfloat16* dY) {
  pdl_enter();
  const int T = min(cum[n_hops], cap);
  const int nvec = d >> 3;
  const int end = dY ? min(cap, (T + 127) / 128 * 128) : T;
  const int64_t n = static_cast<int64_t>(end) * nvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float x[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (i / nvec >= T) { reinterpret_cast<uint4*>(Y)[i] = make_uint4(0, 0, 0, 0); continue; }
    bf16x8_accum(reinterpret_cast<const uint4*>(X)[i], x);
    if (dY) {
      float g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      bf16x8_accum(reinterpret_cast<const uint4*>(dY)[i], g);
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = g[e] * gelu_grad(x[e]);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) x[e] = gelu_f(x[e]);
    }
    reinterpret_cast<uint4*>(Y)[i] = pack_bf16x8(x, 1.f);
  }
}

// Gated skip connection, forward: Z = sigmoid(skip) A + (1 - sigmoid(skip)) X on rows < T.
// Backward (dZ32 or dZ16 given): dA = bf16(sigmoid(skip) dZ) on rows < T, 0 on [T, round_up(T, 128));
// dX += (1 - sigmoid(skip)) dZ (fp32, optional); skip_g += sum dZ (A - X) sigmoid'(skip), one atomic per CTA.
__global__ void __launch_bounds__(256) k_hgt_gate(HgtGateArgs a) {
  pdl_enter();
  __shared__ float s_red[8];
  const int T = min(a.cum[a.n_hops], a.cap);
  const int nvec = a.d >> 3;
  const float sg = sigmoid_f(*a.skip);
  const bool bwd = a.dZ32 != nullptr || a.dZ16 != nullptr;
  const int end = bwd ? min(a.cap, (T + 127) / 128 * 128) : T;
  const int64_t n = static_cast<int64_t>(end) * nvec;
  float red = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    if (i / nvec >= T) { reinterpret_cast<uint4*>(a.out)[i] = make_uint4(0, 0, 0, 0); continue; }
    float x[8] = {0, 0, 0, 0, 0, 0, 0, 0}, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    bf16x8_accum(reinterpret_cast<const uint4*>(a.A)[i], y);
    bf16x8_accum(reinterpret_cast<const uint4*>(a.X)[i], x);
    float o[8];
    if (!bwd) {
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = sg * y[e] + (1.f - sg) * x[e];
    } else {
      float g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (a.dZ32) {
        const float4 u = reinterpret_cast<const float4*>(a.dZ32)[2 * i], w = reinterpret_cast<const float4*>(a.dZ32)[2 * i + 1];
        g[0] = u.x; g[1] = u.y; g[2] = u.z; g[3] = u.w; g[4] = w.x; g[5] = w.y; g[6] = w.z; g[7] = w.w;
      } else {
        bf16x8_accum(reinterpret_cast<const uint4*>(a.dZ16)[i], g);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) { o[e] = sg * g[e]; red = fmaf(g[e], y[e] - x[e], red); }
      if (a.dX) {
        float4* dx = reinterpret_cast<float4*>(a.dX) + 2 * i;
        float4 u = dx[0], w = dx[1];
        const float c = 1.f - sg;
        u.x += c * g[0]; u.y += c * g[1]; u.z += c * g[2]; u.w += c * g[3];
        w.x += c * g[4]; w.y += c * g[5]; w.z += c * g[6]; w.w += c * g[7];
        dx[0] = u; dx[1] = w;
      }
    }
    reinterpret_cast<uint4*>(a.out)[i] = pack_bf16x8(o, 1.f);
  }
  if (!bwd || a.skip_g == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) red += __shfl_xor_sync(0xffffffffu, red, o);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = red;
  __syncthreads();
  if (threadIdx.x == 0) {
    float v = 0.f;
    for (int w = 0; w < (blockDim.x >> 5); ++w) v += s_red[w];
    if (v != 0.f) atomicAdd(a.skip_g, v * sg * (1.f - sg));
  }
}

// Block-diagonal relation images of one (layer, destination type) from the bf16 [n_rel, heads, D, D] parameters:
//   att_img [n_rel * H, H]:  (r H + h D + d, h D + f) = W_att[r, h, d, f]     (qq_r = Q att_img_r^T)
//   msg_img [H, n_rel * H]:  (h D + f, r H + h D + d) = W_msg[r, h, d, f]     (agg = U msg_img^T)
// Off-block entries are written as zeros.  grad mode (att_g != nullptr): the inverse map from the dense fp32 weight
// gradients of the two GEMMs into the parameter gradients (accumulated); the dense buffers are re-zeroed.
__global__ void __launch_bounds__(256) k_hgt_blocks(HgtBlockArgs a) {
  pdl_enter();
  const int H = a.heads * a.D, D = a.D;
  const int64_t n = static_cast<int64_t>(a.n_rel) * H * H;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    {  // att image element i
      const int64_t row = i / H;
      const int col = static_cast<int>(i % H);
      const int r = static_cast<int>(row / H), hr = static_cast<int>(row % H) / D, d = static_cast<int>(row % H) % D;
      const int hc = col / D, f = col % D;
      const int64_t src = ((static_cast<int64_t>(r) * a.heads + hr) * D + d) * D + f;
      if (a.att_g) {
        if (hr == hc) a.att_g[src] += a.att_dense[i];
        a.att_dense[i] = 0.f;
      } else {
        reinterpret_cast<__nv_bfloat16*>(a.att_img)[i] =
            hr == hc ? reinterpret_cast<const __nv_bfloat16*>(a.att)[src] : __float2bfloat16(0.f);
      }
    }
    {  // msg image element i
      const int64_t RH = static_cast<int64_t>(a.n_rel) * H;
      const int row = static_cast<int>(i / RH);
      const int64_t col = i % RH;
      const int h = row / D, f = row % D;
      const int r = static_cast<int>(col / H), hc = static_cast<int>(col % H) / D, d = static_cast<int>(col % H) % D;
      const int64_t src = ((static_cast<int64_t>(r) * a.heads + h) * D + d) * D + f;
      if (a.att_g) {
        if (h == hc) a.msg_g[src] += a.msg_dense[i];
        a.msg_dense[i] = 0.f;
      } else {
        reinterpret_cast<__nv_bfloat16*>(a.msg_img)[i] =
            h == hc ? reinterpret_cast<const __nv_bfloat16*>(a.msg)[src] : __float2bfloat16(0.f);
      }
    }
  }
}

// bf16 gradient rows [dK | dQ | dV] of a type's K/Q/V projection (the A operand of its weight- and data-gradient GEMMs)
// from the fp32 attention gradients dKV = [dK | dV] (rows < n, re-zeroed after reading) and the bf16 dQ (rows < nq,
// nq = min(cum[idx_q], n, rows of dQ)); rows [n, round_up(n, 128)) are zeros.  bias_g [3H] += the column sums of the
// bf16 rows, one atomic per column per CTA.
// Threads: a chunk of up to 128 vectors (blockIdx.y) times 256 / chunk rows.
__global__ void __launch_bounds__(256) k_hgt_kqv_cast(HgtKqvCastArgs a) {
  pdl_enter();
  __shared__ float s_acc[256][8];
  const int nv = a.H >> 3, nvec = 3 * nv;
  const int n = min(a.cum[a.idx], a.cap);
  const int nq = a.dq ? min(min(a.cum[a.idx_q], n), a.cap_q) : 0;
  const int cw = min(nvec, 128);
  const int c0 = blockIdx.y * 128;
  const int cg = threadIdx.x % cw, rl = threadIdx.x / cw;
  const int rpb = 256 / cw;
  const int c = c0 + cg;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (rl < rpb && c < nvec) {
    const int seg = c / nv, cc = c - seg * nv;
    const int end = min(a.cap, (n + 127) / 128 * 128);
    for (int r = blockIdx.x * rpb + rl; r < end; r += gridDim.x * rpb) {
      float o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (r < n) {
        if (seg == 1) {
          if (r < nq) bf16x8_accum(reinterpret_cast<const uint4*>(a.dq)[static_cast<int64_t>(r) * nv + cc], o);
        } else {
          float* p = a.dkv + static_cast<int64_t>(r) * 2 * a.H + (seg == 0 ? 0 : a.H) + cc * 8;
          const float4 u = reinterpret_cast<const float4*>(p)[0], w = reinterpret_cast<const float4*>(p)[1];
          o[0] = u.x; o[1] = u.y; o[2] = u.z; o[3] = u.w; o[4] = w.x; o[5] = w.y; o[6] = w.z; o[7] = w.w;
          reinterpret_cast<float4*>(p)[0] = make_float4(0.f, 0.f, 0.f, 0.f);
          reinterpret_cast<float4*>(p)[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      const uint4 b = pack_bf16x8(o, 1.f);
      reinterpret_cast<uint4*>(a.out)[static_cast<int64_t>(r) * nvec + c] = b;
      if (r < n) bf16x8_accum(b, acc);            // sum exactly what the GEMMs see (bf16-rounded)
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) s_acc[threadIdx.x][q] = acc[q];
  __syncthreads();
  if (a.bias_g == nullptr) return;
  for (int x = threadIdx.x; x < cw * 8; x += blockDim.x) {
    const int col = (c0 + (x >> 3)) * 8 + (x & 7);
    if (c0 + (x >> 3) >= nvec) continue;
    float v = 0.f;
    for (int t = x >> 3; t < rpb * cw; t += cw) v += s_acc[t][x & 7];
    if (v != 0.f) atomicAdd(a.bias_g + col, v);
  }
}

}  // namespace

// lane-group shape from the row width H (a multiple of 64 in [64, 1024]: 8 .. 128 vectors)
void launch_hgt_attention(const HgtAttnArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_hgt_attention<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

void launch_hgt_attention_bwd(const HgtAttnBwdArgs& a, cudaStream_t s) {
  dispatch_lanes<8, 4>(a.H / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_hgt_attention_bwd<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

void launch_hgt_gelu(const void* X, void* Y, const int32_t* cum, int n_hops, int cap, int d, const void* dY,
                     cudaStream_t s) {
  launch_k(k_hgt_gelu, dim3(grid_for(static_cast<int64_t>(cap) * (d / 8), 256, 132 * 8)), dim3(256), 0, s,
           reinterpret_cast<const __nv_bfloat16*>(X), reinterpret_cast<__nv_bfloat16*>(Y), cum, n_hops, cap, d,
           reinterpret_cast<const __nv_bfloat16*>(dY));
}

void launch_hgt_gate(const HgtGateArgs& a, cudaStream_t s) {
  launch_k(k_hgt_gate, dim3(grid_for(static_cast<int64_t>(a.cap) * (a.d / 8), 256, 132 * 8)), dim3(256), 0, s, a);
}

void launch_hgt_blocks(const HgtBlockArgs& a, cudaStream_t s) {
  const int64_t H = static_cast<int64_t>(a.heads) * a.D;
  launch_k(k_hgt_blocks, dim3(grid_for(a.n_rel * H * H, 256, 132 * 8)), dim3(256), 0, s, a);
}

void launch_hgt_kqv_cast(const HgtKqvCastArgs& a, cudaStream_t s) {
  const int nvec = 3 * (a.H / 8);
  const int cw = nvec < 128 ? nvec : 128;
  const int rpb = 256 / cw;
  launch_k(k_hgt_kqv_cast, dim3(grid_for(a.cap, rpb * 4, 132 * 4), (nvec + 127) / 128), dim3(256), 0, s, a);
}

}  // namespace glt
