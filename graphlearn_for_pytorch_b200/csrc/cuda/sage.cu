// GraphSAGE engine kernels (SIMT side): neighbour-mean aggregation straight from
// the sampler's per-hop ELL blocks, its scatter backward, fused loss and Adam.
// Everything reads its extents from device counters (BatchCounters::cum) and is
// launched with worst-case grids, so one training step is a fixed launch
// sequence that is captured into a CUDA graph -- no host sync anywhere.
//
// The reference has no model code (PyG SAGEConv in examples/train_sage_ogbn_products.py:30-59
// does gather -> scatter-mean -> two Linear); the aggregation here consumes the
// feature table *in place* (local or peer HBM) like GatherTensorKernel
// (csrc/cuda/unified_tensor.cu:47-81) but never materialises x[n_id].

#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// LPR lanes cooperate on one target row; each lane owns VPL 16-byte vectors: 8 bf16 elements, or (FP8: the feature
// table holds MXFP8 rows) 16 e4m3 elements that are de-quantised as they are accumulated.  Either way the mean is
// summed in fp32 in ELL slot order, rounded once and written as bf16; the FP8 self block is bf16(de-quantised row).
template <int LPR, int VPL, bool FP8 = false>
__global__ void __launch_bounds__(256) k_sage_aggregate(SageAggArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const unsigned gmask = (LPR == 32) ? 0xffffffffu : (((1u << LPR) - 1u) << (gw * LPR));
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  constexpr int EPV = FP8 ? 16 : 8;
  const int nvec = a.d / EPV;
  for (int base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    const bool valid = t < T;
    float acc[VPL][EPV];
#pragma unroll
    for (int v = 0; v < VPL; ++v)
#pragma unroll
      for (int i = 0; i < EPV; ++i) acc[v][i] = 0.f;
    int dg = 0, k = 0;
    const int32_t* ell = nullptr;
    if (valid) {
      const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
      dg = a.deg[t];
      k = a.k[l.hop];
      ell = a.ell[l.hop] + static_cast<int64_t>(l.row) * k;
    }
    for (int j0 = 0; j0 < dg; j0 += LPR) {
      const uint8_t* my_ptr = nullptr;
      if (j0 + gl < dg) {
        const int s = ell[j0 + gl];
        if (s >= 0) my_ptr = src_row(a, s);
      }
      const int cnt = min(LPR, dg - j0);
      for (int jj = 0; jj < cnt; ++jj) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(
            __shfl_sync(gmask, reinterpret_cast<unsigned long long>(my_ptr), jj, LPR));
        if (p == nullptr) continue;
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = v * LPR + gl;
          if (c < nvec) {
            if (FP8) mxfp8x16_accum_at(p, a.d, c, acc[v]);
            else bf16x8_accum(ld_nc_v4(p + c * 16), acc[v]);
          }
        }
      }
    }
    if (!valid) continue;
    const float inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
    const int ld = a.out_ld ? a.out_ld : 2 * a.d;
    const int mcol = a.out_ld ? a.mean_col : 0;
    const int scol = a.out_ld ? a.self_col : a.d;
    uint8_t* o = reinterpret_cast<uint8_t*>(a.out) + static_cast<int64_t>(t) * ld * 2;
    const uint8_t* self = scol >= 0 ? src_row(a, t) : nullptr;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      if (FP8) {
        uint4* om = reinterpret_cast<uint4*>(o + mcol * 2) + 2 * c;
        om[0] = pack_bf16x8(acc[v], inv);
        om[1] = pack_bf16x8(acc[v] + 8, inv);
      } else {
        reinterpret_cast<uint4*>(o + mcol * 2)[c] = pack_bf16x8(acc[v], inv);
        if (scol >= 0)
          reinterpret_cast<uint4*>(o + scol * 2)[c] = self ? ld_nc_v4(self + c * 16) : make_uint4(0, 0, 0, 0);
      }
    }
    if (FP8 && scol >= 0) {   // after the means, so that the accumulators are dead
      for (int c = gl; c < nvec; c += LPR) {
        float x[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) x[i] = 0.f;
        if (self) mxfp8x16_accum_at(self, a.d, c, x);
        uint4* os = reinterpret_cast<uint4*>(o + scol * 2) + 2 * c;
        os[0] = pack_bf16x8(x, 1.f);
        os[1] = pack_bf16x8(x + 8, 1.f);
      }
    }
  }
}

// 8 blocks per SM: every width variant stays at <= 32 registers, i.e. 64 resident warps to cover the atomics' latency
template <int LPR, int VPL>
__global__ void __launch_bounds__(256, 8) k_sage_scatter_bwd(SageScatterArgs a) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int gl = lane % LPR;
  const int gw = lane / LPR;
  const int T = min(a.cum[a.n_hops_targets], a.cap_targets);
  const int wpb = blockDim.x >> 5;
  const int nvec = a.d >> 3;
  for (int base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * RPW; base < T; base += gridDim.x * wpb * RPW) {
    const int t = base + gw;
    if (t >= T) continue;
    const HopLoc l = locate_hop(a.cum, a.n_hops_targets, t);
    const int dg = a.deg[t];
    const int k = a.k[l.hop];
    const int32_t* ell = a.ell[l.hop] + static_cast<int64_t>(l.row) * k;
    const uint8_t* g = reinterpret_cast<const uint8_t*>(a.dA) + static_cast<int64_t>(t) * a.dA_ld * 2;
    const float inv = dg > 0 ? 1.f / static_cast<float>(dg) : 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = v * LPR + gl;
      if (c >= nvec) continue;
      float gn[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) gn[i] = 0.f;
      bf16x8_accum(reinterpret_cast<const uint4*>(g + a.mean_col * 2)[c], gn);
#pragma unroll
      for (int i = 0; i < 8; ++i) gn[i] *= inv;
      for (int j = 0; j < dg; ++j) {
        const int s = ell[j];
        if (s >= 0) red_add8(a.dH + static_cast<int64_t>(s) * a.d + c * 8, gn);
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_relu_bwd_cast(const float* dH, const __nv_bfloat16* Z, const int32_t* cum,
                                                       int n_hops, int cap, int d, __nv_bfloat16* dPre,
                                                       float* colsum, float gscale, int relu) {
  pdl_enter();
  // gscale: 1/(1-p) when Z is the post-dropout activation (dropped elements are 0 there, so the ReLU test also
  // masks them).  colsum != nullptr: also accumulate the bias gradient (column sums of dPre).  Requires
  // d | 2048 so that a thread keeps the same 8 columns across grid-stride iterations.  relu == 0: no mask, Z is
  // not read (a layer without activation).
  __shared__ float s_acc[256][8];
  const int T = min(cum[n_hops], cap);
  const int64_t n8 = static_cast<int64_t>(cap) * d / 8;
  float acc[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) acc[q] = 0.f;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t e = i * 8;
    const int row = static_cast<int>(e / d);
    uint4 o = make_uint4(0, 0, 0, 0);
    if (row < T) {
      const float4 g0 = reinterpret_cast<const float4*>(dH + e)[0];
      const float4 g1 = reinterpret_cast<const float4*>(dH + e)[1];
      float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      float z[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) z[q] = 1.f;
      if (relu) {
#pragma unroll
        for (int q = 0; q < 8; ++q) z[q] = 0.f;
        bf16x8_accum(*reinterpret_cast<const uint4*>(Z + e), z);
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) g[q] = z[q] > 0.f ? g[q] * gscale : 0.f;
      o = pack_bf16x8(g, 1.f);
      if (colsum) {
        float r[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) r[q] = 0.f;
        bf16x8_accum(o, r);  // sum exactly what the GEMMs will see (bf16-rounded)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] += r[q];
      }
    }
    *reinterpret_cast<uint4*>(dPre + e) = o;
  }
  if (colsum == nullptr) return;
#pragma unroll
  for (int q = 0; q < 8; ++q) s_acc[threadIdx.x][q] = acc[q];
  __syncthreads();
  const int groups = d >> 3;                 // threads t, t + groups, ... share a column group
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float v = 0.f;
    for (int t = c >> 3; t < static_cast<int>(blockDim.x); t += groups) v += s_acc[t][c & 7];
    if (v != 0.f) atomicAdd(colsum + c, v);
  }
}

// warp per seed row: log-softmax + NLL forward and backward in one pass.
__global__ void k_softmax_nll(const __nv_bfloat16* logits, int ld, int C, const int64_t* y,
                              const int64_t* labels_all, const int64_t* nodes,
                              const int32_t* cum, int cap, float* loss, __nv_bfloat16* dlogits,
                              int32_t* correct, float* colsum) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  float csum[8];  // bias gradient: columns lane, lane+32, ... (ld <= 256)
#pragma unroll
  for (int q = 0; q < 8; ++q) csum[q] = 0.f;
  const int wpb = blockDim.x >> 5;
  const int n0 = min(cum[1], cap);
  const float invn = n0 > 0 ? 1.f / static_cast<float>(n0) : 0.f;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < cap; r += gridDim.x * wpb) {
    __nv_bfloat16* dl = dlogits + static_cast<int64_t>(r) * ld;
    if (r >= n0) {
      for (int c = lane; c < ld; c += 32) dl[c] = __float2bfloat16(0.f);
      continue;
    }
    const __nv_bfloat16* x = logits + static_cast<int64_t>(r) * ld;
    float mx = -3.4e38f;
    int arg = 0;
    for (int c = lane; c < C; c += 32) {
      const float v = __bfloat162float(x[c]);
      if (v > mx) { mx = v; arg = c; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, off);
      const int oa = __shfl_xor_sync(0xffffffffu, arg, off);
      if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
    }
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += __expf(__bfloat162float(x[c]) - mx);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float lse = mx + __logf(sum);
    // labels are looked up through the batch's node list: no separate gather launch
    const int64_t label = labels_all ? labels_all[nodes[r]] : y[r];
    for (int c = lane; c < ld; c += 32) {
      float g = 0.f;
      if (c < C) {
        const float p = __expf(__bfloat162float(x[c]) - lse);
        g = (p - (c == label ? 1.f : 0.f)) * invn;
      }
      const __nv_bfloat16 gb = __float2bfloat16(g);
      dl[c] = gb;
      if (colsum) csum[(c >> 5) & 7] += __bfloat162float(gb);
    }
    if (lane == 0) {
      const float xl = (label >= 0 && label < C) ? __bfloat162float(x[label]) : lse;
      atomicAdd(loss, (lse - xl) * invn);
      if (correct && arg == label) atomicAdd(correct, 1);
    }
  }
  if (colsum) {
    for (int c = lane, q = 0; c < ld && q < 8; c += 32, ++q)
      if (csum[q] != 0.f) atomicAdd(colsum + c, csum[q]);
  }
}

// step_dev[0] = number of optimizer steps taken so far, step_dev[1] = block ticket.  The kernel
// uses t = step + 1 and the LAST block to finish publishes it (every block has read the old
// value by then), which saves the separate `step += 1` launch.
__global__ void k_adam(float* p, const float* g, float* m, float* v, __nv_bfloat16* pb, int64_t n,
                       float lr, float b1, float b2, float eps, float wd, int32_t* step_dev,
                       float gscale) {
  pdl_enter();
  const int t = *reinterpret_cast<volatile int32_t*>(step_dev) + 1;
  // bias corrections in double, as k_sparse_adam: 1 - b2^t cancels most of b2^t's bits at small t, which left the
  // error of __powf's approximate log2 in the update at dozens of times its fp32 rounding error
  const float c1 = static_cast<float>(1.0 - pow(static_cast<double>(b1), t));
  const float c2 = static_cast<float>(1.0 - pow(static_cast<double>(b2), t));
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float gi = g[i] * gscale + wd * p[i];
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi; v[i] = vi;
    const float upd = (mi / c1) / (sqrtf(vi / c2) + eps);
    const float pi = p[i] - lr * upd;
    p[i] = pi;
    if (pb) pb[i] = __float2bfloat16(pi);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(step_dev + 1, 1) == static_cast<int>(gridDim.x) - 1) {
      step_dev[1] = 0;
      step_dev[0] += 1;
    }
  }
}

// column sums of the valid rows of a bf16 [rows, d] matrix (bias gradients), accumulated into `out` with atomics;
// replaces a cap-sized torch reduce kernel that was the most expensive launch of the step.  Any d (multiple of 8):
// rows wider than blockDim.x 8-column groups are summed one row per block iteration.
__global__ void __launch_bounds__(256) k_colsum(const __nv_bfloat16* X, const int32_t* cum, int n_hops,
                                                int cap, int d, float* out) {
  pdl_enter();
  extern __shared__ float s_part[];  // [rows_per_block][d]
  const int T = min(cum[n_hops], cap);
  const int groups = d >> 3;               // 8-column groups per row
  if (groups > static_cast<int>(blockDim.x)) {
    for (int cg = threadIdx.x; cg < groups; cg += blockDim.x) {
      float acc[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = 0.f;
      for (int r = blockIdx.x; r < T; r += gridDim.x)
        bf16x8_accum(*reinterpret_cast<const uint4*>(X + static_cast<int64_t>(r) * d + cg * 8), acc);
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (acc[i] != 0.f) atomicAdd(out + cg * 8 + i, acc[i]);
    }
    return;
  }
  const int rpb = blockDim.x / groups;     // rows handled per block iteration
  const int cg = threadIdx.x % groups, rl = threadIdx.x / groups;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  if (rl < rpb) {
    for (int r = blockIdx.x * rpb + rl; r < T; r += gridDim.x * rpb)
      bf16x8_accum(*reinterpret_cast<const uint4*>(X + static_cast<int64_t>(r) * d + cg * 8), acc);
#pragma unroll
    for (int i = 0; i < 8; ++i) s_part[rl * d + cg * 8 + i] = acc[i];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    float v = 0.f;
    for (int q = 0; q < rpb; ++q) v += s_part[q * d + c];
    if (v != 0.f) atomicAdd(out + c, v);
  }
}

__global__ void k_add_block_f32(const __nv_bfloat16* dA, int dA_ld, int col, int d, const int32_t* cum, int n_hops,
                                int cap, float* dH) {
  pdl_enter();
  const int T = min(cum[n_hops], cap);
  const int nvec = d >> 3;
  const int64_t n = static_cast<int64_t>(T) * nvec;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i / nvec), c = static_cast<int>(i % nvec);
    float g[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) g[q] = 0.f;
    bf16x8_accum(*reinterpret_cast<const uint4*>(dA + static_cast<int64_t>(t) * dA_ld + col + c * 8), g);
    float4* o = reinterpret_cast<float4*>(dH + static_cast<int64_t>(t) * d + c * 8);
    float4 a0 = o[0], a1 = o[1];
    a0.x += g[0]; a0.y += g[1]; a0.z += g[2]; a0.w += g[3];
    a1.x += g[4]; a1.y += g[5]; a1.z += g[6]; a1.w += g[7];
    o[0] = a0; o[1] = a1;
  }
}

// start of the gradient phase of a step: flat gradient buffer, loss and #correct back to zero in one launch
__global__ void k_zero_grads(float* g, int64_t n, float* loss, int32_t* correct) {
  pdl_enter();
  const int64_t n4 = n >> 2;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  if (blockIdx.x == 0) {
    for (int64_t i = (n4 << 2) + threadIdx.x; i < n; i += blockDim.x) g[i] = 0.f;
    if (threadIdx.x == 0) {
      if (loss) *loss = 0.f;
      if (correct) *correct = 0;
    }
  }
}

__global__ void k_zero_rows(float* p, const int32_t* cum, int n_hops, int cap, int d) {
  pdl_enter();
  const int T = min(cum[n_hops], cap);
  const int64_t n4 = static_cast<int64_t>(T) * d / 4;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    reinterpret_cast<float4*>(p)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

}  // namespace

int& pdl_flag() {
  static int flag = 1;
  return flag;
}

int set_pdl(int on) {
  const int old = pdl_flag();
  pdl_flag() = on ? 1 : 0;
  return old;
}

void launch_sage_aggregate(const SageAggArgs& a, cudaStream_t s) {
  if (a.feat_fp8) {
    // MXFP8 layer-1 source: d / 16 vectors of 16 elements; <32, 2> holds a 1024-wide row in 32 accumulators per lane
    dispatch_lanes<2, 2>(a.d / 16, [&](auto lpr, auto vpl) {
      constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
      launch_k(k_sage_aggregate<LPR, VPL, true>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
    });
    return;
  }
  // (a variant keeping 4 neighbour rows in flight per lane group before accumulating made the step slower and was
  // removed: the rows are L2-resident activations)
  dispatch_lanes<4, 4>(a.d / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_sage_aggregate<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

void launch_sage_scatter_bwd(const SageScatterArgs& a, cudaStream_t s) {
  dispatch_lanes<4, 4>(a.d / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_sage_scatter_bwd<LPR, VPL>, dim3(grid_for(a.cap_targets, 8 * (32 / LPR))), dim3(256), 0, s, a);
  });
}

// In-place inverted dropout on the first cum[n_hops] rows of a bf16 activation.  The keep mask is a pure function
// of (seed, layer, optimizer step, element), so a replayed step drops the same elements; the step is read from the
// device-side Adam counter, which makes the kernel CUDA-graph friendly.
__global__ void __launch_bounds__(256) k_dropout_bf16(__nv_bfloat16* Z, const int32_t* cum, int n_hops, int cap, int d,
                                                      uint32_t thresh16, float scale, uint64_t seed, int layer,
                                                      const int32_t* step_dev) {
  pdl_enter();
  const int T = min(cum[n_hops], cap);
  const int64_t n8 = static_cast<int64_t>(T) * d / 8;
  const uint32_t step = step_dev ? static_cast<uint32_t>(*step_dev) : 0u;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n8;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const U4 r = dropout_bits(seed, layer, step, i);
    const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
    uint4 v = *reinterpret_cast<const uint4*>(Z + i * 8);
    float z[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) z[q] = 0.f;
    bf16x8_accum(v, z);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint32_t u = (rr[q >> 1] >> ((q & 1) * 16)) & 0xFFFFu;
      z[q] = u >= thresh16 ? z[q] : 0.f;
    }
    *reinterpret_cast<uint4*>(Z + i * 8) = pack_bf16x8(z, scale);
  }
}

void launch_dropout_bf16(void* Z, const int32_t* cum, int n_hops, int cap, int d, float p, uint64_t seed, int layer,
                         const int32_t* step_dev, cudaStream_t s) {
  const uint32_t thresh = static_cast<uint32_t>(fminf(fmaxf(p, 0.f), 1.f) * 65536.f);
  const float scale = p < 1.f ? 1.f / (1.f - p) : 0.f;
  launch_k(k_dropout_bf16, dim3(grid_for(static_cast<int64_t>(cap) * d / 8, 256, 132 * 8)), dim3(256), 0, s,
           reinterpret_cast<__nv_bfloat16*>(Z), cum, n_hops, cap, d, thresh, scale, seed, layer, step_dev);
}

// Accumulates the column sums of the first min(cum[n_hops], cap) rows of X into `out` (not zeroed here).
void launch_colsum_accum(const void* X, const int32_t* cum, int n_hops, int cap, int d, float* out,
                         cudaStream_t s) {
  const int groups = d / 8;
  const int rpb = 256 / groups > 0 ? 256 / groups : 1;
  const size_t smem = groups <= 256 ? sizeof(float) * rpb * d : 0;
  launch_k(k_colsum, dim3(grid_for(cap, rpb * 8, 132 * 2)), dim3(256), smem, s,
           reinterpret_cast<const __nv_bfloat16*>(X), cum, n_hops, cap, d, out);
}

void launch_relu_bwd_cast(const float* dH, const void* Z, const int32_t* cum, int n_hops, int cap,
                          int d, void* dPre, float* colsum, cudaStream_t s, bool prezeroed, float gscale, bool relu) {
  // the fused column sum needs d | 2048 (a thread keeps its 8 columns across grid-stride iterations); other widths
  // sum the bf16 dPre in a second pass
  const bool fused = colsum && 2048 % d == 0;
  if (colsum && !prezeroed) cudaMemsetAsync(colsum, 0, sizeof(float) * d, s);
  launch_k(k_relu_bwd_cast, dim3(grid_for(static_cast<int64_t>(cap) * d / 8, 256 * 2, 132 * 4)), dim3(256), 0, s,
           dH, reinterpret_cast<const __nv_bfloat16*>(Z), cum, n_hops, cap, d,
           reinterpret_cast<__nv_bfloat16*>(dPre), fused ? colsum : nullptr, gscale, relu ? 1 : 0);
  if (colsum && !fused) launch_colsum_accum(dPre, cum, n_hops, cap, d, colsum, s);
}

void launch_softmax_nll(const void* logits, int ld, int C, const int64_t* y, const int64_t* labels_all,
                        const int64_t* nodes, const int32_t* cum, int cap, float* loss, void* dlogits,
                        int32_t* correct, float* colsum, cudaStream_t s, bool prezeroed) {
  // the loss kernel sums the bias gradient in registers for ld <= 256; wider rows sum the bf16 dlogits in a second
  // pass over the n0 = cum[1] seed rows
  const bool fused = colsum && ld <= 256;
  if (!prezeroed) {   // memset nodes would break the programmatic-launch chain: the engine zeroes these in k_zero_grads
    if (colsum) cudaMemsetAsync(colsum, 0, sizeof(float) * ld, s);
    cudaMemsetAsync(loss, 0, sizeof(float), s);
    if (correct) cudaMemsetAsync(correct, 0, sizeof(int32_t), s);
  }
  launch_k(k_softmax_nll, dim3(grid_for(cap, 8)), dim3(256), 0, s, reinterpret_cast<const __nv_bfloat16*>(logits), ld,
           C, y, labels_all, nodes, cum, cap, loss, reinterpret_cast<__nv_bfloat16*>(dlogits), correct,
           fused ? colsum : nullptr);
  if (colsum && !fused) launch_colsum_accum(dlogits, cum, 1, cap, ld, colsum, s);
}

void launch_adam(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr,
                 float b1, float b2, float eps, float wd, int32_t* step_dev, float gscale,
                 cudaStream_t s) {
  launch_k(k_adam, dim3(grid_for(n, 256, 132 * 4)), dim3(256), 0, s, p, g, m, v,
           reinterpret_cast<__nv_bfloat16*>(p_bf16), n, lr, b1, b2, eps, wd, step_dev, gscale);
}

void launch_colsum_bf16(const void* X, const int32_t* cum, int n_hops, int cap, int d, float* out,
                        cudaStream_t s) {
  cudaMemsetAsync(out, 0, sizeof(float) * d, s);
  launch_colsum_accum(X, cum, n_hops, cap, d, out, s);
}

void launch_add_block_f32(const void* dA, int dA_ld, int col, int d, const int32_t* cum, int n_hops, int cap,
                          float* dH, cudaStream_t s) {
  launch_k(k_add_block_f32, dim3(grid_for(static_cast<int64_t>(cap) * d / 8, 256)), dim3(256), 0, s,
           reinterpret_cast<const __nv_bfloat16*>(dA), dA_ld, col, d, cum, n_hops, cap, dH);
}

void launch_zero_grads(float* g, int64_t n, float* loss, int32_t* correct, cudaStream_t s) {
  launch_k(k_zero_grads, dim3(grid_for(n / 4 + 1, 256, 132 * 2)), dim3(256), 0, s, g, n, loss, correct);
}

void launch_zero_rows(float* p, const int32_t* cum, int n_hops, int cap, int d, cudaStream_t s) {
  launch_k(k_zero_rows, dim3(grid_for(static_cast<int64_t>(cap) * d / 4, 256 * 4)), dim3(256), 0, s, p, cum, n_hops, cap, d);
}

}  // namespace glt
