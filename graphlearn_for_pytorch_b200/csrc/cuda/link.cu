// Link-prediction kernels of GraphSageLinkEngine (models/sage_link.py): binary negatives drawn inside the captured
// step, and the fused edge loss (dot-product logits, BCE forward + backward) over the last layer's embeddings.
// Like every engine kernel they read batch extents from device memory and never sync with the host.
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// Philox stream of the negative draws.  The homogeneous sampler arena draws hop h of a batch from stream
// h + 8 * step with h < 4, so an id that is 7 mod 8 is never used by a neighbour draw.
constexpr uint32_t kLinkNegStream = 0x4C4E4B07u;
// strict negatives with padding: up to this many draws are rejected while they hit an edge, then the last is kept
// (RandomNegativeSampler.sample(trials_num=5, padding=True))
constexpr int kLinkNegTrials = 5;

// seeds[p] / seeds[P + p] = source / destination of pair p, P = (1 + k) * B.  Pairs [0, B) are the positives as
// given; pair B + i * k + j is the j-th negative of positive i, a uniform (r, c) over [0, N)^2 redrawn while (r, c)
// is an edge.  Each negative is a pure function of (seed, step, p): one thread per output slot, no compaction.
__global__ void __launch_bounds__(256) k_link_seeds(GraphTable g, const int64_t* pos, int B, int k, int64_t num_nodes,
                                                    uint64_t seed, const int32_t* step_dev, int64_t* seeds,
                                                    int32_t* n_pairs) {
  pdl_enter();
  const int P = (1 + k) * B;
  const uint64_t step = static_cast<uint32_t>(*step_dev);
  const uint32_t n = static_cast<uint32_t>(num_nodes);
  if (blockIdx.x == 0) {
    // number of valid pairs, counted exactly by one CTA: no pre-zeroed counter in the launch chain
    int valid = 0;
    for (int base = 0; base < B; base += blockDim.x) {
      const int i = base + threadIdx.x;
      valid += __syncthreads_count(i < B && pos[i] >= 0 && pos[B + i] >= 0);
    }
    if (threadIdx.x == 0) *n_pairs = (1 + k) * valid;
  }
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < P; p += gridDim.x * blockDim.x) {
    int64_t r, c;
    if (p < B) {
      r = pos[p];
      c = pos[B + p];
    } else {
      const int i = (p - B) / k;
      r = c = -1;                                   // a padded positive pads its negatives too
      if (pos[i] >= 0 && pos[B + i] >= 0) {
        const uint64_t row = (step << 32) | static_cast<uint32_t>(p);
        for (int t = 0; t < kLinkNegTrials; ++t) {
          r = bounded(philox_draw(seed, kLinkNegStream, row, 2 * t), n);
          c = bounded(philox_draw(seed, kLinkNegStream, row, 2 * t + 1), n);
          if (!edge_exists(g, r, c)) break;
        }
      }
    }
    seeds[p] = r;
    seeds[P + p] = c;
  }
}

// LPR lanes per pair, VPL 8-column vectors per lane.  For pair p < P with local ids ls = seed_local[p],
// ld = seed_local[P + p] (skipped when either is negative): s = <Z[ls, :C], Z[ld, :C]> in fp32, y = (p < B),
//   loss    += softplus((1 - 2y) s) / n_pairs          (= binary_cross_entropy_with_logits, mean over valid pairs)
//   correct += ((s > 0) == y)
//   dZ[ls]  += g Z[ld],  dZ[ld] += g Z[ls]  with g = (sigmoid(s) - y) / n_pairs   (fp32 red.add; dZ may be null)
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_link_bce(const __nv_bfloat16* Z, int ld, int C, const int32_t* seed_local,
                                                  int P, int B, const int32_t* n_pairs, float* loss,
                                                  int32_t* correct, float* dZ) {
  pdl_enter();
  constexpr int RPW = 32 / LPR;                     // pairs per warp and iteration
  const int lane = threadIdx.x & 31, gl = lane % LPR, gw = lane / LPR;
  const int wpb = blockDim.x >> 5;
  const int np = *n_pairs;
  const float invn = np > 0 ? 1.f / static_cast<float>(np) : 0.f;
  const int nvec = C >> 3;
  float l_acc = 0.f;
  int c_acc = 0;
  for (int base = (blockIdx.x * wpb + (threadIdx.x >> 5)) * RPW; base < P; base += gridDim.x * wpb * RPW) {
    const int p = base + gw;
    const int ls = p < P ? seed_local[p] : -1;
    const int lt = p < P ? seed_local[P + p] : -1;
    const bool ok = ls >= 0 && lt >= 0;
    float zs[VPL][8], zt[VPL][8];
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
#pragma unroll
      for (int q = 0; q < 8; ++q) zs[v][q] = zt[v][q] = 0.f;
      const int c = gl + v * LPR;
      if (ok && c < nvec) {
        bf16x8_accum(*reinterpret_cast<const uint4*>(Z + static_cast<int64_t>(ls) * ld + c * 8), zs[v]);
        bf16x8_accum(*reinterpret_cast<const uint4*>(Z + static_cast<int64_t>(lt) * ld + c * 8), zt[v]);
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) s = fmaf(zs[v][q], zt[v][q], s);
    }
#pragma unroll
    for (int off = LPR / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
    if (ok) {
      const bool pos = p < B;
      const float x = pos ? -s : s;
      const float sp = fmaxf(x, 0.f) + log1pf(expf(-fabsf(x)));
      const float e = expf(-fabsf(s));
      const float sig = s >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
      const float g = (sig - (pos ? 1.f : 0.f)) * invn;
      if (gl == 0) {
        l_acc += sp * invn;
        c_acc += ((s > 0.f) == pos) ? 1 : 0;
      }
      if (dZ) {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const int c = gl + v * LPR;
          if (c >= nvec) continue;
          float4* ds = reinterpret_cast<float4*>(dZ + static_cast<int64_t>(ls) * ld + c * 8);
          float4* dt = reinterpret_cast<float4*>(dZ + static_cast<int64_t>(lt) * ld + c * 8);
          atomicAdd(ds, make_float4(g * zt[v][0], g * zt[v][1], g * zt[v][2], g * zt[v][3]));
          atomicAdd(ds + 1, make_float4(g * zt[v][4], g * zt[v][5], g * zt[v][6], g * zt[v][7]));
          atomicAdd(dt, make_float4(g * zs[v][0], g * zs[v][1], g * zs[v][2], g * zs[v][3]));
          atomicAdd(dt + 1, make_float4(g * zs[v][4], g * zs[v][5], g * zs[v][6], g * zs[v][7]));
        }
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    l_acc += __shfl_xor_sync(0xffffffffu, l_acc, off);
    c_acc += __shfl_xor_sync(0xffffffffu, c_acc, off);
  }
  if (lane == 0) {
    if (l_acc != 0.f) atomicAdd(loss, l_acc);
    if (correct && c_acc != 0) atomicAdd(correct, c_acc);
  }
}

}  // namespace

void launch_link_seeds(GraphTable g, const int64_t* pos, int B, int k, int64_t num_nodes, uint64_t seed,
                       const int32_t* step_dev, int64_t* seeds, int32_t* n_pairs, cudaStream_t s) {
  launch_k(k_link_seeds, dim3(grid_for(static_cast<int64_t>(1 + k) * B, 256)), dim3(256), 0, s, g, pos, B, k,
           num_nodes, seed, step_dev, seeds, n_pairs);
}

void launch_link_bce(const void* Z, int ld, int C, const int32_t* seed_local, int P, int B, const int32_t* n_pairs,
                     float* loss, int32_t* correct, float* dZ, cudaStream_t s) {
  const __nv_bfloat16* z = reinterpret_cast<const __nv_bfloat16*>(Z);
  dispatch_lanes<4, 2>(C / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_link_bce<LPR, VPL>, dim3(grid_for(P, 8 * (32 / LPR))), dim3(256), 0, s, z, ld, C, seed_local, P, B,
             n_pairs, loss, correct, dZ);
  });
}

}  // namespace glt
