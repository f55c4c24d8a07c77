// Multi-label loss of GraphSageMultiLabelEngine (models/sage_multilabel.py): mean sigmoid binary cross-entropy over
// T independent binary tasks per seed, forward and backward in one pass, the counterpart of k_softmax_nll (sage.cu).
// Like every engine kernel it reads the batch extent from the device counters and never syncs with the host.
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// Columns [c0, c0 + 32) of one seed row, one per lane; `word` holds their 32 label bits (the same word for the whole
// warp).  Accumulates the lane's loss terms and confusion counts and returns the bf16 gradient it wrote.
__device__ __forceinline__ float bce_cols(const __nv_bfloat16* x, __nv_bfloat16* dl, int c0, int lane, int T, int ld,
                                          uint32_t word, float inv, float& l, int& tp, int& fp, int& fn) {
  const int c = c0 + lane;
  float g = 0.f;
  if (c < T) {
    const float z = __bfloat162float(x[c]);
    const bool y = (word >> lane) & 1u;
    // max(z, 0) - y z + log1p(exp(-|z|)) and sigmoid(z) from the same exp(-|z|) <= 1: finite at any |z|
    const float e = expf(-fabsf(z));
    l += fmaxf(z, 0.f) - (y ? z : 0.f) + log1pf(e);
    const float sig = z >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
    g = (sig - (y ? 1.f : 0.f)) * inv;
    const bool pred = z > 0.f;
    tp += pred && y;
    fp += pred && !y;
    fn += !pred && y;
  }
  const __nv_bfloat16 gb = __float2bfloat16(g);
  if (c < ld) dl[c] = gb;
  return __bfloat162float(gb);
}

// Warp per seed row r < n0 = min(cum[1], cap), labels bits[nodes[r]] (uint32 [n_nodes, W], bit c & 31 of word c >> 5
// is task c; a node id outside [0, n_nodes) reads as all zeros):
//   loss    += sum_c (max(z, 0) - y z + log1p(exp(-|z|))) / (n0 T)
//   dlogits  = (sigmoid(z) - y) / (n0 T) in columns < T, 0 in columns [T, ld) and in rows [n0, cap)
//   counts  += (TP, FP, FN) with prediction z > 0
//   colsum  += column sums of the bf16 dlogits (ld <= 256: eight 32-column groups in registers; nullptr otherwise)
__global__ void __launch_bounds__(256) k_sigmoid_bce(const __nv_bfloat16* logits, int ld, int T, const uint32_t* bits,
                                                     int W, int64_t n_nodes, const int64_t* nodes, const int32_t* cum,
                                                     int cap, float* loss, __nv_bfloat16* dlogits, int32_t* counts,
                                                     float* colsum) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  float csum[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) csum[q] = 0.f;
  int tp = 0, fp = 0, fn = 0;
  const int wpb = blockDim.x >> 5;
  const int n0 = min(cum[1], cap);
  const float inv = n0 > 0 ? 1.f / static_cast<float>(static_cast<int64_t>(n0) * T) : 0.f;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < cap; r += gridDim.x * wpb) {
    __nv_bfloat16* dl = dlogits + static_cast<int64_t>(r) * ld;
    if (r >= n0) {
      for (int v = lane; v < ld / 8; v += 32) reinterpret_cast<uint4*>(dl)[v] = make_uint4(0, 0, 0, 0);
      continue;
    }
    const __nv_bfloat16* x = logits + static_cast<int64_t>(r) * ld;
    const int64_t node = nodes[r];
    const uint32_t* row_bits = (node >= 0 && node < n_nodes) ? bits + node * W : nullptr;
    float l = 0.f;
    if (colsum) {
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int c0 = q * 32;
        if (c0 >= ld) break;
        const uint32_t word = (row_bits && c0 < T) ? row_bits[c0 >> 5] : 0u;
        csum[q] += bce_cols(x, dl, c0, lane, T, ld, word, inv, l, tp, fp, fn);
      }
    } else {
      for (int c0 = 0; c0 < ld; c0 += 32) {
        const uint32_t word = (row_bits && c0 < T) ? row_bits[c0 >> 5] : 0u;
        bce_cols(x, dl, c0, lane, T, ld, word, inv, l, tp, fp, fn);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) l += __shfl_xor_sync(0xffffffffu, l, off);
    if (lane == 0 && l != 0.f) atomicAdd(loss, l * inv);
  }
  if (colsum) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int c = q * 32 + lane;
      if (c < ld && csum[q] != 0.f) atomicAdd(colsum + c, csum[q]);
    }
  }
  if (counts) {
    tp = __reduce_add_sync(0xffffffffu, tp);
    fp = __reduce_add_sync(0xffffffffu, fp);
    fn = __reduce_add_sync(0xffffffffu, fn);
    if (lane == 0) {
      if (tp) atomicAdd(counts, tp);
      if (fp) atomicAdd(counts + 1, fp);
      if (fn) atomicAdd(counts + 2, fn);
    }
  }
}

}  // namespace

void launch_sigmoid_bce(const void* logits, int ld, int T, const uint32_t* bits, int64_t n_nodes,
                        const int64_t* nodes, const int32_t* cum, int cap, float* loss, void* dlogits,
                        int32_t* counts, float* colsum, cudaStream_t s, bool prezeroed) {
  // as launch_softmax_nll: the bias gradient is summed in registers for ld <= 256, by a second pass over the n0 seed
  // rows of the bf16 dlogits otherwise
  const bool fused = colsum && ld <= 256;
  if (!prezeroed) {
    if (colsum) cudaMemsetAsync(colsum, 0, sizeof(float) * ld, s);
    cudaMemsetAsync(loss, 0, sizeof(float), s);
    if (counts) cudaMemsetAsync(counts, 0, 3 * sizeof(int32_t), s);
  }
  launch_k(k_sigmoid_bce, dim3(grid_for(cap, 8)), dim3(256), 0, s, reinterpret_cast<const __nv_bfloat16*>(logits), ld,
           T, bits, (T + 31) / 32, n_nodes, nodes, cum, cap, loss, reinterpret_cast<__nv_bfloat16*>(dlogits), counts,
           fused ? colsum : nullptr);
  if (colsum && !fused) launch_colsum_accum(dlogits, cum, 1, cap, ld, colsum, s);
}

}  // namespace glt
