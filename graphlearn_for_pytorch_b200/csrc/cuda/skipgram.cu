// Skip-gram kernels of MetaPath2VecEngine (models/metapath2vec.py): metapath random walks, SGNS negatives, the fused
// SGNS loss + gradient, and a sparse Adam over the rows the step looked up.  One training step is
//   k_m2v_begin       advance the device step counters (walk step, Adam step)
//   k_metapath_walk   thread per walk: uniform neighbour in relation metapath[(s - 1) % R]; counts valid windows
//     or k_node2vec_walk  warp per walk: node2vec's p / q second-order rule, 32 rejection-sampling proposals at a time
//   k_sgns_negatives  thread per (window, k): a negative window keeps the centre, draws each context position
//   k_sgns_loss_grad  lane group per window: its C - 1 positive pairs and K negative windows share the centre row
//   k_sparse_adam     warp per 32 rows: the rows flagged "touched" get torch.optim.SparseAdam's update
// and never reads anything back to the host, so the step is captured into one CUDA graph.
//
// Touched-row protocol: k_sgns_loss_grad stores touched[row] = 1 for every row it looks up (a plain byte store,
// idempotent) and red.adds its gradient into the fp32 grad row; k_sparse_adam scans the flags and updates only the
// flagged rows, then zeroes their gradient rows and flags, so the next step starts from zero without a memset of the
// tables.  Rows whose flag is clear are neither read nor written.
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// Philox streams of the walk and negative draws; the draw row is (step << 32) | item, so steps never collide.
constexpr uint32_t kWalkStream = 0x4D325657u;
constexpr uint32_t kNegStream = 0x4D32564Eu;
constexpr uint32_t kN2vStream = 0x4E325657u;   // node2vec proposals: the counter word is (walk step, proposal)
constexpr float kSgnsEps = 1e-15f;   // PyG MetaPath2Vec's EPS inside the logs

// Position p of a walk has the node type of slot(p): slot 0 is the source type of metapath[0], slot r + 1 the
// destination type of metapath[r] (equal to the source type of metapath[(r + 1) % R] on a chained path).
__device__ __forceinline__ int pos_slot(int p, int R) { return p == 0 ? 0 : (p - 1) % R + 1; }

__global__ void k_m2v_begin(int32_t* state) {
  // state = [next walk step, Adam step, walk step of this step]
  state[2] = state[0];
  state[0] += 1;
  state[1] += 1;
}

// Walk i starts at starts[i / W]; step s moves to a uniform neighbour in relation rel[(s - 1) % R], drawn as
// Philox(seed, kWalkStream, (step << 32) | i, s - 1).  An id outside [0, n of its position's type), a dead end or a
// padded start ends the walk: every later entry is -1.  n_valid += the walk's windows of C valid entries.
__global__ void __launch_bounds__(128) k_metapath_walk(const GraphTable* rel, int R, MetaPathTypes types,
                                                       const int64_t* starts, int n_walks, int W, int L, int C,
                                                       uint64_t seed, const int32_t* step_dev, int64_t* out,
                                                       int32_t* n_valid) {
  pdl_enter();
  const uint64_t step = static_cast<uint32_t>(*step_dev);
  const int n_up = (n_walks + 31) / 32 * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += gridDim.x * blockDim.x) {
    int valid = 0;
    if (i < n_walks) {
      int64_t* w = out + static_cast<int64_t>(i) * (L + 1);
      int64_t cur = starts[i / W];
      if (cur < 0 || cur >= types.n[0]) cur = -1;
      w[0] = cur;
      valid = cur >= 0;
      const uint64_t row = (step << 32) | static_cast<uint32_t>(i);
      for (int s = 1; s <= L; ++s) {
        if (cur >= 0) {
          const RowRef r = load_row(rel[(s - 1) % R], cur);
          int64_t nxt = -1;
          if (r.deg > 0) {
            nxt = load_col(rel[(s - 1) % R], r.part,
                           r.start + bounded(philox_draw(seed, kWalkStream, row, s - 1), static_cast<uint32_t>(r.deg)));
            if (nxt >= types.n[pos_slot(s, R)]) nxt = -1;
          }
          cur = nxt;
          valid += cur >= 0;
        }
        w[s] = cur;
      }
    }
    int win = valid >= C ? valid - C + 1 : 0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) win += __shfl_xor_sync(0xffffffffu, win, off);
    if ((threadIdx.x & 31) == 0 && win > 0) atomicAdd(n_valid, win);
  }
}

// node2vec's second-order walk (Grover & Leskovec 2016) over one relation from a type to itself, warp per walk.  Walk
// i starts at starts[i / W].  Step 1 moves to a uniform neighbour.  Step s >= 2, at v with previous node t, weighs every
// entry x of v's row 1/p if x == t, 1 if t's row holds x, 1/q otherwise, and samples it by rejection: propose x
// uniformly from v's row and accept with probability w(x) / max(1, 1/p, 1/q) (w_ret / w_in / w_out are the normalised
// weights).  Proposal k of step s draws Philox(seed, kN2vStream, (step << 32) | i, counter (s - 1) * 4096 + k): word
// x picks the entry, word y is the acceptance uniform.  Lane l evaluates proposals l, l + 32, ... (its own binary
// search of t's row) and the warp takes the lowest-indexed accepted one, which has exactly the distribution of
// sequential rejection sampling, so a walk is a function of (seed, step, i) alone.  After kNode2VecMaxProposals
// rejections the last proposal is taken: with r = max/min weight <= 64 (enforced by the binding) each proposal is
// accepted with probability >= 1/64, so this happens with probability < (63/64)^4096 ~ 1e-28 per walk step.
// Dead ends, ids outside [0, n) and padded starts end the walk (-1 tail) exactly as in k_metapath_walk, and n_valid +=
// the walk's windows of C valid entries.  Rows must be column-sorted for row_has_col's binary search.
__global__ void __launch_bounds__(128) k_node2vec_walk(const GraphTable* rel, MetaPathTypes types,
                                                       const int64_t* starts, int n_walks, int W, int L, int C,
                                                       float w_ret, float w_in, float w_out, uint64_t seed,
                                                       const int32_t* step_dev, int64_t* out, int32_t* n_valid) {
  pdl_enter();
  const GraphTable& g = *rel;
  const uint64_t step = static_cast<uint32_t>(*step_dev);
  const int lane = threadIdx.x & 31;
  const int64_t n = types.n[0];
  // the membership search only decides acceptance when u falls between the two weights of x != t
  const float w_lo = fminf(w_in, w_out), w_hi = fmaxf(w_in, w_out);
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_walks; i += (gridDim.x * blockDim.x) >> 5) {
    int64_t* w = out + static_cast<int64_t>(i) * (L + 1);
    int64_t cur = starts[i / W];
    if (cur < 0 || cur >= n) cur = -1;
    if (lane == 0) w[0] = cur;
    int valid = cur >= 0;
    int64_t prev = -1;
    RowRef prow{};
    const uint32_t row_lo = static_cast<uint32_t>(i), row_hi = static_cast<uint32_t>(step);
    for (int s = 1; s <= L; ++s) {
      if (cur >= 0) {                                 // warp-uniform: every lane holds the same walk state
        const RowRef r = load_row(g, cur);
        int64_t nxt = -1;
        if (r.deg > 0) {
          for (int k0 = 0; k0 < kNode2VecMaxProposals; k0 += 32) {
            const U4 d = philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32),
                                       U4{row_lo, row_hi, static_cast<uint32_t>(s - 1) * kNode2VecMaxProposals +
                                                              static_cast<uint32_t>(k0 + lane), kN2vStream});
            const int64_t x = load_col(g, r.part, r.start + bounded(d.x, static_cast<uint32_t>(r.deg)));
            const float u = u01(d.y);
            bool acc;
            if (prev < 0) acc = true;                 // step 1: uniform
            else if (x == prev) acc = u < w_ret;
            else if (u < w_lo) acc = true;
            else if (u >= w_hi) acc = false;
            else acc = row_has_col(g, prow, x) ? u < w_in : u < w_out;
            const unsigned hit = __ballot_sync(0xffffffffu, acc);
            const int src = hit ? __ffs(hit) - 1 : 31;
            nxt = __shfl_sync(0xffffffffu, x, src);
            if (hit) break;
          }
          if (nxt >= n) nxt = -1;
        }
        prev = cur;
        prow = r;
        cur = nxt;
        valid += cur >= 0;
      }
      if (lane == 0) w[s] = cur;
    }
    const int win = valid >= C ? valid - C + 1 : 0;
    if (lane == 0 && win > 0) atomicAdd(n_valid, win);
  }
}

// Negative window (i, j, k) of walk i, window start j (J = L + 2 - C windows per walk), k < K, at
// neg[((i * J + j) * K + k) * C ...]: entry 0 is the centre walk[i, j], entry c >= 1 is uniform over the node type of
// position j + c, drawn as Philox(seed, kNegStream, (step << 32) | ((i * J + j) * K + k), c - 1).  An invalid
// window (an entry outside its position's type) gets an all -1 negative.
__global__ void __launch_bounds__(256) k_sgns_negatives(const int64_t* walks, int n_walks, int L, int C, int K, int R,
                                                        MetaPathTypes types, uint64_t seed, const int32_t* step_dev,
                                                        int64_t* neg) {
  pdl_enter();
  const uint64_t step = static_cast<uint32_t>(*step_dev);
  const int J = L + 2 - C;
  const int64_t total = static_cast<int64_t>(n_walks) * J * K;
  for (int64_t q = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; q < total;
       q += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int64_t win = q / K;
    const int i = static_cast<int>(win / J), j = static_cast<int>(win % J);
    const int64_t* w = walks + static_cast<int64_t>(i) * (L + 1) + j;
    int64_t* o = neg + q * C;
    bool ok = true;
    for (int c = 0; c < C; ++c) ok = ok && w[c] >= 0 && w[c] < types.n[pos_slot(j + c, R)];
    o[0] = ok ? w[0] : -1;
    const uint64_t row = (step << 32) | static_cast<uint32_t>(q);
    for (int c = 1; c < C; ++c)
      o[c] = ok ? static_cast<int64_t>(bounded(philox_draw(seed, kNegStream, row, c - 1),
                                               static_cast<uint32_t>(types.n[pos_slot(j + c, R)])))
                : -1;
  }
}

// sigma(x) without overflow
__device__ __forceinline__ float sigmoidf_stable(float x) {
  const float e = expf(-fabsf(x));
  return x >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
}

// LPR lanes per window, VPL 8-column vectors per lane.  Window (i, j) is valid when its C entries are ids of their
// position's type.  With h = emb[row], n_pos = n_valid (C - 1), n_neg = K n_pos:
//   loss += -log(sigma(h_c . h_x) + EPS) / n_pos     over its context rows x
//   loss += -log(sigma(-h_c . h_y) + EPS) / n_neg    over the context rows y of its K negative windows
// (sigma(-s) = 1 - sigma(s), evaluated without cancellation), and the gradients of those terms go to grad with
// red.add: the centre's summed over all (1 + K)(C - 1) pairs in registers and added once, every other row per pair.
template <int LPR, int VPL>
__global__ void __launch_bounds__(256) k_sgns_loss_grad(const int64_t* walks, const int64_t* neg, int n_walks, int L,
                                                        int C, int K, int R, MetaPathTypes types, const float* emb,
                                                        int D, const int32_t* n_valid, float* grad, uint8_t* touched,
                                                        float* loss) {
  pdl_enter();
  constexpr int GPW = 32 / LPR;                     // windows per warp and iteration
  const int lane = threadIdx.x & 31, gl = lane % LPR, gw = lane / LPR;
  const int wpb = blockDim.x >> 5;
  const int J = L + 2 - C;
  const int64_t n_win = static_cast<int64_t>(n_walks) * J;
  const int nv = *n_valid;
  const float inv_pos = nv > 0 ? 1.f / (static_cast<float>(nv) * (C - 1)) : 0.f;
  const float inv_neg = inv_pos / K;
  const int nvec = D >> 3;
  float l_acc = 0.f;
  for (int64_t base = (static_cast<int64_t>(blockIdx.x) * wpb + (threadIdx.x >> 5)) * GPW; base < n_win;
       base += static_cast<int64_t>(gridDim.x) * wpb * GPW) {
    const int64_t win = base + gw;
    if (win >= n_win) continue;                     // no warp-wide collectives below span lane groups
    const int i = static_cast<int>(win / J), j = static_cast<int>(win % J);
    const int64_t* w = walks + static_cast<int64_t>(i) * (L + 1) + j;
    bool ok = true;
    for (int c = 0; c < C; ++c) {
      const int64_t v = w[c];
      ok = ok && v >= 0 && v < types.n[pos_slot(j + c, R)];
    }
    if (!ok) continue;
    const int64_t rc = types.off[pos_slot(j, R)] + w[0];
    float hc[VPL][8], gc[VPL][8];
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int c = gl + v * LPR;
#pragma unroll
      for (int q = 0; q < 8; ++q) hc[v][q] = gc[v][q] = 0.f;
      if (c < nvec) {
        const float4* p = reinterpret_cast<const float4*>(emb + rc * D + c * 8);
        const float4 a = p[0], b = p[1];
        hc[v][0] = a.x; hc[v][1] = a.y; hc[v][2] = a.z; hc[v][3] = a.w;
        hc[v][4] = b.x; hc[v][5] = b.y; hc[v][6] = b.z; hc[v][7] = b.w;
      }
    }
    if (gl == 0) touched[rc] = 1;
    // pair t < C - 1: positive context w[t + 1]; pair t >= C - 1: context (t % (C - 1)) + 1 of negative window
    // (t / (C - 1)) - 1
    const int n_pairs = (1 + K) * (C - 1);
    const int64_t* nw = neg + win * K * C;
    for (int t = 0; t < n_pairs; ++t) {
      const int kk = t / (C - 1), c = t % (C - 1) + 1;
      const bool pos = kk == 0;
      int64_t id = pos ? w[c] : nw[(kk - 1) * C + c];
      const int64_t nt = types.n[pos_slot(j + c, R)];
      if (id < 0 || id >= nt) continue;             // a foreign negative buffer entry: skip the pair, never read it
      const int64_t rx = types.off[pos_slot(j + c, R)] + id;
      float hx[VPL][8];
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int cc = gl + v * LPR;
#pragma unroll
        for (int q = 0; q < 8; ++q) hx[v][q] = 0.f;
        if (cc < nvec) {
          const float4* p = reinterpret_cast<const float4*>(emb + rx * D + cc * 8);
          const float4 a = p[0], b = p[1];
          hx[v][0] = a.x; hx[v][1] = a.y; hx[v][2] = a.z; hx[v][3] = a.w;
          hx[v][4] = b.x; hx[v][5] = b.y; hx[v][6] = b.z; hx[v][7] = b.w;
        }
#pragma unroll
        for (int q = 0; q < 8; ++q) s = fmaf(hc[v][q], hx[v][q], s);
      }
#pragma unroll
      for (int off = LPR / 2; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu >> (32 - LPR) << (gw * LPR), s, off);
      const float sp = sigmoidf_stable(s), sn = sigmoidf_stable(-s);
      float g;
      if (pos) {
        l_acc -= gl == 0 ? logf(sp + kSgnsEps) * inv_pos : 0.f;
        g = -sp * sn / (sp + kSgnsEps) * inv_pos;
      } else {
        l_acc -= gl == 0 ? logf(sn + kSgnsEps) * inv_neg : 0.f;
        g = sp * sn / (sn + kSgnsEps) * inv_neg;
      }
      if (gl == 0) touched[rx] = 1;
#pragma unroll
      for (int v = 0; v < VPL; ++v) {
        const int cc = gl + v * LPR;
        if (cc >= nvec) continue;
        float d[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          d[q] = g * hc[v][q];
          gc[v][q] = fmaf(g, hx[v][q], gc[v][q]);
        }
        red_add8(grad + rx * D + cc * 8, d);
      }
    }
#pragma unroll
    for (int v = 0; v < VPL; ++v) {
      const int cc = gl + v * LPR;
      if (cc < nvec) red_add8(grad + rc * D + cc * 8, gc[v]);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) l_acc += __shfl_xor_sync(0xffffffffu, l_acc, off);
  if (lane == 0 && l_acc != 0.f) atomicAdd(loss, l_acc);
}

// Warp per 32 consecutive rows: every row with touched[row] set gets torch.optim.SparseAdam's update at step
// t = *t_dev,
//   m += (g - m)(1 - b1);  v += (g^2 - v)(1 - b2);  w -= lr sqrt(1 - b2^t) / (1 - b1^t) * m / (sqrt(v) + eps)
// then its gradient row and flag are cleared.  Lanes stride the row in float4s.
__global__ void __launch_bounds__(256) k_sparse_adam(float* w, float* grad, float* m, float* v, uint8_t* touched,
                                                     int64_t rows, int D, const int32_t* t_dev, float lr, float b1,
                                                     float b2, float eps) {
  pdl_enter();
  const int lane = threadIdx.x & 31;
  const int t = *t_dev;
  const double bc1 = 1.0 - pow(static_cast<double>(b1), t), bc2 = 1.0 - pow(static_cast<double>(b2), t);
  const float step_size = static_cast<float>(static_cast<double>(lr) * sqrt(bc2) / bc1);
  const float a1 = 1.f - b1, a2 = 1.f - b2;
  const int n4 = D >> 2;
  const int64_t wpg = static_cast<int64_t>(gridDim.x) * (blockDim.x >> 5);
  for (int64_t r0 = (static_cast<int64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 32; r0 < rows;
       r0 += wpg * 32) {
    const int64_t mine = r0 + lane;
    const bool hit = mine < rows && touched[mine];
    unsigned mask = __ballot_sync(0xffffffffu, hit);
    if (hit) touched[mine] = 0;
    while (mask) {
      const int b = __ffs(mask) - 1;
      mask &= mask - 1;
      const int64_t off = (r0 + b) * D;
      for (int c = lane; c < n4; c += 32) {
        float4* gp = reinterpret_cast<float4*>(grad + off) + c;
        float4* mp = reinterpret_cast<float4*>(m + off) + c;
        float4* vp = reinterpret_cast<float4*>(v + off) + c;
        float4* wp = reinterpret_cast<float4*>(w + off) + c;
        const float4 g4 = *gp;
        float4 m4 = *mp, v4 = *vp, w4 = *wp;
        const float gs[4] = {g4.x, g4.y, g4.z, g4.w};
        float* ms[4] = {&m4.x, &m4.y, &m4.z, &m4.w};
        float* vs[4] = {&v4.x, &v4.y, &v4.z, &v4.w};
        float* ws[4] = {&w4.x, &w4.y, &w4.z, &w4.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float mo = *ms[q], vo = *vs[q];
          const float mn = (gs[q] - mo) * a1 + mo;
          const float vn = (gs[q] * gs[q] - vo) * a2 + vo;
          *ms[q] = mn;
          *vs[q] = vn;
          *ws[q] += -step_size * (mn / (sqrtf(vn) + eps));
        }
        *mp = m4;
        *vp = v4;
        *wp = w4;
        *gp = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
}

}  // namespace

void launch_m2v_begin(int32_t* state, cudaStream_t s) { launch_k(k_m2v_begin, dim3(1), dim3(1), 0, s, state); }

void launch_metapath_walk(const GraphTable* rel, int R, MetaPathTypes types, const int64_t* starts, int n_walks, int W,
                          int L, int C, uint64_t seed, const int32_t* step_dev, int64_t* out, int32_t* n_valid,
                          cudaStream_t s) {
  cudaMemsetAsync(n_valid, 0, sizeof(int32_t), s);
  launch_k(k_metapath_walk, dim3(grid_for(n_walks, 128)), dim3(128), 0, s, rel, R, types, starts, n_walks, W, L, C,
           seed, step_dev, out, n_valid);
}

void launch_node2vec_walk(const GraphTable* rel, MetaPathTypes types, const int64_t* starts, int n_walks, int W, int L,
                          int C, float w_ret, float w_in, float w_out, uint64_t seed, const int32_t* step_dev,
                          int64_t* out, int32_t* n_valid, cudaStream_t s) {
  cudaMemsetAsync(n_valid, 0, sizeof(int32_t), s);
  launch_k(k_node2vec_walk, dim3(grid_for(n_walks, 4)), dim3(128), 0, s, rel, types, starts, n_walks, W, L, C, w_ret,
           w_in, w_out, seed, step_dev, out, n_valid);
}

void launch_sgns_negatives(const int64_t* walks, int n_walks, int L, int C, int K, int R, MetaPathTypes types,
                           uint64_t seed, const int32_t* step_dev, int64_t* neg, cudaStream_t s) {
  const int64_t total = static_cast<int64_t>(n_walks) * (L + 2 - C) * K;
  launch_k(k_sgns_negatives, dim3(grid_for(total, 256)), dim3(256), 0, s, walks, n_walks, L, C, K, R, types, seed,
           step_dev, neg);
}

void launch_sgns_loss_grad(const int64_t* walks, const int64_t* neg, int n_walks, int L, int C, int K, int R,
                           MetaPathTypes types, const float* emb, int D, const int32_t* n_valid, float* grad,
                           uint8_t* touched, float* loss, cudaStream_t s) {
  cudaMemsetAsync(loss, 0, sizeof(float), s);
  const int64_t n_win = static_cast<int64_t>(n_walks) * (L + 2 - C);
  dispatch_lanes<4, 2>(D / 8, [&](auto lpr, auto vpl) {
    constexpr int LPR = decltype(lpr)::value, VPL = decltype(vpl)::value;
    launch_k(k_sgns_loss_grad<LPR, VPL>, dim3(grid_for(n_win, 8 * (32 / LPR))), dim3(256), 0, s, walks, neg, n_walks,
             L, C, K, R, types, emb, D, n_valid, grad, touched, loss);
  });
}

void launch_sparse_adam(float* w, float* grad, float* m, float* v, uint8_t* touched, int64_t rows, int D,
                        const int32_t* t_dev, float lr, float b1, float b2, float eps, cudaStream_t s) {
  launch_k(k_sparse_adam, dim3(grid_for((rows + 31) / 32, 8)), dim3(256), 0, s, w, grad, m, v, touched, rows, D, t_dev,
           lr, b1, b2, eps);
}

}  // namespace glt
