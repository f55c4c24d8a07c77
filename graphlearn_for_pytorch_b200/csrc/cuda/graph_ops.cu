// sm_90a kernels for negative sampling, induced subgraphs, random walks and
// hotness propagation.  All of them read the (possibly multi-GPU) GraphTable in
// place, so strict negative sampling and induced subgraphs work *across*
// partitions -- the reference gives up on both in distributed mode
// (distributed/dist_neighbor_sampler.py:411-413 non-strict local negatives,
// :555-571 broadcasts whole node sets over RPC).
#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

// Fused draw + reject + compaction (warp ballot + one atomic per warp); the
// reference needs a kernel plus Thrust copy_if/gather/reduce passes
// (csrc/cuda/random_negative_sampler.cu:95-160).
__global__ void k_negative_sample(GraphTable g, int64_t num_rows, int64_t num_cols, int req,
                                  int trials, int padding, uint64_t seed, uint32_t stream,
                                  int64_t* out_rows, int64_t* out_cols, int32_t* out_count) {
  const int lane = threadIdx.x & 31;
  const int n_up = (req + 31) / 32 * 32;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_up; i += gridDim.x * blockDim.x) {
    bool ok = false;
    int64_t rr = 0, cc = 0;
    if (i < req) {
      for (int t = 0; t < trials && !ok; ++t) {
        rr = bounded(philox_draw(seed, stream, i, 2 * t), static_cast<uint32_t>(num_rows));
        cc = bounded(philox_draw(seed, stream, i, 2 * t + 1), static_cast<uint32_t>(num_cols));
        ok = !edge_exists(g, rr, cc);
      }
      if (!ok && padding) {
        rr = bounded(philox_draw(seed, stream + 0x40000000u, i, 0), static_cast<uint32_t>(num_rows));
        cc = bounded(philox_draw(seed, stream + 0x40000000u, i, 1), static_cast<uint32_t>(num_cols));
        ok = true;
      }
    }
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    int base = 0;
    if (m) {
      if (lane == 0) base = atomicAdd(out_count, __popc(m));
      base = __shfl_sync(0xffffffffu, base, 0);
    }
    if (ok) {
      const int o = base + __popc(m & lanemask_lt());
      out_rows[o] = rr;
      out_cols[o] = cc;
    }
  }
}

// Induced subgraph: warp per node, count pass then fill pass (exact offsets come
// from an exclusive scan in between; sizes never exceed what was counted, unlike
// the reference's col_mask sizing assumption, csrc/cuda/subgraph_op.cu:59,254-264).
__global__ void k_subgraph_count(GraphTable g, HashTable t, const int64_t* nodes, int n, int64_t* cnt) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const RowRef row = load_row(g, nodes[r]);
    int c = 0;
    for (int j = lane; j < row.deg; j += 32)
      c += table_find_slot(t, load_col(g, row.part, row.start + j)) >= 0;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) c += __shfl_xor_sync(0xffffffffu, c, off);
    if (lane == 0) cnt[r] = c;
  }
}

__global__ void k_subgraph_fill(GraphTable g, HashTable t, const int64_t* nodes, int n,
                                const int64_t* offs, int64_t* rows, int64_t* cols, int64_t* eids) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const RowRef row = load_row(g, nodes[r]);
    int64_t o = offs[r];
    for (int base = 0; base < row.deg; base += 32) {
      const int j = base + lane;
      int32_t s = -1;
      if (j < row.deg) s = table_find_slot(t, load_col(g, row.part, row.start + j));
      const unsigned m = __ballot_sync(0xffffffffu, s >= 0);
      if (s >= 0) {
        const int64_t p = o + __popc(m & lanemask_lt());
        rows[p] = r;
        cols[p] = t.vals[s];
        if (eids) eids[p] = __ldg(g.parts[row.part].eids + row.start + j);
      }
      o += __popc(m);
    }
  }
}

// Random walk, thread per walker (new functionality).  A step draws one Philox word for a uniform position, or runs
// node2vec's rejection sampler (philox.h) with two words per proposal: the position, then the acceptance uniform.  A
// walker on a node without out-edges (or outside every shard) stays in place.
__global__ void k_random_walk(GraphTable g, const int64_t* starts, int n, int walk_len, bool biased,
                              Node2VecWeights w, uint64_t seed, uint32_t stream, int64_t* out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int64_t cur = starts[i], prev = -1;
    out[static_cast<int64_t>(i) * (walk_len + 1)] = cur;
    uint32_t draw = 0;
    for (int s = 1; s <= walk_len; ++s) {
      const RowRef row = load_row(g, cur);
      int64_t nxt = cur;
      if (row.deg > 0) {
        if (!biased || prev < 0) {
          nxt = load_col(g, row.part, row.start + bounded(philox_draw(seed, stream, i, draw++), row.deg));
        } else {
          for (int tries = 0; tries < kNode2VecMaxProposals; ++tries) {
            nxt = load_col(g, row.part, row.start + bounded(philox_draw(seed, stream, i, draw++), row.deg));
            const float u = u01(philox_draw(seed, stream, i, draw++));
            if (node2vec_accept(w, nxt == prev, u, [&] { return edge_exists(g, prev, nxt); })) break;
          }
        }
      }
      out[static_cast<int64_t>(i) * (walk_len + 1) + s] = nxt;
      prev = cur;
      cur = nxt;
    }
  }
}

// Hotness propagation (reference CalNbrProbKernel, random_sampler.cu:167-209),
// warp per row instead of a serial thread per row.
__global__ void k_nbr_prob(GraphTable g, GraphTable ng, const float* last, const float* nbr_last,
                           int64_t n, int64_t n_nbr, int k, float* cur) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int64_t v = blockIdx.x * wpb + (threadIdx.x >> 5); v < n; v += static_cast<int64_t>(gridDim.x) * wpb) {
    const RowRef row = load_row(g, v);
    if (row.deg == 0) { if (lane == 0) cur[v] = 0.f; continue; }
    float acc = 1.f;
    for (int j = lane; j < row.deg; j += 32) {
      const int64_t u = load_col(g, row.part, row.start + j);
      if (u < 0 || u >= n_nbr) continue;
      const int du = load_row(ng, u).deg;
      if (du == 0) continue;
      const float pu = nbr_last[u];
      acc *= (du <= k || k < 0) ? 1.f - pu : 1.f - pu * static_cast<float>(k) / static_cast<float>(du);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc *= __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0) cur[v] = 1.f - (1.f - last[v]) * acc;
  }
}

}  // namespace

void launch_negative_sample(GraphTable g, int64_t num_rows, int64_t num_cols, int req, int trials,
                            int padding, uint64_t seed, uint32_t stream, int64_t* out_rows,
                            int64_t* out_cols, int32_t* out_count, cudaStream_t s) {
  cudaMemsetAsync(out_count, 0, sizeof(int32_t), s);
  if (req <= 0) return;
  k_negative_sample<<<grid_for(req, 256), 256, 0, s>>>(g, num_rows, num_cols, req, trials, padding,
                                                        seed, stream, out_rows, out_cols, out_count);
}

void launch_subgraph_count(GraphTable g, HashTable t, const int64_t* nodes, int n, int64_t* cnt,
                           cudaStream_t s) {
  if (n <= 0) return;
  k_subgraph_count<<<grid_for(n, 8), 256, 0, s>>>(g, t, nodes, n, cnt);
}

void launch_subgraph_fill(GraphTable g, HashTable t, const int64_t* nodes, int n, const int64_t* offs,
                          int64_t* rows, int64_t* cols, int64_t* eids, cudaStream_t s) {
  if (n <= 0) return;
  k_subgraph_fill<<<grid_for(n, 8), 256, 0, s>>>(g, t, nodes, n, offs, rows, cols, eids);
}

void launch_random_walk(GraphTable g, const int64_t* starts, int n, int walk_len, bool biased, Node2VecWeights w,
                        uint64_t seed, uint32_t stream, int64_t* out, cudaStream_t s) {
  if (n <= 0) return;
  k_random_walk<<<grid_for(n, 128), 128, 0, s>>>(g, starts, n, walk_len, biased, w, seed, stream, out);
}

void launch_nbr_prob(GraphTable g, GraphTable nbr_g, const float* last, const float* nbr_last,
                     int64_t n, int64_t n_nbr, int k, float* cur, cudaStream_t s) {
  if (n <= 0) return;
  k_nbr_prob<<<grid_for(n, 8), 256, 0, s>>>(g, nbr_g, last, nbr_last, n, n_nbr, k, cur);
}

}  // namespace glt
