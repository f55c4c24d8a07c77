// sm_90a neighbour-sampling kernels.
//
// Design (vs. the reference's DGL-style kernel, csrc/cuda/random_sampler.cu:59-165,
// + 3-kernel hash-table dedup, csrc/cuda/hash_table.cu:26-107):
//   * a sub-warp group (8/16/32 lanes, chosen from the fanout) owns one frontier
//     row -- not a 128-thread CTA per row;
//   * without-replacement sampling is Floyd's k-subset driven by counter-based
//     Philox: O(k) work per row independent of the degree, no curand state, no
//     reads of col_idx except the k winners (each may be a remote NVLink load);
//   * rows live in a GraphTable of up to 16 shards (local HBM / peer HBM / pinned
//     host) and are dereferenced in place;
//   * outputs are fixed-stride (ELL) per hop and every size stays on the device:
//     no D2H count read-back, no exclusive scan, no event sync between hops;
//   * dedup/relabel is fused: winners are inserted into the hash table by the
//     sampling warp itself (warp-aggregated cursor bump), a second tiny kernel
//     resolves slot -> local id.
#include <climits>

#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

constexpr uint32_t kNoPick = 0xFFFFFFFFu;

// Inverse CDF of a row's weights, scanned G consecutive weights at a time with the running sum carried: `pick` is
// the first position of positive weight whose running sum exceeds `target`, or kNoPick.  Without a pick, `total` is
// the row's sum and `last` its last position of positive weight (kNoPick if none).  Every lane of the group returns
// the same.  The sums are fp64: in fp32 one ulp of the running sum of a wide row outgrows its small weights (at 1e5
// weights alternating 1 and 1000 the ulp is 4), which would skew their probabilities.
struct CdfScan { double total; uint32_t pick, last; };

template <int G>
__device__ __forceinline__ CdfScan weight_cdf_find(const float* w, uint32_t d, int gl, unsigned gmask, double target) {
  const int lane0 = (threadIdx.x & 31) - gl;
  double carry = 0.0;
  uint32_t last = kNoPick;
  for (uint32_t base = 0; base < d; base += G) {
    const uint32_t e = base + gl;
    const float we = e < d ? __ldg(w + e) : 0.f;
    double x = we;
#pragma unroll
    for (int off = 1; off < G; off <<= 1) {
      const double y = __shfl_up_sync(gmask, x, off, G);
      if (gl >= off) x += y;
    }
    const bool pos = we > 0.f;
    const unsigned hit = (__ballot_sync(gmask, pos && carry + x > target) & gmask) >> lane0;
    if (hit) return CdfScan{0.0, base + (__ffs(hit) - 1), last};
    const unsigned any = (__ballot_sync(gmask, pos) & gmask) >> lane0;
    if (any) last = base + (31 - __clz(any));
    carry += __shfl_sync(gmask, x, G - 1, G);
  }
  return CdfScan{carry, kNoPick, last};
}

template <int G, int MAXC>
__device__ __forceinline__ void pick_positions(const GraphTable& g, const RowRef& row, int64_t v,
                                               int k, int gl, unsigned gmask, int weighted,
                                               int replace, uint64_t seed, uint32_t stream,
                                               uint32_t (&picks)[MAXC], int& take) {
  const uint32_t d = static_cast<uint32_t>(row.deg);
  const uint32_t uk = static_cast<uint32_t>(k);
#pragma unroll
  for (int c = 0; c < MAXC; ++c) picks[c] = kNoPick;
  take = static_cast<int>(d < uk ? d : uk);
  if (d == 0) return;
  if (d <= uk) {
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      uint32_t j = c * G + gl;
      if (j < d) picks[c] = j;
    }
    return;
  }
  if (replace && !weighted) {
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      uint32_t j = c * G + gl;
      if (j < uk) picks[c] = bounded(philox_draw(seed, stream, v, j), d);
    }
    take = static_cast<int>(uk);
    return;
  }
  if (replace) {
    // weighted with replacement: k independent draws, position e with probability w[e] / W.  Draw i inverts the
    // row's CDF at u_i * W, u_i from counter i as in the uniform draws above.  A row of zero weights picks nothing.
    const float* w = g.parts[row.part].weights + row.start;
    const CdfScan row_sum = weight_cdf_find<G>(w, d, gl, gmask, __longlong_as_double(0x7ff0000000000000ll));
    if (row_sum.last == kNoPick) { take = 0; return; }
    for (uint32_t i = 0; i < uk; ++i) {
      const double target = static_cast<double>(u01(philox_draw(seed, stream, v, i))) * row_sum.total;
      uint32_t pick = weight_cdf_find<G>(w, d, gl, gmask, target).pick;
      if (pick == kNoPick) pick = row_sum.last;   // u * W rounded up past the scan's own running sums
#pragma unroll
      for (int c = 0; c < MAXC; ++c)
        if (i == static_cast<uint32_t>(c * G + gl)) picks[c] = pick;
    }
    take = static_cast<int>(uk);
    return;
  }
  if (!weighted) {
    U4 rnd; rnd.x = rnd.y = rnd.z = rnd.w = 0;
    for (uint32_t i = 0; i < uk; ++i) {
      if ((i & 3u) == 0) {
        U4 c;
        c.x = static_cast<uint32_t>(v); c.y = static_cast<uint32_t>(static_cast<uint64_t>(v) >> 32);
        c.z = i >> 2; c.w = stream;
        rnd = philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), c);
      }
      const uint32_t r = ((i & 3u) == 0) ? rnd.x : ((i & 3u) == 1) ? rnd.y : ((i & 3u) == 2) ? rnd.z : rnd.w;
      const uint32_t j = d - uk + i;
      const uint32_t t = bounded(r, j + 1u);
      bool match = false;
#pragma unroll
      for (int c = 0; c < MAXC; ++c) match |= (picks[c] == t);
      const bool dup = __any_sync(gmask, match);
      const uint32_t pick = dup ? j : t;
#pragma unroll
      for (int c = 0; c < MAXC; ++c)
        if (i == static_cast<uint32_t>(c * G + gl)) picks[c] = pick;
    }
    return;
  }
  // weighted: k rounds of group-argmin over exponential-race keys
  const float* w = g.parts[row.part].weights + row.start;
  float last_key = -1.f;
  uint32_t last_idx = 0;
  for (uint32_t i = 0; i < uk; ++i) {
    float best = 3.4e38f;
    uint32_t bidx = kNoPick;
    for (uint32_t e = gl; e < d; e += G) {
      const float key = weighted_key(seed, stream, v, e, __ldg(w + e));
      const bool after = (i == 0) || key > last_key || (key == last_key && e > last_idx);
      if (after && (key < best || (key == best && e < bidx))) { best = key; bidx = e; }
    }
#pragma unroll
    for (int off = G / 2; off > 0; off >>= 1) {
      const float ok = __shfl_xor_sync(gmask, best, off, G);
      const uint32_t oi = __shfl_xor_sync(gmask, bidx, off, G);
      if (ok < best || (ok == best && oi < bidx)) { best = ok; bidx = oi; }
    }
    last_key = best; last_idx = bidx;
#pragma unroll
    for (int c = 0; c < MAXC; ++c)
      if (i == static_cast<uint32_t>(c * G + gl)) picks[c] = bidx;
  }
}

template <int G, int MAXC>
__device__ __forceinline__ void sample_hop_body(const HopArgs& a) {
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const int gw = lane / G;
  constexpr int RPW = 32 / G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gw * G));
  const int f_begin = a.c.cum[a.hop];
  const int n_rows = min(a.c.cum[a.hop + 1] - f_begin, a.cap_rows);
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5;
  // under CUDA-graph replay the host-side stream id is frozen: advance it from the device
  const uint32_t rng_stream = a.stream + (a.stream_dev ? static_cast<uint32_t>(*a.stream_dev) *
                                                         (a.stream_stride ? a.stream_stride : 8u) : 0u);
  int64_t* nodes_out = a.nodes_out ? a.nodes_out : a.nodes;
  int edge_acc = 0;
  for (int base = (blockIdx.x * warps_per_block + warp) * RPW; base < n_rows;
       base += gridDim.x * warps_per_block * RPW) {
    const int r = base + gw;
    const bool valid = r < n_rows;
    const int64_t v = valid ? a.nodes[f_begin + r] : -1;
    RowRef row; row.start = 0; row.deg = 0; row.part = -1;
    if (valid) row = load_row(a.g, v);
    uint32_t picks[MAXC];
    int take = 0;
    pick_positions<G, MAXC>(a.g, row, v, a.k, gl, gmask, a.weighted, a.replace, a.seed, rng_stream,
                            picks, take);
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int j = c * G + gl;
      int64_t key = -1, eid = -1;
      bool have = valid && picks[c] != kNoPick;
      if (have) {
        key = load_col(a.g, row.part, row.start + picks[c]);
        if (a.ell_eids) eid = __ldg(a.g.parts[row.part].eids + row.start + picks[c]);
      }
      bool is_new = false;
      uint32_t slot = 0;
      if (have) {
        slot = table_insert(a.t, key, &is_new);
        if (slot == kTableFull) {  // table exhausted: drop the neighbour (relabel compacts the row)
          have = false;
          if (a.c.overflow) atomicAdd(a.c.overflow, 1);
        }
      }
      // warp-aggregated local-id assignment
      const unsigned nm = __ballot_sync(0xffffffffu, is_new);
      int id_base = 0;
      if (nm) {
        if (lane == 0) id_base = atomicAdd(a.c.cursor, __popc(nm));
        id_base = __shfl_sync(0xffffffffu, id_base, 0);
      }
      if (is_new) {
        const int id = id_base + __popc(nm & lanemask_lt());
        if (id < a.cap_nodes) { a.t.vals[slot] = id; nodes_out[id] = key; }
        else a.t.vals[slot] = -1;  // arena overflow: the node is dropped (counted by the relabel pass)
      }
      if (valid && j < a.k) {
        const int64_t o = static_cast<int64_t>(r) * a.k + j;
        a.ell[o] = have ? static_cast<int32_t>(slot) : -1;
        if (a.ell_eids) a.ell_eids[o] = eid;
      }
    }
    if (valid && gl == 0) { a.deg[f_begin + r] = take; edge_acc += take; }
  }
  // one atomic per warp for the hop's edge counter
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) edge_acc += __shfl_xor_sync(0xffffffffu, edge_acc, off);
  if (lane == 0 && edge_acc) atomicAdd(a.c.edges + a.hop, edge_acc);
}

template <int G, int MAXC>
__global__ void __launch_bounds__(256) k_sample_hop(HopArgs a) {
  pdl_enter();
  sample_hop_body<G, MAXC>(a);
}

// one launch for every relation of a heterogeneous hop: blockIdx.y = relation
template <int G, int MAXC>
__global__ void __launch_bounds__(256) k_sample_hop_grouped(const HopArgs* descs) {
  pdl_enter();
  const HopArgs& a = descs[blockIdx.y];
  if (a.k <= 0) return;
  sample_hop_body<G, MAXC>(a);
}

// G lanes per frontier row (the same group width as the sampling kernel): slot -> local id for the row's
// entries in parallel, and rows that lost a neighbour (arena / table overflow) are compacted in place with a
// ballot + prefix count, deg[] and the hop's edge counter corrected, so the mean divides by the neighbours that
// exist and to_coo never emits -1.  (A thread-per-row version of this pass cost 18 us on a 1024-row frontier: 15
// serial table reads per thread on four CTAs.)
template <int G>
__device__ __forceinline__ void relabel_hop_body(const HopArgs& a) {
  const int f_begin = a.c.cum[a.hop];
  const int n_rows = min(a.c.cum[a.hop + 1] - f_begin, a.cap_rows);
  // Capacity guard (arenas may be sized from calibration instead of the worst case): the
  // next frontier holds at most cap_rows_next rows and the arena cap_nodes nodes.  Nodes past
  // the bound are dropped: their slot is poisoned (-1) so later hops treat them as absent.
  // Every thread derives the same bound from stable inputs; the cursor reset is idempotent.
  const int bound = a.bound_ptr ? *a.bound_ptr
                                : min(min(*a.c.cursor, a.cap_nodes), a.c.cum[a.hop + 1] + a.cap_rows_next);
  constexpr int RPW = 32 / G;
  const int lane = threadIdx.x & 31;
  const int gl = lane % G, gw = lane / G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gw * G));
  const int warps_per_block = blockDim.x >> 5;
  int dropped = 0;
  for (int base = (blockIdx.x * warps_per_block + (threadIdx.x >> 5)) * RPW; base < n_rows;
       base += gridDim.x * warps_per_block * RPW) {
    const int r = base + gw;
    const bool valid_row = r < n_rows;
    int32_t* row = a.ell + static_cast<int64_t>(valid_row ? r : 0) * a.k;
    int64_t* erow = a.ell_eids ? a.ell_eids + static_cast<int64_t>(valid_row ? r : 0) * a.k : nullptr;
    const int dg = valid_row ? min(a.deg[f_begin + r], a.k) : 0;
    int w = 0;                                   // compacted entries written so far (uniform inside the group)
    for (int j0 = 0; j0 < a.k; j0 += G) {        // uniform trip count across the warp
      const int j = j0 + gl;
      int32_t v = -1;
      int64_t e = -1;
      if (j < dg) {
        const int32_t s = row[j];
        if (s >= 0) {
          v = a.t.vals[s];
          if (v >= bound) { a.t.vals[s] = -1; v = -1; }
        }
        if (erow) e = erow[j];
      }
      const unsigned m = (__ballot_sync(0xffffffffu, v >= 0) & gmask) >> (gw * G);
      const int pos = w + __popc(m & ((1u << gl) - 1u));
      __syncwarp();                              // every lane has read its entry before anyone overwrites the row
      if (v >= 0) { row[pos] = v; if (erow) erow[pos] = e; }
      w += __popc(m);
    }
    if (w < dg) {                                // holes: blank the tail, fix the degree
      for (int j = w + gl; j < dg; j += G) { row[j] = -1; if (erow) erow[j] = -1; }
      if (gl == 0) { a.deg[f_begin + r] = w; dropped += dg - w; }
    }
  }
  if (dropped) {
    if (a.c.overflow) atomicAdd(a.c.overflow, dropped);
    atomicSub(a.c.edges + a.hop, dropped);
  }
  if (a.bound_ptr == nullptr && blockIdx.x == 0 && threadIdx.x == 0) {
    a.c.cum[a.hop + 2] = bound;
    *a.c.cursor = bound;
  }
}

template <int G>
__global__ void __launch_bounds__(256) k_relabel_hop(HopArgs a) {
  pdl_enter();
  relabel_hop_body<G>(a);
}

template <int G>
__global__ void __launch_bounds__(256) k_relabel_hop_grouped(const HopArgs* descs) {
  pdl_enter();
  const HopArgs& a = descs[blockIdx.y];
  if (a.k <= 0) return;
  relabel_hop_body<G>(a);
}

__global__ void k_hetero_finalize(const HeteroTypeState* types, int n_types, int hop) {
  pdl_enter();
  const int t = threadIdx.x;
  if (t >= n_types) return;
  const HeteroTypeState& ty = types[t];
  const int bound = min(min(*ty.cursor, ty.cap_nodes), ty.cum[hop + 1] + ty.cap_rows[hop + 1]);
  ty.cum[hop + 2] = bound;
  *ty.cursor = bound;
}

// ---- deterministic local-id order (opt-in) -------------------------------------------------------------
// The sampling kernel hands out the local ids of a hop's NEW nodes with an atomic cursor, i.e. in arrival order,
// which varies from run to run.  With the option on, the new ids of every hop are re-assigned in ascending
// global-id order between the sampling and the relabel pass:
//   k_det_keys    tmp[i] = nodes[i] for the hop's new range [cum[hop+1], min(cursor, cap)), +inf elsewhere
//   (device sort of tmp; static size = arena capacity)
//   k_det_assign  nodes[start + j] = sorted[j]; vals[slot(sorted[j])] = start + j
// The relabel pass then maps slots to the new ids as usual.
__global__ void k_det_keys(const int64_t* nodes, const int32_t* cum, const int32_t* cursor, int hop, int cap_nodes,
                           int64_t* tmp) {
  pdl_enter();
  const int start = cum[hop + 1];
  const int end = min(*cursor, cap_nodes);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < cap_nodes; i += gridDim.x * blockDim.x)
    tmp[i] = (i >= start && i < end) ? nodes[i] : INT64_MAX;
}

__global__ void k_det_assign(HashTable t, int64_t* nodes, const int32_t* cum, const int32_t* cursor, int hop,
                             int cap_nodes, const int64_t* sorted) {
  pdl_enter();
  const int start = cum[hop + 1];
  const int n_new = min(*cursor, cap_nodes) - start;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_new; j += gridDim.x * blockDim.x) {
    const int64_t key = sorted[j];
    nodes[start + j] = key;
    const int32_t slot = table_find_slot(t, key);
    if (slot >= 0) t.vals[slot] = start + j;
  }
}

// Ordered (first-occurrence) seed insertion; single CTA, seeds are few.
__global__ void __launch_bounds__(1024) k_init_seeds(const int64_t* seeds, int n_host,
                                                     const int32_t* n_dev, HashTable t,
                                                     int64_t* nodes, int32_t* seed_local,
                                                     int32_t* slot_of, BatchCounters c, int max_hops,
                                                     int32_t* step_dev, int step_inc) {
  pdl_enter();
  __shared__ int s_warp[32];
  __shared__ int s_running;
  // first kernel of a batch: advance the device-side Philox step here instead of paying a
  // separate elementwise launch (the hop kernels that follow read the new value)
  if (threadIdx.x == 0 && step_dev) *step_dev += step_inc;
  const int n = n_dev ? min(*n_dev, n_host) : n_host;
  const int tid = threadIdx.x;
  // 1a: claim slots; the claimer seeds aux with its own index
  for (int i = tid; i < n; i += blockDim.x) {
    const int64_t key = seeds[i];
    if (key < 0) { slot_of[i] = -1; continue; }
    bool is_new;
    const uint32_t s = table_insert(t, key, &is_new);
    slot_of[i] = (s == kTableFull) ? -1 : static_cast<int32_t>(s);
    if (is_new) t.aux[s] = i;
  }
  __syncthreads();
  // 1b: first occurrence = min index over duplicates
  for (int i = tid; i < n; i += blockDim.x)
    if (slot_of[i] >= 0) atomicMin(t.aux + slot_of[i], i);
  if (tid == 0) s_running = 0;
  __syncthreads();
  // 2: block scan over "is first occurrence" flags, chunk by chunk
  for (int base = 0; base < n; base += blockDim.x) {
    const int i = base + tid;
    int flag = 0, s = -1;
    if (i < n) { s = slot_of[i]; flag = (s >= 0 && t.aux[s] == i) ? 1 : 0; }
    int x = flag;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, x, off);
      if ((tid & 31) >= off) x += y;
    }
    if ((tid & 31) == 31) s_warp[tid >> 5] = x;
    __syncthreads();
    if (tid < 32) {
      int w = (tid < (blockDim.x >> 5)) ? s_warp[tid] : 0;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, w, off);
        if (tid >= off) w += y;
      }
      s_warp[tid] = w;
    }
    __syncthreads();
    const int warp_off = (tid >> 5) ? s_warp[(tid >> 5) - 1] : 0;
    const int id = s_running + warp_off + x - flag;
    if (flag) { t.vals[s] = id; nodes[id] = seeds[i]; }
    __syncthreads();
    if (tid == 0) s_running += s_warp[(blockDim.x >> 5) - 1];
    __syncthreads();
  }
  // 3: inverse map + counters
  for (int i = tid; i < n; i += blockDim.x)
    if (seed_local) seed_local[i] = slot_of[i] >= 0 ? t.vals[slot_of[i]] : -1;
  if (tid == 0) {
    c.cum[0] = 0; c.cum[1] = s_running; *c.cursor = s_running;
    for (int h = 0; h < max_hops; ++h) { c.edges[h] = 0; c.cum[h + 2] = s_running; }
  }
}

template <int G, int MAXC>
__global__ void __launch_bounds__(256) k_sample_one_hop(GraphTable g, const int64_t* seeds, int n,
                                                        int k, int weighted, int replace,
                                                        uint64_t seed, uint32_t stream,
                                                        int64_t* out_nbrs, int64_t* out_eids,
                                                        int32_t* out_cnt) {
  const int lane = threadIdx.x & 31;
  const int gl = lane % G;
  const int gw = lane / G;
  constexpr int RPW = 32 / G;
  const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (gw * G));
  const int warps_per_block = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5;
  for (int base = (blockIdx.x * warps_per_block + warp) * RPW; base < n;
       base += gridDim.x * warps_per_block * RPW) {
    const int r = base + gw;
    const bool valid = r < n;
    const int64_t v = valid ? seeds[r] : -1;
    RowRef row; row.start = 0; row.deg = 0; row.part = -1;
    if (valid) row = load_row(g, v);
    uint32_t picks[MAXC];
    int take = 0;
    pick_positions<G, MAXC>(g, row, v, k, gl, gmask, weighted, replace, seed, stream, picks, take);
#pragma unroll
    for (int c = 0; c < MAXC; ++c) {
      const int j = c * G + gl;
      if (valid && j < k) {
        const bool have = picks[c] != kNoPick;
        const int64_t o = static_cast<int64_t>(r) * k + j;
        out_nbrs[o] = have ? load_col(g, row.part, row.start + picks[c]) : -1;
        if (out_eids) out_eids[o] = have ? __ldg(g.parts[row.part].eids + row.start + picks[c]) : -1;
      }
    }
    if (valid && gl == 0) out_cnt[r] = take;
  }
}

__global__ void k_lookup_degree(GraphTable g, const int64_t* ids, int n, int64_t* out) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    out[i] = load_row(g, ids[i]).deg;
}

// warp per row full-neighbourhood copy
__global__ void k_copy_neighbors(GraphTable g, const int64_t* ids, int n, const int64_t* offs,
                                 int64_t* out_nbrs, int64_t* out_eids) {
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  for (int r = blockIdx.x * wpb + (threadIdx.x >> 5); r < n; r += gridDim.x * wpb) {
    const RowRef row = load_row(g, ids[r]);
    const int64_t o = offs[r];
    for (int j = lane; j < row.deg; j += 32) {
      out_nbrs[o + j] = load_col(g, row.part, row.start + j);
      if (out_eids) out_eids[o + j] = __ldg(g.parts[row.part].eids + row.start + j);
    }
  }
}

__global__ void k_ell_to_coo(const int32_t* ell, const int64_t* ell_eids, const int32_t* deg,
                             const int64_t* offs, const int32_t* cum, int hop, int k, int cap_rows,
                             int64_t* rows, int64_t* cols, int64_t* eids) {
  const int f_begin = cum[hop];
  const int n_rows = min(cum[hop + 1] - f_begin, cap_rows);
  const int64_t n = static_cast<int64_t>(n_rows) * k;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / k), j = static_cast<int>(i % k);
    const int t = f_begin + r;
    if (j < deg[t]) {
      const int64_t o = offs[t] + j;
      rows[o] = ell[i];
      cols[o] = t;
      if (eids) eids[o] = ell_eids[i];
    }
  }
}

__global__ void k_table_insert(HashTable t, const int64_t* keys, int64_t n, int64_t* nodes,
                               int32_t* cursor, int cap_nodes, int32_t* out_slots) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const int64_t n_up = (n + 31) / 32 * 32;
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n_up; i += stride) {
    bool is_new = false;
    uint32_t slot = 0;
    const bool have = i < n && keys[i] >= 0;
    bool full = false;
    if (have) { slot = table_insert(t, keys[i], &is_new); full = (slot == kTableFull); }
    const unsigned nm = __ballot_sync(0xffffffffu, is_new);
    int id_base = 0;
    if (nm) {
      if (lane == 0) id_base = atomicAdd(cursor, __popc(nm));
      id_base = __shfl_sync(0xffffffffu, id_base, 0);
    }
    if (is_new) {
      const int id = id_base + __popc(nm & lanemask_lt());
      if (id < cap_nodes) { t.vals[slot] = id; nodes[id] = keys[i]; }
    }
    if (i < n) out_slots[i] = (have && !full) ? static_cast<int32_t>(slot) : -1;
  }
}

__global__ void k_table_resolve(HashTable t, int32_t* slots, int64_t n) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int32_t s = slots[i];
    if (s >= 0) slots[i] = t.vals[s];
  }
}

__global__ void k_table_lookup(HashTable t, const int64_t* keys, int64_t n, int32_t* out) {
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const int32_t s = keys[i] >= 0 ? table_find_slot(t, keys[i]) : -1;
    out[i] = s >= 0 ? t.vals[s] : -1;
  }
}

}  // namespace

void launch_table_clear(HashTable t, cudaStream_t s) {
  cudaMemsetAsync(t.keys, 0xFF, (static_cast<size_t>(t.mask) + 1) * sizeof(int64_t), s);
}

void launch_init_seeds(const int64_t* seeds, int n_seeds, const int32_t* n_seeds_dev, HashTable t,
                       int64_t* nodes, int32_t* seed_local, int32_t* scratch, BatchCounters c,
                       int32_t* step_dev, int step_inc, cudaStream_t s) {
  launch_k(k_init_seeds, dim3(1), dim3(1024), 0, s, seeds, n_seeds, n_seeds_dev, t, nodes, seed_local, scratch, c, 4,
           step_dev, step_inc);
}

#define GLT_DISPATCH_FANOUT(K, ...)                                  \
  do {                                                               \
    if ((K) <= 8) { constexpr int G = 8, MAXC = 1; __VA_ARGS__; }    \
    else if ((K) <= 16) { constexpr int G = 16, MAXC = 1; __VA_ARGS__; } \
    else if ((K) <= 32) { constexpr int G = 32, MAXC = 1; __VA_ARGS__; } \
    else if ((K) <= 128) { constexpr int G = 32, MAXC = 4; __VA_ARGS__; } \
    else { constexpr int G = 32, MAXC = 16; __VA_ARGS__; }           \
  } while (0)

void launch_sample_hop(const HopArgs& a, cudaStream_t s) {
  GLT_DISPATCH_FANOUT(a.k, {
    const int rows_per_block = (256 / 32) * (32 / G);
    launch_k(k_sample_hop<G, MAXC>, dim3(grid_for(a.cap_rows, rows_per_block)), dim3(256), 0, s, a);
  });
}

#define GLT_DISPATCH_GROUP(K, ...)                        \
  do {                                                   \
    if ((K) <= 8) { constexpr int G = 8; __VA_ARGS__; }  \
    else if ((K) <= 16) { constexpr int G = 16; __VA_ARGS__; } \
    else { constexpr int G = 32; __VA_ARGS__; }          \
  } while (0)

void launch_det_keys(const HopArgs& a, int64_t* tmp, cudaStream_t s) {
  launch_k(k_det_keys, dim3(grid_for(a.cap_nodes, 256)), dim3(256), 0, s, static_cast<const int64_t*>(a.nodes),
           static_cast<const int32_t*>(a.c.cum), static_cast<const int32_t*>(a.c.cursor), a.hop, a.cap_nodes, tmp);
}

void launch_det_assign(const HopArgs& a, const int64_t* sorted, cudaStream_t s) {
  launch_k(k_det_assign, dim3(grid_for(a.cap_rows_next, 256)), dim3(256), 0, s, a.t, a.nodes,
           static_cast<const int32_t*>(a.c.cum), static_cast<const int32_t*>(a.c.cursor), a.hop, a.cap_nodes, sorted);
}

void launch_relabel_hop(const HopArgs& a, cudaStream_t s) {
  GLT_DISPATCH_GROUP(a.k, {
    const int rows_per_block = (256 / 32) * (32 / G);
    launch_k(k_relabel_hop<G>, dim3(grid_for(a.cap_rows, rows_per_block)), dim3(256), 0, s, a);
  });
}

void launch_sample_hop_grouped(const HopArgs* descs, int n_rel, int max_k, int max_rows, cudaStream_t s) {
  if (n_rel <= 0 || max_k <= 0) return;
  GLT_DISPATCH_FANOUT(max_k, {
    const int rows_per_block = (256 / 32) * (32 / G);
    dim3 grid(grid_for(max_rows, rows_per_block, 132 * 8), n_rel);
    launch_k(k_sample_hop_grouped<G, MAXC>, grid, dim3(256), 0, s, descs);
  });
}

void launch_relabel_hop_grouped(const HopArgs* descs, int n_rel, int max_k, int max_rows, cudaStream_t s) {
  if (n_rel <= 0 || max_k <= 0) return;
  GLT_DISPATCH_GROUP(max_k, {
    const int rows_per_block = (256 / 32) * (32 / G);
    dim3 grid(grid_for(max_rows, rows_per_block, 132 * 8), n_rel);
    launch_k(k_relabel_hop_grouped<G>, grid, dim3(256), 0, s, descs);
  });
}

void launch_hetero_finalize(const HeteroTypeState* types, int n_types, int hop, cudaStream_t s) {
  if (n_types <= 0) return;
  launch_k(k_hetero_finalize, dim3(1), dim3(32 * ((n_types + 31) / 32)), 0, s, types, n_types, hop);
}

void launch_sample_one_hop(GraphTable g, const int64_t* seeds, int n, int k, int weighted,
                           int replace, uint64_t seed, uint32_t stream, int64_t* out_nbrs,
                           int64_t* out_eids, int32_t* out_cnt, cudaStream_t s) {
  if (n <= 0) return;
  GLT_DISPATCH_FANOUT(k, {
    const int rows_per_block = (256 / 32) * (32 / G);
    k_sample_one_hop<G, MAXC><<<grid_for(n, rows_per_block), 256, 0, s>>>(
        g, seeds, n, k, weighted, replace, seed, stream, out_nbrs, out_eids, out_cnt);
  });
}

void launch_lookup_degree(GraphTable g, const int64_t* ids, int n, int64_t* out, cudaStream_t s) {
  if (n <= 0) return;
  k_lookup_degree<<<grid_for(n, 256), 256, 0, s>>>(g, ids, n, out);
}

void launch_copy_neighbors(GraphTable g, const int64_t* ids, int n, const int64_t* offs,
                           int64_t* out_nbrs, int64_t* out_eids, cudaStream_t s) {
  if (n <= 0) return;
  k_copy_neighbors<<<grid_for(n, 8), 256, 0, s>>>(g, ids, n, offs, out_nbrs, out_eids);
}

void launch_ell_to_coo(const int32_t* ell, const int64_t* ell_eids, const int32_t* deg,
                       const int64_t* offs, const int32_t* cum, int hop, int k, int cap_rows,
                       int64_t* rows, int64_t* cols, int64_t* eids, cudaStream_t s) {
  k_ell_to_coo<<<grid_for(static_cast<int64_t>(cap_rows) * k, 256 * 4), 256, 0, s>>>(
      ell, ell_eids, deg, offs, cum, hop, k, cap_rows, rows, cols, eids);
}

void launch_table_insert(HashTable t, const int64_t* keys, int64_t n, int64_t* nodes,
                         int32_t* cursor, int cap_nodes, int32_t* out_slots, cudaStream_t s) {
  if (n <= 0) return;
  k_table_insert<<<grid_for(n, 256), 256, 0, s>>>(t, keys, n, nodes, cursor, cap_nodes, out_slots);
}

void launch_table_resolve(HashTable t, int32_t* slots, int64_t n, cudaStream_t s) {
  if (n <= 0) return;
  k_table_resolve<<<grid_for(n, 256 * 4), 256, 0, s>>>(t, slots, n);
}

void launch_table_lookup(HashTable t, const int64_t* keys, int64_t n, int32_t* out, cudaStream_t s) {
  if (n <= 0) return;
  k_table_lookup<<<grid_for(n, 256), 256, 0, s>>>(t, keys, n, out);
}

}  // namespace glt
