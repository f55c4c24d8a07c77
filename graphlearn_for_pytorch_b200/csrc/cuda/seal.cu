// SEAL link-prediction kernels of SealEngine (models/seal_engine.py), one CTA per link.  One training step is
//   k_seal_extract   the link's num_hops enclosing subgraph in a shared-memory hash, its induced edges without the
//                    target pair as local CSRs by source and by destination, and DRNL labels from two BFS passes
//   k_seal_forward   DGCNN: GCN stack (layer 1 = row gather of W1 by z), sort-pool, conv1 / maxpool / conv2, MLP, BCE
//   k_seal_backward  the reverse, into a per-link row of weight-gradient partials
//   k_seal_reduce    gradient = the valid links' partials summed in link order; loss likewise
// followed by the flat Adam (launch_adam).  No kernel reads anything back to the host and every sum has a fixed order,
// so the step is bitwise deterministic and is captured into one CUDA graph.
#include <climits>

#include "device_utils.cuh"
#include "launch_utils.h"

namespace glt {

namespace {

constexpr int kSealThreads = 256;
constexpr int kSealLin = 128;                 // hidden width of the MLP
constexpr uint32_t kSealNbrStream = 0x5EA1A8B5u;
constexpr uint32_t kSealDropStream = 0x5EA1D509u;

__host__ __device__ inline int hash_slots_for(int max_nodes) {
  int hs = 1;
  while (hs < 2 * (max_nodes + kSealThreads)) hs <<= 1;
  return hs;
}

// Draw i of the neighbour subset of `node` for link `link` at step `step`.
__device__ __forceinline__ uint32_t seal_nbr_draw(uint64_t seed, uint32_t step, int link, int64_t node, uint32_t i) {
  const U4 c{static_cast<uint32_t>(node), (static_cast<uint32_t>(node >> 32) & 0xFFu) | (static_cast<uint32_t>(link) << 8),
             i >> 2, step};
  const U4 r = philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32) ^ kSealNbrStream, c);
  switch (i & 3u) {
    case 0: return r.x;
    case 1: return r.y;
    case 2: return r.z;
    default: return r.w;
  }
}

__device__ __forceinline__ float seal_drop_u01(uint64_t seed, uint32_t step, int link, int j) {
  const U4 c{static_cast<uint32_t>(j), static_cast<uint32_t>(link), step, kSealDropStream};
  return u01(philox4x32_10(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32), c).x);
}

// Exclusive scan of a[0, m) in shared memory, in place; returns the total.  Every thread of the block calls it.
__device__ int block_scan_excl(int* a, int m, int* tmp) {
  const int t = threadIdx.x, per = (m + blockDim.x - 1) / blockDim.x;
  const int lo = min(m, t * per), hi = min(m, lo + per);
  int s = 0;
  for (int i = lo; i < hi; ++i) s += a[i];
  const int lane = t & 31, w = t >> 5;
  int inc = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += y;
  }
  if (lane == 31) tmp[w] = inc;
  __syncthreads();
  if (t == 0) {
    int r = 0;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) { const int x = tmp[i]; tmp[i] = r; r += x; }
    tmp[32] = r;
  }
  __syncthreads();
  int run = tmp[w] + inc - s;
  for (int i = lo; i < hi; ++i) { const int x = a[i]; a[i] = run; run += x; }
  const int total = tmp[32];
  __syncthreads();
  return total;
}

// Rank of this thread's flag among the set flags of lower threads; *total = set flags of the block.
__device__ int block_rank(bool f, int* tmp, int* total) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, f);
  if (lane == 0) tmp[w] = __popc(bal);
  __syncthreads();
  if (t == 0) {
    int r = 0;
    for (int i = 0; i < static_cast<int>(blockDim.x >> 5); ++i) { const int x = tmp[i]; tmp[i] = r; r += x; }
    tmp[32] = r;
  }
  __syncthreads();
  const int rank = tmp[w] + __popc(bal & lanemask_lt());
  *total = tmp[32];
  __syncthreads();
  return rank;
}

// Shared-memory set of the link's nodes: keys = global ids (-1 empty); vals < 0 encode local id -(val + 2), vals >= 0
// are the first candidate index of a node seen but not (yet) taken.
__device__ __forceinline__ int smem_insert(long long* keys, uint32_t mask, int64_t key) {
  uint32_t s = hash_slot(key, mask);
  for (uint32_t p = 0; p <= mask; ++p) {
    const long long prev = atomicCAS(reinterpret_cast<unsigned long long*>(keys + s), static_cast<unsigned long long>(-1LL),
                                     static_cast<unsigned long long>(key));
    if (prev == -1LL || prev == key) return static_cast<int>(s);
    s = (s + 1) & mask;
  }
  return -1;
}

__device__ __forceinline__ int smem_local(const long long* keys, const int* vals, uint32_t mask, int64_t key) {
  uint32_t s = hash_slot(key, mask);
  for (uint32_t p = 0; p <= mask; ++p) {
    const long long k = keys[s];
    if (k == key) { const int v = vals[s]; return v < 0 ? -v - 2 : -1; }
    if (k == -1LL) return -1;
    s = (s + 1) & mask;
  }
  return -1;
}

__device__ __forceinline__ bool seal_valid(const int64_t* links, int B, int64_t N, int b) {
  const int64_t s = links[b], d = links[B + b];
  return s >= 0 && s < N && d >= 0 && d < N && s != d;
}

// Level-synchronous BFS over the local edges taken as undirected, with node `rem` deleted; dist -1 = unreachable.
__device__ void seal_bfs(short* dist, int src, int rem, int n, const int32_t* sp, const int16_t* sc, const int32_t* dp,
                         const int16_t* dc, int* flag) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) dist[i] = i == src ? 0 : -1;
  for (int level = 0; level < n; ++level) {
    if (threadIdx.x == 0) *flag = 0;
    __syncthreads();
    for (int u = threadIdx.x; u < n; u += blockDim.x) {
      if (dist[u] != level) continue;
      for (int e = sp[u]; e < sp[u + 1]; ++e) {
        const int v = sc[e];
        if (v != rem && dist[v] < 0) { dist[v] = static_cast<short>(level + 1); *flag = 1; }
      }
      for (int e = dp[u]; e < dp[u + 1]; ++e) {
        const int v = dc[e];
        if (v != rem && dist[v] < 0) { dist[v] = static_cast<short>(level + 1); *flag = 1; }
      }
    }
    __syncthreads();
    const int more = *flag;
    __syncthreads();
    if (!more) break;
  }
}

// Link b = (s, d).  Nodes in discovery order: s, d, then hop by hop each frontier node's row (or its drawn subset, in
// row order) in frontier order; the first max_nodes are kept.  Edges: for each kept u in local order, the entries of
// u's row that are kept nodes, except s -> d and d -> s; the first max_edges are kept.
__global__ void __launch_bounds__(kSealThreads) k_seal_extract(SealExtractArgs e, SealArenaPtrs a) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int tmp[34];
  __shared__ int flag;
  const int Nmax = a.max_nodes, Emax = a.max_edges, HS = hash_slots_for(Nmax);
  long long* keys = reinterpret_cast<long long*>(smem);
  long long* nid = keys + HS;
  int* vals = reinterpret_cast<int*>(nid + Nmax);
  int* sa = vals + HS;
  int* sp = sa + Nmax + 1;
  int* dp = sp + Nmax + 1;
  short* ds = reinterpret_cast<short*>(dp + Nmax + 1);
  short* dd = ds + Nmax;
  pdl_enter();
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, w = t >> 5, nw = blockDim.x >> 5;
  int32_t* meta = a.meta + b * kSealMeta;
  if (!seal_valid(e.links, a.B, e.num_nodes, b)) {
    if (t < kSealMeta) meta[t] = 0;
    return;
  }
  const int64_t s = e.links[b], d = e.links[a.B + b];
  const uint32_t mask = HS - 1;
  const uint32_t step = static_cast<uint32_t>(*e.step);
  for (int i = t; i < HS; i += blockDim.x) { keys[i] = -1LL; vals[i] = INT_MAX; }
  __syncthreads();
  if (t == 0) {
    vals[smem_insert(keys, mask, s)] = -2;
    vals[smem_insert(keys, mask, d)] = -3;
    nid[0] = s;
    nid[1] = d;
  }
  __syncthreads();
  int cnt = 2, fb = 0, fe = 2;
  bool trunc = false;
  for (int h = 0; h < e.hops && !trunc && fb < fe; ++h) {
    const int cap = e.caps[h], nf = fe - fb;
    for (int i = t; i < nf; i += blockDim.x) {
      const RowRef r = load_row(e.g, nid[fb + i]);
      int c = r.deg;
      if (cap > 0 && r.deg > cap) {
        // Floyd's uniform cap-subset of the row positions, then sorted into row order
        int32_t* out = e.samp + (static_cast<int64_t>(b) * Nmax + i) * e.cap_max;
        for (int q = 0; q < cap; ++q) {
          const int j = r.deg - cap + q;
          const int pick = static_cast<int>(bounded(seal_nbr_draw(e.seed, step, b, nid[fb + i], q), j + 1u));
          bool dup = false;
          for (int x = 0; x < q; ++x) dup |= out[x] == pick;
          int v = dup ? j : pick, x = q;
          while (x > 0 && out[x - 1] > v) { out[x] = out[x - 1]; --x; }
          out[x] = v;
        }
        c = cap;
      }
      sa[i] = c;
    }
    __syncthreads();
    const int T = block_scan_excl(sa, nf, tmp);
    for (int base = 0; base < T; base += blockDim.x) {
      const int c = base + t;
      int slot = -1;
      int64_t v = -1;
      if (c < T) {
        int lo = 0, hi = nf - 1;                      // the last frontier entry whose candidates start at or before c
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (sa[mid] <= c) lo = mid; else hi = mid - 1;
        }
        const RowRef r = load_row(e.g, nid[fb + lo]);
        int pos = c - sa[lo];
        if (cap > 0 && r.deg > cap) pos = e.samp[(static_cast<int64_t>(b) * Nmax + lo) * e.cap_max + pos];
        v = load_col(e.g, r.part, r.start + pos);
        if (v >= 0 && v < e.num_nodes) {
          slot = smem_insert(keys, mask, v);
          if (slot >= 0) atomicMin(&vals[slot], c);
        }
      }
      __syncthreads();
      const bool first = slot >= 0 && vals[slot] == c;
      int n_new;
      const int rank = block_rank(first, tmp, &n_new);
      if (first && cnt + rank < Nmax) {
        vals[slot] = -(cnt + rank + 2);
        nid[cnt + rank] = v;
      }
      __syncthreads();
      if (cnt + n_new > Nmax) { trunc = true; cnt = Nmax; break; }
      cnt += n_new;
    }
    fb = fe;
    fe = cnt;
  }
  const int n = cnt;
  int64_t* nodes = a.nodes + static_cast<int64_t>(b) * Nmax;
  for (int i = t; i < n; i += blockDim.x) nodes[i] = nid[i];

  // induced edges: count per source, scan, then write in (source, row position) order
  for (int u = w; u < n; u += nw) {
    const RowRef r = load_row(e.g, nid[u]);
    int c = 0;
    for (int j = lane; j < r.deg; j += 32) {
      const int lv = smem_local(keys, vals, mask, load_col(e.g, r.part, r.start + j));
      c += lv >= 0 && !((u == 0 && lv == 1) || (u == 1 && lv == 0));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) sa[u] = c;
  }
  __syncthreads();
  const int e_full = block_scan_excl(sa, n, tmp);
  const int E = min(e_full, Emax);
  int16_t* scol = a.scol + static_cast<int64_t>(b) * Emax;
  int16_t* dcol = a.dcol + static_cast<int64_t>(b) * Emax;
  for (int u = w; u < n; u += nw) {
    const RowRef r = load_row(e.g, nid[u]);
    int base = sa[u];
    for (int j0 = 0; j0 < r.deg && base < Emax; j0 += 32) {
      const int j = j0 + lane;
      int lv = -1;
      if (j < r.deg) lv = smem_local(keys, vals, mask, load_col(e.g, r.part, r.start + j));
      const bool ok = lv >= 0 && !((u == 0 && lv == 1) || (u == 1 && lv == 0));
      const unsigned bal = __ballot_sync(0xffffffffu, ok);
      const int pos = base + __popc(bal & lanemask_lt());
      if (ok && pos < Emax) scol[pos] = static_cast<int16_t>(lv);
      base += __popc(bal);
    }
  }
  for (int i = t; i < n; i += blockDim.x) { sp[i] = min(sa[i], Emax); dp[i] = 0; }
  if (t == 0) sp[n] = E;
  __syncthreads();
  // CSR by destination: stable counting sort, so each destination lists its sources in source order
  for (int i = t; i < E; i += blockDim.x) atomicAdd(&dp[scol[i]], 1);
  __syncthreads();
  block_scan_excl(dp, n, tmp);
  for (int i = t; i < n; i += blockDim.x) sa[i] = dp[i];
  if (t == 0) dp[n] = E;
  __syncthreads();
  if (w == 0) {
    for (int e0 = 0; e0 < E; e0 += 32) {
      const int i = e0 + lane;
      int v = -1, u = 0;
      if (i < E) {
        v = scol[i];
        int lo = 0, hi = n - 1;                       // source: the last u with sp[u] <= i
        while (lo < hi) {
          const int mid = (lo + hi + 1) >> 1;
          if (sp[mid] <= i) lo = mid; else hi = mid - 1;
        }
        u = lo;
      }
      const unsigned grp = __match_any_sync(0xffffffffu, v);
      if (i < E) dcol[sa[v] + __popc(grp & lanemask_lt())] = static_cast<int16_t>(u);
      __syncwarp();
      if (i < E && lane == __ffs(grp) - 1) sa[v] += __popc(grp);
      __syncwarp();
    }
  }
  int32_t* sptr = a.sptr + static_cast<int64_t>(b) * (Nmax + 1);
  int32_t* dptr = a.dptr + static_cast<int64_t>(b) * (Nmax + 1);
  for (int i = t; i <= n; i += blockDim.x) { sptr[i] = sp[i]; dptr[i] = dp[i]; }
  __syncthreads();

  // DRNL: ds from s with d deleted, dd from d with s deleted
  seal_bfs(ds, 0, 1, n, sp, scol, dp, dcol, &flag);
  seal_bfs(dd, 1, 0, n, sp, scol, dp, dcol, &flag);
  int32_t* z = a.z + static_cast<int64_t>(b) * Nmax;
  for (int u = t; u < n; u += blockDim.x) {
    int zz;
    if (u < 2) {
      zz = 1;
    } else if (ds[u] < 0 || dd[u] < 0) {
      zz = 0;
    } else {
      const int D = ds[u] + dd[u], hh = D / 2;
      zz = 1 + min(ds[u], dd[u]) + hh * (hh + D % 2 - 1);
    }
    if (e.max_z >= 0) zz = min(zz, e.max_z);
    z[u] = zz;
  }
  const bool tr = trunc || e_full > Emax;
  if (t == 0) {
    meta[0] = n; meta[1] = E; meta[2] = 1; meta[3] = tr; meta[4] = e_full;
    if (tr) atomicAdd(e.truncated, 1);
  }
}

struct SealSmem {   // forward / backward shared-memory carve-up (floats)
  int stage, dinv, sel, lin, M, dpre2, dM, dC1, total;
};

__host__ __device__ inline SealSmem seal_smem(const SealModel& m, int Nmax) {
  const int Kp = m.k / 2;
  SealSmem s;
  int stage = m.H * m.H;
  if (16 * m.total > stage) stage = 16 * m.total;
  if (32 * 16 * 5 > stage) stage = 32 * 16 * 5;
  s.stage = 0;
  s.dinv = stage;
  s.sel = s.dinv + Nmax;                 // also the sort keys in the forward ([Nmax] after sel)
  s.lin = s.sel + m.k + Nmax;
  s.M = s.lin + kSealLin;                // the forward uses [0, dpre2)
  s.dpre2 = s.M + 16 * Kp;
  s.dM = s.dpre2 + m.dense;
  s.dC1 = s.dM + 16 * Kp;
  s.total = s.dC1 + 16 * m.k;
  return s;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// dinv[v] = (1 + in-edges of v other than self-loops)^-1/2: PyG's gcn_norm with add_remaining_self_loops.
__device__ void seal_dinv(float* dinv, int n, const int32_t* dp, const int16_t* dc) {
  for (int v = threadIdx.x; v < n; v += blockDim.x) {
    int c = 1;
    for (int e = dp[v]; e < dp[v + 1]; ++e) c += dc[e] != v;
    dinv[v] = rsqrtf(static_cast<float>(c));
  }
}

__global__ void __launch_bounds__(kSealThreads) k_seal_forward(SealModel m, SealArenaPtrs a, const float* prm,
                                                               const float* labels, int training, float p_drop,
                                                               uint64_t seed, const int32_t* step_dev) {
  extern __shared__ __align__(16) float fs[];
  __shared__ int nv_s;
  pdl_enter();
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x, lane = t & 31, w = t >> 5;
  const int Nmax = a.max_nodes, H = m.H, T = m.total, k = m.k, Kp = k / 2, T2 = Kp - 4;
  const int32_t* meta = a.meta + b * kSealMeta;
  if (t == 0) nv_s = 0;
  __syncthreads();
  int nv = 0;
  for (int i = t; i < a.B; i += nt) nv += a.meta[i * kSealMeta + 2];
  nv = __reduce_add_sync(0xffffffffu, nv);
  if (lane == 0 && nv) atomicAdd(&nv_s, nv);
  __syncthreads();
  if (!meta[2]) {
    if (t == 0) { a.logits[b] = 0.f; a.lossv[b] = 0.f; a.dlogit[b] = 0.f; }
    return;
  }
  const float inv_nv = 1.f / static_cast<float>(nv_s);
  const SealSmem L = seal_smem(m, Nmax);
  float* Wst = fs + L.stage;
  float* dinv = fs + L.dinv;
  int* sel = reinterpret_cast<int*>(fs + L.sel);
  float* key = fs + L.sel + k;
  float* h1 = fs + L.lin;
  float* M = fs + L.M;
  const int n = meta[0];
  const int32_t* dp = a.dptr + static_cast<int64_t>(b) * (Nmax + 1);
  const int16_t* dc = a.dcol + static_cast<int64_t>(b) * a.max_edges;
  const int32_t* z = a.z + static_cast<int64_t>(b) * Nmax;
  float* X = a.X + static_cast<int64_t>(b) * Nmax * T;
  float* XW = a.XW + static_cast<int64_t>(b) * Nmax * H;
  seal_dinv(dinv, n, dp, dc);
  for (int i = t; i < n * H; i += nt) XW[i] = prm[m.w[0] + static_cast<int64_t>(i % H) * m.Z + min(z[i / H], m.Z - 1)];
  __syncthreads();
  for (int l = 0; l <= m.L; ++l) {
    const int Ho = l < m.L ? H : 1, col = l * H;
    if (l > 0) {
      for (int i = t; i < Ho * H; i += nt) Wst[(i % H) * Ho + i / H] = prm[m.w[l] + i];   // Wst[kk][c] = W[c][kk]
      __syncthreads();
      for (int i = t; i < n * Ho; i += nt) {
        const int u = i / Ho, c = i % Ho;
        const float* xr = X + static_cast<int64_t>(u) * T + (l - 1) * H;
        float acc = 0.f;
        for (int kk = 0; kk < H; ++kk) acc = fmaf(xr[kk], Wst[kk * Ho + c], acc);
        XW[u * H + c] = acc;
      }
      __syncthreads();
    }
    for (int i = t; i < n * Ho; i += nt) {
      const int v = i / Ho, c = i % Ho;
      const float dv = dinv[v];
      float acc = dv * dv * XW[v * H + c];
      for (int q = dp[v]; q < dp[v + 1]; ++q) {
        const int u = dc[q];
        if (u != v) acc = fmaf(dinv[u] * dv, XW[u * H + c], acc);
      }
      X[static_cast<int64_t>(v) * T + col + c] = tanhf(acc + prm[m.bias[l] + c]);
    }
    __syncthreads();
  }
  // sort-pool: top k by the last channel, descending, ties to the lower local id; rows past n are zero
  for (int v = t; v < n; v += nt) key[v] = X[static_cast<int64_t>(v) * T + T - 1];
  for (int r = n + t; r < k; r += nt) sel[r] = -1;
  __syncthreads();
  for (int i = t; i < n; i += nt) {
    const float ki = key[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const float kj = key[j];
      r += kj > ki || (kj == ki && j < i);
    }
    if (r < k) sel[r] = i;
  }
  for (int i = t; i < 16 * T; i += nt) Wst[i] = prm[m.c1w + i];
  __syncthreads();
  for (int r = t; r < k; r += nt) a.sel[static_cast<int64_t>(b) * k + r] = sel[r];
  float* C1 = a.C1 + static_cast<int64_t>(b) * 16 * k;
  for (int i = t; i < 16 * k; i += nt) {
    const int r = i / 16, o = i % 16;
    float acc = prm[m.c1b + o];
    if (sel[r] >= 0) {
      const float* xr = X + static_cast<int64_t>(sel[r]) * T;
      const float* wr = Wst + o * T;
      float s = 0.f;
      for (int q = 0; q < T; ++q) s = fmaf(wr[q], xr[q], s);
      acc += s;
    }
    C1[o * k + r] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  for (int i = t; i < 16 * Kp; i += nt) {
    const int c = i / Kp, r = i % Kp;
    const float x0 = C1[c * k + 2 * r], x1 = C1[c * k + 2 * r + 1];
    M[i] = x1 > x0 ? x1 : x0;
  }
  __syncthreads();
  float* flat = a.flat + static_cast<int64_t>(b) * m.dense;
  for (int i = t; i < 32 * T2; i += nt) {
    const int o = i / T2, tt = i % T2;
    float acc = 0.f;
    for (int c = 0; c < 16; ++c)
      for (int kk = 0; kk < 5; ++kk) acc = fmaf(prm[m.c2w + (o * 16 + c) * 5 + kk], M[c * Kp + tt + kk], acc);
    flat[i] = fmaxf(acc + prm[m.c2b + o], 0.f);
  }
  __syncthreads();
  const uint32_t step = static_cast<uint32_t>(*step_dev);
  for (int j = w; j < kSealLin; j += nt >> 5) {
    const float* wr = prm + m.l1w + static_cast<int64_t>(j) * m.dense;
    float s = 0.f;
    for (int i = lane; i < m.dense; i += 32) s = fmaf(wr[i], flat[i], s);
    s = warp_sum(s);
    if (lane == 0) {
      const float hv = fmaxf(s + prm[m.l1b + j], 0.f);
      float mk = 1.f;
      if (training && p_drop > 0.f) mk = seal_drop_u01(seed, step, b, j) >= p_drop ? 1.f / (1.f - p_drop) : 0.f;
      a.H1[b * kSealLin + j] = hv;
      a.mask[b * kSealLin + j] = mk;
      h1[j] = hv * mk;
    }
  }
  __syncthreads();
  if (w == 0) {
    float s = 0.f;
    for (int j = lane; j < kSealLin; j += 32) s = fmaf(prm[m.l2w + j], h1[j], s);
    s = warp_sum(s);
    if (lane == 0) {
      const float x = s + prm[m.l2b];
      const float y = labels[b];
      a.logits[b] = x;
      a.lossv[b] = (fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x)))) * inv_nv;
      a.dlogit[b] = (1.f / (1.f + expf(-x)) - y) * inv_nv;
    }
  }
}

__global__ void __launch_bounds__(kSealThreads) k_seal_backward(SealModel m, SealArenaPtrs a, const float* prm,
                                                                float* partials) {
  extern __shared__ __align__(16) float fs[];
  pdl_enter();
  const int b = blockIdx.x, t = threadIdx.x, nt = blockDim.x;
  const int Nmax = a.max_nodes, H = m.H, T = m.total, k = m.k, Kp = k / 2, T2 = Kp - 4, dense = m.dense;
  const int32_t* meta = a.meta + b * kSealMeta;
  if (!meta[2]) return;
  const SealSmem L = seal_smem(m, Nmax);
  float* Wst = fs + L.stage;
  float* dinv = fs + L.dinv;
  int* sel = reinterpret_cast<int*>(fs + L.sel);
  float* d1 = fs + L.lin;
  float* dpre2 = fs + L.dpre2;
  float* M = fs + L.M;
  float* dM = fs + L.dM;
  float* dC1 = fs + L.dC1;
  const int n = meta[0];
  float* pp = partials + static_cast<int64_t>(b) * m.P;
  const int32_t* sp = a.sptr + static_cast<int64_t>(b) * (Nmax + 1);
  const int16_t* sc = a.scol + static_cast<int64_t>(b) * a.max_edges;
  const int32_t* dp = a.dptr + static_cast<int64_t>(b) * (Nmax + 1);
  const int16_t* dc = a.dcol + static_cast<int64_t>(b) * a.max_edges;
  const int32_t* z = a.z + static_cast<int64_t>(b) * Nmax;
  const float* X = a.X + static_cast<int64_t>(b) * Nmax * T;
  float* XW = a.XW + static_cast<int64_t>(b) * Nmax * H;
  float* G = a.G + static_cast<int64_t>(b) * Nmax * T;
  const float* C1 = a.C1 + static_cast<int64_t>(b) * 16 * k;
  const float* flat = a.flat + static_cast<int64_t>(b) * dense;
  const float* H1 = a.H1 + b * kSealLin;
  const float* mk = a.mask + b * kSealLin;
  const float g = a.dlogit[b];
  seal_dinv(dinv, n, dp, dc);
  for (int r = t; r < k; r += nt) sel[r] = a.sel[static_cast<int64_t>(b) * k + r];
  for (int j = t; j < kSealLin; j += nt) {
    pp[m.l2w + j] = g * H1[j] * mk[j];
    d1[j] = H1[j] > 0.f ? g * prm[m.l2w + j] * mk[j] : 0.f;
  }
  if (t == 0) pp[m.l2b] = g;
  for (int i = t; i < 16 * Kp; i += nt) {
    const int c = i / Kp, r = i % Kp;
    const float x0 = C1[c * k + 2 * r], x1 = C1[c * k + 2 * r + 1];
    M[i] = x1 > x0 ? x1 : x0;
  }
  __syncthreads();
  for (int i = t; i < kSealLin * dense; i += nt) pp[m.l1w + i] = d1[i / dense] * flat[i % dense];
  for (int j = t; j < kSealLin; j += nt) pp[m.l1b + j] = d1[j];
  for (int i = t; i < dense; i += nt) {
    float s = 0.f;
    for (int j = 0; j < kSealLin; ++j) s = fmaf(d1[j], prm[m.l1w + static_cast<int64_t>(j) * dense + i], s);
    dpre2[i] = flat[i] > 0.f ? s : 0.f;
  }
  __syncthreads();
  for (int o = t; o < 32; o += nt) {
    float s = 0.f;
    for (int tt = 0; tt < T2; ++tt) s += dpre2[o * T2 + tt];
    pp[m.c2b + o] = s;
  }
  for (int i = t; i < 32 * 16 * 5; i += nt) {
    const int o = i / 80, c = (i / 5) % 16, kk = i % 5;
    float s = 0.f;
    for (int tt = 0; tt < T2; ++tt) s = fmaf(dpre2[o * T2 + tt], M[c * Kp + tt + kk], s);
    pp[m.c2w + i] = s;
  }
  for (int i = t; i < 16 * Kp; i += nt) {
    const int c = i / Kp, r = i % Kp;
    float s = 0.f;
    for (int o = 0; o < 32; ++o)
      for (int kk = 0; kk < 5; ++kk) {
        const int tt = r - kk;
        if (tt >= 0 && tt < T2) s = fmaf(dpre2[o * T2 + tt], prm[m.c2w + (o * 16 + c) * 5 + kk], s);
      }
    dM[i] = s;
  }
  __syncthreads();
  // maxpool (first index on a tie) and ReLU
  for (int i = t; i < 16 * k; i += nt) {
    const int c = i / k, r = i % k, q = r / 2;
    float v = 0.f;
    if (q < Kp) {
      const int win = C1[c * k + 2 * q + 1] > C1[c * k + 2 * q] ? 1 : 0;
      if ((r & 1) == win) v = dM[c * Kp + q];
    }
    dC1[i] = C1[i] > 0.f ? v : 0.f;
  }
  for (int i = t; i < n * T; i += nt) G[i] = 0.f;
  __syncthreads();
  for (int o = t; o < 16; o += nt) {
    float s = 0.f;
    for (int r = 0; r < k; ++r) s += dC1[o * k + r];
    pp[m.c1b + o] = s;
  }
  for (int i = t; i < 16 * T; i += nt) {
    const int o = i / T, q = i % T;
    float s = 0.f;
    for (int r = 0; r < k; ++r)
      if (sel[r] >= 0) s = fmaf(dC1[o * k + r], X[static_cast<int64_t>(sel[r]) * T + q], s);
    pp[m.c1w + i] = s;
    Wst[i] = prm[m.c1w + i];
  }
  __syncthreads();
  const int nk = min(n, k);
  for (int i = t; i < nk * T; i += nt) {
    const int r = i / T, q = i % T;
    float s = 0.f;
    for (int o = 0; o < 16; ++o) s = fmaf(dC1[o * k + r], Wst[o * T + q], s);
    G[static_cast<int64_t>(sel[r]) * T + q] = s;
  }
  __syncthreads();
  for (int l = m.L; l >= 0; --l) {
    const int Ho = l < m.L ? H : 1, col = l * H;
    for (int i = t; i < n * Ho; i += nt) {
      const int64_t x = static_cast<int64_t>(i / Ho) * T + col + i % Ho;
      const float y = X[x];
      G[x] *= 1.f - y * y;
    }
    __syncthreads();
    for (int c = t; c < Ho; c += nt) {
      float s = 0.f;
      for (int v = 0; v < n; ++v) s += G[static_cast<int64_t>(v) * T + col + c];
      pp[m.bias[l] + c] = s;
    }
    for (int i = t; i < n * Ho; i += nt) {
      const int u = i / Ho, c = i % Ho;
      const float du = dinv[u];
      float acc = du * du * G[static_cast<int64_t>(u) * T + col + c];
      for (int q = sp[u]; q < sp[u + 1]; ++q) {
        const int v = sc[q];
        if (v != u) acc = fmaf(du * dinv[v], G[static_cast<int64_t>(v) * T + col + c], acc);
      }
      XW[u * H + c] = acc;
    }
    if (l == 0) {
      for (int i = t; i < H * m.Z; i += nt) pp[m.w[0] + i] = 0.f;
    } else {
      for (int i = t; i < Ho * H; i += nt) Wst[i] = prm[m.w[l] + i];
    }
    __syncthreads();
    if (l > 0) {
      for (int i = t; i < Ho * H; i += nt) {
        const int c = i / H, kk = i % H;
        float s = 0.f;
        for (int u = 0; u < n; ++u) s = fmaf(XW[u * H + c], X[static_cast<int64_t>(u) * T + (l - 1) * H + kk], s);
        pp[m.w[l] + i] = s;
      }
      for (int i = t; i < n * H; i += nt) {
        const int u = i / H, kk = i % H;
        float s = 0.f;
        for (int c = 0; c < Ho; ++c) s = fmaf(XW[u * H + c], Wst[c * H + kk], s);
        G[static_cast<int64_t>(u) * T + (l - 1) * H + kk] += s;
      }
      __syncthreads();
    } else {
      // embedding-row gradient of layer 1: column z[u] of W1 (one thread per output channel, nodes in order)
      for (int c = t; c < H; c += nt) {
        float* wr = pp + m.w[0] + static_cast<int64_t>(c) * m.Z;
        for (int u = 0; u < n; ++u) wr[min(z[u], m.Z - 1)] += XW[u * H + c];
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_seal_reduce(const float* partials, const int32_t* meta, int B, int64_t P,
                                                     float* grad, const float* lossv, float* loss) {
  pdl_enter();
  for (int64_t i = blockIdx.x * static_cast<int64_t>(blockDim.x) + threadIdx.x; i < P;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    float s = 0.f;
    for (int b = 0; b < B; ++b)
      if (meta[b * kSealMeta + 2]) s += partials[static_cast<int64_t>(b) * P + i];
    grad[i] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b)
      if (meta[b * kSealMeta + 2]) s += lossv[b];
    *loss = s;
  }
}

template <typename K>
void set_smem(K kernel, size_t bytes) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
}

}  // namespace

size_t seal_extract_smem(int max_nodes) {
  const size_t hs = hash_slots_for(max_nodes);
  return hs * 12 + static_cast<size_t>(max_nodes) * 8 + 3 * static_cast<size_t>(max_nodes + 1) * 4 +
         2 * static_cast<size_t>(max_nodes) * 2;
}

size_t seal_forward_smem(const SealModel& m, int max_nodes) {
  return static_cast<size_t>(seal_smem(m, max_nodes).dpre2) * 4;
}

size_t seal_backward_smem(const SealModel& m, int max_nodes) {
  return static_cast<size_t>(seal_smem(m, max_nodes).total) * 4;
}

void launch_seal_extract(const SealExtractArgs& e, const SealArenaPtrs& a, cudaStream_t s) {
  const size_t smem = seal_extract_smem(a.max_nodes);
  set_smem(k_seal_extract, smem);
  launch_k(k_seal_extract, dim3(a.B), dim3(kSealThreads), smem, s, e, a);
}

void launch_seal_forward(const SealModel& m, const SealArenaPtrs& a, const float* prm, const float* labels,
                         int training, float p_drop, uint64_t seed, const int32_t* step, cudaStream_t s) {
  const size_t smem = seal_forward_smem(m, a.max_nodes);
  set_smem(k_seal_forward, smem);
  launch_k(k_seal_forward, dim3(a.B), dim3(kSealThreads), smem, s, m, a, prm, labels, training, p_drop, seed, step);
}

void launch_seal_backward(const SealModel& m, const SealArenaPtrs& a, const float* prm, float* partials,
                          cudaStream_t s) {
  const size_t smem = seal_backward_smem(m, a.max_nodes);
  set_smem(k_seal_backward, smem);
  launch_k(k_seal_backward, dim3(a.B), dim3(kSealThreads), smem, s, m, a, prm, partials);
}

void launch_seal_reduce(const SealModel& m, const SealArenaPtrs& a, const float* partials, float* grad, float* loss,
                        cudaStream_t s) {
  launch_k(k_seal_reduce, dim3(grid_for(m.P, 256, 132 * 4)), dim3(256), 0, s, partials, a.meta, a.B, m.P, grad,
           a.lossv, loss);
}

}  // namespace glt
