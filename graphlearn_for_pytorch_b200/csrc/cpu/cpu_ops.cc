// CPU reference implementations of every graph op of the engine.
//
// These are the ground truth the sm_90a kernels are tested against (same
// Philox streams => identical samples), and the fallback used when a Graph is
// created with mode='CPU'.  Capability parity with the reference's csrc/cpu/*
// (random_sampler.cc, weighted_sampler.cc, random_negative_sampler.cc,
// inducer.cc, subgraph_op.cc, stitch_sample_results.cc) -- re-designed around
// counter-based RNG, flat hash tables and no stack VLAs.
#include <ATen/Parallel.h>
#include <torch/extension.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <numeric>
#include <vector>

#include "../philox.h"
#include "cpu_ops.h"
#include "parallel.h"

namespace glt {

using torch::Tensor;

// One message argument per TORCH_CHECK (see fmt in bindings.cc): the message is built first.
static inline void check_i64(const Tensor& t, const char* name) {
  TORCH_CHECK(t.device().is_cpu(), std::string(name) + " must be a CPU tensor");
  TORCH_CHECK(t.scalar_type() == torch::kInt64, std::string(name) + " must be int64");
  TORCH_CHECK(t.is_contiguous(), std::string(name) + " must be contiguous");
}

// ----------------------------------------------------------------------------
// Row gather on the host: out[pos[i]] = table[map(ids[i])], map = id2index lookup or `- offset`.
// One fused pass (no temporary for the gathered rows, no second scatter pass), rows moved with memcpy, split over
// the intra-op thread pool; ids out of range raise instead of reading out of bounds.
// (The reference indexes with torch on the host: python/data/feature.py:158-165.)
// ----------------------------------------------------------------------------
void cpu_gather_rows(const Tensor& table, const Tensor& ids, const c10::optional<Tensor>& id2index, int64_t offset,
                     Tensor out, const c10::optional<Tensor>& pos) {
  check_i64(ids, "ids");
  TORCH_CHECK(table.device().is_cpu() && out.device().is_cpu(), "cpu_gather_rows: host tensors only");
  TORCH_CHECK(table.dim() >= 1 && table.is_contiguous() && out.is_contiguous(), "cpu_gather_rows: contiguous tensors");
  TORCH_CHECK(table.scalar_type() == out.scalar_type(), "cpu_gather_rows: dtype mismatch");
  const int64_t n = ids.numel();
  const int64_t rows = table.size(0), out_rows = out.dim() ? out.size(0) : 0;
  const int64_t row_bytes = rows ? (int64_t)(table.nbytes() / rows) : 0;
  TORCH_CHECK(out_rows == 0 || (int64_t)(out.nbytes() / out_rows) == row_bytes || row_bytes == 0,
              "cpu_gather_rows: row width mismatch");
  const int64_t* id = ids.data_ptr<int64_t>();
  const int64_t* map = nullptr;
  int64_t map_n = 0;
  if (id2index.has_value() && id2index->defined()) {
    check_i64(*id2index, "id2index");
    map = id2index->data_ptr<int64_t>();
    map_n = id2index->numel();
  }
  const int64_t* ps = nullptr;
  if (pos.has_value() && pos->defined()) {
    check_i64(*pos, "pos");
    TORCH_CHECK(pos->numel() == n, "cpu_gather_rows: pos/ids size mismatch");
    ps = pos->data_ptr<int64_t>();
  } else {
    TORCH_CHECK(out_rows >= n, "cpu_gather_rows: out too small");
  }
  const char* src = static_cast<const char*>(table.data_ptr());
  char* dst = static_cast<char*>(out.data_ptr());
  std::atomic<int> bad{0};
  glt::parallel_for(0, n, 2048, [&](int64_t lo, int64_t hi) {
    for (int64_t i = lo; i < hi; ++i) {
      int64_t v = id[i];
      int64_t r;
      if (map) {
        if (v < 0 || v >= map_n) { bad.store(1); continue; }
        r = map[v];
      } else {
        r = v - offset;
      }
      const int64_t o = ps ? ps[i] : i;
      if (r < 0 || r >= rows || o < 0 || o >= out_rows) { bad.store(1); continue; }
      if (i + 4 < hi) {   // rows are random: start the miss of a later row early
        const int64_t v2 = id[i + 4];
        const int64_t r2 = map ? ((v2 >= 0 && v2 < map_n) ? map[v2] : -1) : v2 - offset;
        if (r2 >= 0 && r2 < rows) __builtin_prefetch(src + r2 * row_bytes);
      }
      std::memcpy(dst + o * row_bytes, src + r * row_bytes, (size_t)row_bytes);
    }
  });
  TORCH_CHECK(bad.load() == 0, "cpu_gather_rows: id / row / output position out of range");
}

// ----------------------------------------------------------------------------
// COO -> CSR (counting sort by row, optional per-row column sort).
// Replaces the reference's torch_sparse dependency (utils/topo.py:29-91).
// ----------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor, Tensor> coo_to_csr(
    const Tensor& rows, const Tensor& cols, const c10::optional<Tensor>& eids,
    const c10::optional<Tensor>& weights, int64_t num_rows, bool sort_cols) {
  check_i64(rows, "rows");
  check_i64(cols, "cols");
  const int64_t E = rows.numel();
  TORCH_CHECK(cols.numel() == E, "rows/cols size mismatch");
  const int64_t* r = rows.data_ptr<int64_t>();
  const int64_t* c = cols.data_ptr<int64_t>();
  if (num_rows < 0) {
    num_rows = 0;
    for (int64_t i = 0; i < E; ++i) num_rows = std::max(num_rows, r[i] + 1);
  }
  Tensor indptr = torch::zeros({num_rows + 1}, torch::kInt64);
  int64_t* ip = indptr.data_ptr<int64_t>();
  // Large inputs: the histogram and the bucket scatter -- the two passes with random accesses -- are split by ROW
  // RANGE over T threads.  Every thread streams the whole row array (sequential reads are cheap) and touches only
  // the counters / output slots of its own rows, so there is nothing to merge, the accessed slice of `indptr` /
  // `perm` shrinks to 1/T (cache-resident counters), and edges keep their input order inside a row exactly as in
  // the serial pass.
  const int64_t T = std::min<int64_t>(at::get_num_threads(), 16);
  const bool par = T > 1 && E >= (int64_t(1) << 20) && num_rows >= T && !at::in_parallel_region();
  if (par) {
    std::atomic<bool> bad{false};
    glt::parallel_for(0, E, int64_t(1) << 18, [&](int64_t b, int64_t e) {
      for (int64_t i = b; i < e; ++i)
        if (r[i] < 0 || r[i] >= num_rows) { bad.store(true, std::memory_order_relaxed); return; }
    });
    TORCH_CHECK(!bad.load(), "row id out of range");
    glt::parallel_for(0, T, 1, [&](int64_t tb, int64_t te) {
      for (int64_t t = tb; t < te; ++t) {
        const int64_t lo = num_rows * t / T, hi = num_rows * (t + 1) / T;
        const uint64_t span = (uint64_t)(hi - lo);
        for (int64_t i = 0; i < E; ++i) {
          const int64_t row = r[i];
          if ((uint64_t)(row - lo) < span) ip[row + 1]++;
        }
      }
    });
  } else {
    for (int64_t i = 0; i < E; ++i) {
      TORCH_CHECK(r[i] >= 0 && r[i] < num_rows, "row id out of range");
      ip[r[i] + 1]++;
    }
  }
  for (int64_t i = 0; i < num_rows; ++i) ip[i + 1] += ip[i];
  // perm[pos] = original edge position
  std::vector<int64_t> perm(E);
  {
    std::vector<int64_t> cursor(ip, ip + num_rows);
    if (par) {
      std::vector<int64_t> bound(T + 1, num_rows);      // row ranges holding ~E/T edges each
      bound[0] = 0;
      for (int64_t t = 1; t < T; ++t) {
        const int64_t at_edge = E / T * t;
        int64_t row = std::lower_bound(ip, ip + num_rows + 1, at_edge) - ip;
        bound[t] = std::min(std::max(row, bound[t - 1]), num_rows);
      }
      int64_t* cur = cursor.data();
      int64_t* pm = perm.data();
      glt::parallel_for(0, T, 1, [&](int64_t tb, int64_t te) {
        for (int64_t t = tb; t < te; ++t) {
          const int64_t lo = bound[t], hi = bound[t + 1];
          if (lo >= hi) continue;
          const uint64_t span = (uint64_t)(hi - lo);
          for (int64_t i = 0; i < E; ++i) {
            const int64_t row = r[i];
            if ((uint64_t)(row - lo) < span) pm[cur[row]++] = i;
          }
        }
      });
    } else {
      for (int64_t i = 0; i < E; ++i) perm[cursor[r[i]]++] = i;
    }
  }
  if (sort_cols) {
    glt::parallel_for(0, num_rows, 1024, [&](int64_t b, int64_t e) {
      for (int64_t v = b; v < e; ++v) {
        std::stable_sort(perm.begin() + ip[v], perm.begin() + ip[v + 1],
                         [&](int64_t a, int64_t bb) { return c[a] < c[bb]; });
      }
    });
  }
  Tensor indices = torch::empty({E}, torch::kInt64);
  Tensor out_eids = torch::empty({E}, torch::kInt64);
  int64_t* ind = indices.data_ptr<int64_t>();
  int64_t* oe = out_eids.data_ptr<int64_t>();
  const int64_t* ie = nullptr;
  if (eids.has_value() && eids->defined()) {
    check_i64(*eids, "eids");
    ie = eids->data_ptr<int64_t>();
  }
  Tensor out_w;
  const float* iw = nullptr;
  float* ow = nullptr;
  Tensor w32;
  if (weights.has_value() && weights->defined()) {
    w32 = weights->to(torch::kFloat32).contiguous();
    iw = w32.data_ptr<float>();
    out_w = torch::empty({E}, torch::kFloat32);
    ow = out_w.data_ptr<float>();
  }
  glt::parallel_for(0, E, 1 << 16, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) {
      int64_t p = perm[i];
      ind[i] = c[p];
      oe[i] = ie ? ie[p] : p;
      if (ow) ow[i] = iw[p];
    }
  });
  return {indptr, indices, out_eids, out_w};
}

// ----------------------------------------------------------------------------
// Uniform neighbour sampling (Floyd k-subset, without replacement by default).
// Reference semantics: csrc/cpu/random_sampler.cc:26-153 (req_num<0 => all).
// ----------------------------------------------------------------------------
// Rows per parallel chunk of the uniform sampler: a row costs about k random reads (k < 0: its whole adjacency), and
// a chunk has to be worth far more than starting a thread (tens of microseconds).
static inline int64_t sample_grain(int64_t k) {
  return std::max<int64_t>(256, 32768 / std::max<int64_t>(k < 0 ? 32 : k, 1));
}

static inline int64_t row_degree(const int64_t* ip, int64_t num_rows, int64_t v) {
  // Ids beyond the local CSR have no neighbours (partition shards only cover
  // rows up to their max local src id; reference random_sampler.cu:45-50).
  if (v < 0 || v >= num_rows) return 0;
  return ip[v + 1] - ip[v];
}

std::tuple<Tensor, Tensor, Tensor> cpu_sample_neighbors(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& seeds, int64_t k, bool with_edge, bool replace, int64_t seed,
    int64_t stream) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  check_i64(seeds, "seeds");
  const int64_t num_rows = indptr.numel() - 1;
  const int64_t bs = seeds.numel();
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t* sd = seeds.data_ptr<int64_t>();
  const int64_t* ei = nullptr;
  if (with_edge) {
    TORCH_CHECK(eids.has_value() && eids->defined(), "with_edge needs edge ids");
    check_i64(*eids, "eids");
    ei = eids->data_ptr<int64_t>();
  }
  Tensor counts = torch::empty({bs}, torch::kInt64);
  int64_t* cnt = counts.data_ptr<int64_t>();
  std::vector<int64_t> offs(bs + 1, 0);
  glt::parallel_for(0, bs, 16384, [&](int64_t b, int64_t e) {   // degree reads are random: spread the misses
    for (int64_t i = b; i < e; ++i) {
      int64_t d = row_degree(ip, num_rows, sd[i]);
      cnt[i] = (k < 0) ? d : (replace ? (d > 0 ? k : 0) : std::min(d, k));
      if (replace && k >= 0 && d <= k) cnt[i] = d;  // small rows are copied
    }
  });
  for (int64_t i = 0; i < bs; ++i) offs[i + 1] = offs[i] + cnt[i];
  Tensor nbrs = torch::empty({offs[bs]}, torch::kInt64);
  Tensor out_e = with_edge ? torch::empty({offs[bs]}, torch::kInt64) : Tensor();
  int64_t* nb = nbrs.data_ptr<int64_t>();
  int64_t* oe = with_edge ? out_e.data_ptr<int64_t>() : nullptr;
  glt::parallel_for(0, bs, sample_grain(k), [&](int64_t b, int64_t e) {
    std::vector<uint32_t> chosen;
    for (int64_t i = b; i < e; ++i) {
      const int64_t v = sd[i];
      const int64_t d = row_degree(ip, num_rows, v);
      if (d == 0) continue;
      const int64_t start = ip[v];
      int64_t* o = nb + offs[i];
      if (k < 0 || d <= k) {
        std::memcpy(o, ind + start, sizeof(int64_t) * d);
        if (oe) std::memcpy(oe + offs[i], ei + start, sizeof(int64_t) * d);
        continue;
      }
      if (replace) {
        for (int64_t j = 0; j < k; ++j) {
          uint32_t t = bounded(philox_draw(seed, stream, v, j), (uint32_t)d);
          o[j] = ind[start + t];
          if (oe) oe[offs[i] + j] = ei[start + t];
        }
        continue;
      }
      chosen.assign(k, 0);
      for (int64_t j = 0; j < k; ++j) {
        uint32_t t = floyd_candidate(seed, stream, v, j, (uint32_t)d, (uint32_t)k);
        bool dup = false;
        for (int64_t q = 0; q < j; ++q) dup |= (chosen[q] == t);
        uint32_t pick = dup ? (uint32_t)(d - k + j) : t;
        chosen[j] = pick;
        o[j] = ind[start + pick];
        if (oe) oe[offs[i] + j] = ei[start + pick];
      }
    }
  });
  return {nbrs, counts, out_e};
}

// ----------------------------------------------------------------------------
// Weighted neighbour sampling; a row of degree d <= k (or k < 0) is copied whole.
//   replace=false: a weighted k-subset by exponential race (Efraimidis-Spirakis):
//     key_j = -log(u_j)/w_j, keep the k smallest keys.  Zero-weight neighbours
//     come last, in position order, when fewer than k weights are positive.
//   replace=true: k independent draws, neighbour j with probability w_j / W
//     (the reference's std::discrete_distribution, weighted_sampler.cc:147-165).
//     Draw i inverts the row's CDF at u_i * W with u_i from Philox counter i;
//     a row whose weights are all 0 picks nothing (count 0).
// The reference has no GPU implementation (weighted_sampler.cuh:28-36); both
// formulations run on the GPU as well (cuda/sampling.cu pick_positions).
// ----------------------------------------------------------------------------
// Running sums of a row's weights in position order (fp64, as on the GPU); returns the row's total.
static inline double weight_prefix(const float* w, int64_t d, std::vector<double>& cdf) {
  cdf.resize(d);
  double s = 0.0;
  for (int64_t j = 0; j < d; ++j) cdf[j] = (s += w[j]);
  return s;
}

static inline bool any_positive(const float* w, int64_t d) {
  return std::any_of(w, w + d, [](float x) { return x > 0.f; });
}

std::tuple<Tensor, Tensor, Tensor> cpu_sample_neighbors_weighted(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& weights, const Tensor& seeds, int64_t k, bool with_edge,
    int64_t seed, int64_t stream, bool replace) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  check_i64(seeds, "seeds");
  TORCH_CHECK(weights.scalar_type() == torch::kFloat32 && weights.is_contiguous(),
              "weights must be contiguous float32");
  const int64_t num_rows = indptr.numel() - 1;
  const int64_t bs = seeds.numel();
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t* sd = seeds.data_ptr<int64_t>();
  const float* w = weights.data_ptr<float>();
  const int64_t* ei = nullptr;
  if (with_edge) {
    TORCH_CHECK(eids.has_value() && eids->defined(), "with_edge needs edge ids");
    ei = eids->data_ptr<int64_t>();
  }
  Tensor counts = torch::empty({bs}, torch::kInt64);
  int64_t* cnt = counts.data_ptr<int64_t>();
  std::vector<int64_t> offs(bs + 1, 0);
  glt::parallel_for(0, bs, 16384, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) {
      const int64_t v = sd[i];
      const int64_t d = row_degree(ip, num_rows, v);
      cnt[i] = (k < 0) ? d : std::min(d, k);
      if (replace && k >= 0 && d > k && !any_positive(w + ip[v], d)) cnt[i] = 0;
    }
  });
  for (int64_t i = 0; i < bs; ++i) offs[i + 1] = offs[i] + cnt[i];
  Tensor nbrs = torch::empty({offs[bs]}, torch::kInt64);
  Tensor out_e = with_edge ? torch::empty({offs[bs]}, torch::kInt64) : Tensor();
  int64_t* nb = nbrs.data_ptr<int64_t>();
  int64_t* oe = with_edge ? out_e.data_ptr<int64_t>() : nullptr;
  glt::parallel_for(0, bs, 256, [&](int64_t b, int64_t e) {
    std::vector<std::pair<float, int64_t>> keys;
    std::vector<double> cdf;
    for (int64_t i = b; i < e; ++i) {
      const int64_t v = sd[i];
      const int64_t d = row_degree(ip, num_rows, v);
      if (d == 0 || cnt[i] == 0) continue;
      const int64_t start = ip[v];
      int64_t* o = nb + offs[i];
      if (k < 0 || d <= k) {
        std::memcpy(o, ind + start, sizeof(int64_t) * d);
        if (oe) std::memcpy(oe + offs[i], ei + start, sizeof(int64_t) * d);
        continue;
      }
      if (replace) {
        const double total = weight_prefix(w + start, d, cdf);
        int64_t last = d - 1;
        while (!(w[start + last] > 0.f)) --last;   // cnt > 0: some weight is positive
        for (int64_t j = 0; j < k; ++j) {
          const double target = static_cast<double>(u01(philox_draw(seed, stream, v, (uint32_t)j))) * total;
          // first running sum above the target (sums are non-decreasing, so it sits on a positive weight)
          int64_t t = std::upper_bound(cdf.begin(), cdf.end(), target) - cdf.begin();
          if (t > last) t = last;
          o[j] = ind[start + t];
          if (oe) oe[offs[i] + j] = ei[start + t];
        }
        continue;
      }
      keys.resize(d);
      for (int64_t j = 0; j < d; ++j) {
        keys[j] = {weighted_key(seed, stream, v, (uint32_t)j, w[start + j]), j};
      }
      std::partial_sort(keys.begin(), keys.begin() + k, keys.end());
      for (int64_t j = 0; j < k; ++j) {
        o[j] = ind[start + keys[j].second];
        if (oe) oe[offs[i] + j] = ei[start + keys[j].second];
      }
    }
  });
  return {nbrs, counts, out_e};
}

// ----------------------------------------------------------------------------
// IdTable: global id -> dense local id, first-seen order, persistent across
// hops.  One table per node type gives the hetero inducer.  (Reference:
// csrc/cpu/inducer.cc:25-181 keeps unordered_map<int64,int32> per type.)
// ----------------------------------------------------------------------------
static inline uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33;
  return x;
}

// Slots pack {key, local id, generation} into 16 bytes (one cache line touch per probe); a slot is live only when
// its generation equals the table's, so reset() is O(1) and a table can be recycled batch after batch
// (ops/tables.py keeps a small pool): clearing a worst-case table for every batch used to cost as much as the
// inserts themselves.  The first allocation is bounded (1 << 22 slots = 64 MB); the table doubles when it fills.
static constexpr int64_t kInitialSlotsMax = int64_t(1) << 22;

CpuIdTable::CpuIdTable(int64_t capacity_hint) {
  rehash(std::min<int64_t>(std::max<int64_t>(64, capacity_hint * 2), kInitialSlotsMax));
}

void CpuIdTable::rehash(int64_t min_slots) {
  int64_t cap = 64;
  while (cap < min_slots) cap <<= 1;
  slots_.assign(cap, Slot{0, 0, 0});
  gen_ = 1;
  mask_ = cap - 1;
  for (int64_t i = 0; i < (int64_t)keys_.size(); ++i) {
    uint64_t p = mix64((uint64_t)keys_[i]) & mask_;
    while (slots_[p].gen == gen_) p = (p + 1) & mask_;
    slots_[p] = Slot{keys_[i], (int32_t)i, gen_};
  }
}

void CpuIdTable::reset() {
  keys_.clear();
  if (++gen_ == 0) {   // generation counter wrapped: really clear once every 2^32 resets
    std::fill(slots_.begin(), slots_.end(), Slot{0, 0, 0});
    gen_ = 1;
  }
}

int64_t CpuIdTable::insert_one(int64_t key) {
  if ((int64_t)(keys_.size() + 1) * 2 > (int64_t)slots_.size()) rehash(slots_.size() * 2);
  uint64_t p = mix64((uint64_t)key) & mask_;
  while (true) {
    Slot& s = slots_[p];
    if (s.gen != gen_) {
      TORCH_CHECK(keys_.size() < (size_t)INT32_MAX, "IdTable: more than 2^31 distinct ids");
      s = Slot{key, (int32_t)keys_.size(), gen_};
      keys_.push_back(key);
      return s.val;
    }
    if (s.key == key) return s.val;
    p = (p + 1) & mask_;
  }
}

int64_t CpuIdTable::find_one(int64_t key) const {
  uint64_t p = mix64((uint64_t)key) & mask_;
  while (true) {
    const Slot& s = slots_[p];
    if (s.gen != gen_) return -1;
    if (s.key == key) return s.val;
    p = (p + 1) & mask_;
  }
}

Tensor CpuIdTable::insert(const Tensor& keys) {
  check_i64(keys, "keys");
  Tensor out = torch::empty_like(keys);
  const int64_t* k = keys.data_ptr<int64_t>();
  int64_t* o = out.data_ptr<int64_t>();
  const int64_t n = keys.numel();
  // Kept serial on purpose: with the home slots prefetched a dozen keys ahead one thread sustains ~18 ns per key on
  // a 32 MB table, and an owner-partitioned parallel version (measured on 8 vCPUs) lost more in its extra passes
  // (partitioning, first-seen id assignment, id patch-up) than the probes gained.
  constexpr int64_t kAhead = 12;   // the home slot of a later key is a random line: start its miss early
  for (int64_t i = 0; i < n; ++i) {
    if (i + kAhead < n && k[i + kAhead] >= 0)
      __builtin_prefetch(&slots_[mix64((uint64_t)k[i + kAhead]) & mask_], 1);
    o[i] = (k[i] < 0) ? -1 : insert_one(k[i]);
  }
  return out;
}

Tensor CpuIdTable::lookup(const Tensor& keys) const {
  check_i64(keys, "keys");
  Tensor out = torch::empty_like(keys);
  const int64_t* k = keys.data_ptr<int64_t>();
  int64_t* o = out.data_ptr<int64_t>();
  glt::parallel_for(0, keys.numel(), 8192, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) o[i] = find_one(k[i]);
  });
  return out;
}

Tensor CpuIdTable::keys(int64_t from) const {
  from = std::min<int64_t>(std::max<int64_t>(from, 0), keys_.size());
  Tensor out = torch::empty({(int64_t)keys_.size() - from}, torch::kInt64);
  std::memcpy(out.data_ptr<int64_t>(), keys_.data() + from, sizeof(int64_t) * out.numel());
  return out;
}

// ----------------------------------------------------------------------------
// Negative sampling.  Reference: csrc/cpu/random_negative_sampler.cc:26-83.
// Row and column draws use independent Philox words (the reference's CUDA
// path correlates them, random_negative_sampler.cu:69-70).
// ----------------------------------------------------------------------------
static inline bool edge_in_row(const int64_t* ind, int64_t b, int64_t e, int64_t c, bool sorted) {
  if (sorted) return std::binary_search(ind + b, ind + e, c);
  for (int64_t i = b; i < e; ++i)
    if (ind[i] == c) return true;
  return false;
}

std::tuple<Tensor, Tensor> cpu_negative_sample(
    const Tensor& indptr, const Tensor& indices, int64_t num_rows, int64_t num_cols,
    int64_t req, int64_t trials, bool padding, bool sorted, int64_t seed, int64_t stream) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t csr_rows = indptr.numel() - 1;
  if (num_rows <= 0) num_rows = csr_rows;
  TORCH_CHECK(num_cols > 0, "num_cols must be positive");
  std::vector<int64_t> r(req), c(req);
  std::vector<uint8_t> ok(req, 0);
  // The membership test of a candidate is two dependent cache misses (indptr[row], then the row's column list) on
  // a graph far larger than the caches.  Candidates are therefore handled in groups of 16: draw all, prefetch their
  // indptr entries, prefetch their column lists, then search -- the misses of a group overlap instead of
  // serialising.  Draw (i, t) is the same Philox value as in a one-at-a-time loop, so results do not depend on the
  // grouping or on the thread count.
  constexpr int64_t G = 16;
  glt::parallel_for(0, req, 2048, [&](int64_t b, int64_t e) {
    int64_t rr[G], cc[G];
    for (int64_t g0 = b; g0 < e; g0 += G) {
      const int64_t gn = std::min<int64_t>(G, e - g0);
      for (int64_t t = 0; t < trials; ++t) {
        bool any = false;
        for (int64_t j = 0; j < gn; ++j) {
          const int64_t i = g0 + j;
          if (ok[i]) continue;
          any = true;
          rr[j] = bounded(philox_draw(seed, stream, i, 2 * t), (uint32_t)num_rows);
          cc[j] = bounded(philox_draw(seed, stream, i, 2 * t + 1), (uint32_t)num_cols);
          if (rr[j] < csr_rows) __builtin_prefetch(ip + rr[j]);
        }
        if (!any) break;
        for (int64_t j = 0; j < gn; ++j) {
          if (ok[g0 + j] || rr[j] >= csr_rows) continue;
          const int64_t lo = ip[rr[j]], hi = ip[rr[j] + 1];
          if (hi > lo) {
            __builtin_prefetch(ind + lo);
            __builtin_prefetch(ind + lo + (hi - lo) / 2);
          }
        }
        for (int64_t j = 0; j < gn; ++j) {
          const int64_t i = g0 + j;
          if (ok[i]) continue;
          bool hit = rr[j] < csr_rows && edge_in_row(ind, ip[rr[j]], ip[rr[j] + 1], cc[j], sorted);
          if (!hit) { r[i] = rr[j]; c[i] = cc[j]; ok[i] = 1; }
        }
      }
      if (padding) {
        for (int64_t i = g0; i < g0 + gn; ++i) {
          if (ok[i]) continue;
          // non-strict fill, same as the reference's padding pass (:63-67)
          r[i] = bounded(philox_draw(seed, stream + 0x40000000u, i, 0), (uint32_t)num_rows);
          c[i] = bounded(philox_draw(seed, stream + 0x40000000u, i, 1), (uint32_t)num_cols);
          ok[i] = 1;
        }
      }
    }
  });
  int64_t n = 0;
  for (int64_t i = 0; i < req; ++i) n += ok[i];
  Tensor rows = torch::empty({n}, torch::kInt64), cols = torch::empty({n}, torch::kInt64);
  int64_t* pr = rows.data_ptr<int64_t>();
  int64_t* pc = cols.data_ptr<int64_t>();
  for (int64_t i = 0, j = 0; i < req; ++i)
    if (ok[i]) { pr[j] = r[i]; pc[j] = c[i]; ++j; }
  return {rows, cols};
}

// ----------------------------------------------------------------------------
// Induced subgraph on a node set.  Reference: csrc/cpu/subgraph_op.cc:61-89.
// ----------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor, Tensor> cpu_node_subgraph(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& srcs, bool with_edge) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  check_i64(srcs, "srcs");
  const int64_t num_rows = indptr.numel() - 1;
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t* ei = nullptr;
  if (with_edge) {
    TORCH_CHECK(eids.has_value() && eids->defined(), "with_edge needs edge ids");
    ei = eids->data_ptr<int64_t>();
  }
  CpuIdTable table(srcs.numel());
  table.insert(srcs);
  Tensor nodes = table.keys(0);
  const int64_t n = nodes.numel();
  const int64_t* nd = nodes.data_ptr<int64_t>();
  std::vector<int64_t> cnt(n + 1, 0);
  glt::parallel_for(0, n, 1024, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) {
      int64_t v = nd[i], c = 0;
      if (v >= 0 && v < num_rows)
        for (int64_t p = ip[v]; p < ip[v + 1]; ++p) c += table.find_one(ind[p]) >= 0;
      cnt[i + 1] = c;
    }
  });
  for (int64_t i = 0; i < n; ++i) cnt[i + 1] += cnt[i];
  Tensor rows = torch::empty({cnt[n]}, torch::kInt64), cols = torch::empty({cnt[n]}, torch::kInt64);
  Tensor oe = with_edge ? torch::empty({cnt[n]}, torch::kInt64) : Tensor();
  int64_t* pr = rows.data_ptr<int64_t>();
  int64_t* pc = cols.data_ptr<int64_t>();
  int64_t* pe = with_edge ? oe.data_ptr<int64_t>() : nullptr;
  glt::parallel_for(0, n, 1024, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) {
      int64_t v = nd[i], o = cnt[i];
      if (v < 0 || v >= num_rows) continue;
      for (int64_t p = ip[v]; p < ip[v + 1]; ++p) {
        int64_t l = table.find_one(ind[p]);
        if (l >= 0) {
          pr[o] = i; pc[o] = l;
          if (pe) pe[o] = ei[p];
          ++o;
        }
      }
    }
  });
  return {nodes, rows, cols, oe};
}

// ----------------------------------------------------------------------------
// Random walks (uniform / node2vec p,q by rejection, philox.h).  New functionality:
// the reference only declares SamplingType.RANDOM_WALK (sampler/base.py:335).
// Same draws and the same float accept test as k_random_walk, so the planes'
// walks are bit-identical.  A walker on a node without out-edges stays in place.
// ----------------------------------------------------------------------------
Tensor cpu_random_walk(const Tensor& indptr, const Tensor& indices, const Tensor& starts,
                       int64_t walk_length, double p, double q, int64_t seed, int64_t stream) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  check_i64(starts, "starts");
  TORCH_CHECK(walk_length >= 0, "random_walk: walk_length must be >= 0");
  Node2VecWeights nw;
  const char* bad = node2vec_weights(p, q, &nw);
  TORCH_CHECK(bad == nullptr, std::string("random_walk: ") + (bad ? bad : ""));
  const int64_t num_rows = indptr.numel() - 1;
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t* st = starts.data_ptr<int64_t>();
  const int64_t n = starts.numel();
  Tensor out = torch::empty({n, walk_length + 1}, torch::kInt64);
  int64_t* o = out.data_ptr<int64_t>();
  const bool biased = !(p == 1.0 && q == 1.0);
  glt::parallel_for(0, n, 512, [&](int64_t b, int64_t e) {
    for (int64_t i = b; i < e; ++i) {
      int64_t cur = st[i], prev = -1;
      o[i * (walk_length + 1)] = cur;
      uint32_t draw = 0;
      for (int64_t s = 1; s <= walk_length; ++s) {
        int64_t d = row_degree(ip, num_rows, cur);
        int64_t nxt = cur;
        if (d > 0) {
          if (!biased || prev < 0) {
            nxt = ind[ip[cur] + bounded(philox_draw(seed, stream, i, draw++), (uint32_t)d)];
          } else {
            const int64_t pd = row_degree(ip, num_rows, prev);
            for (int tries = 0; tries < kNode2VecMaxProposals; ++tries) {
              nxt = ind[ip[cur] + bounded(philox_draw(seed, stream, i, draw++), (uint32_t)d)];
              const float u = u01(philox_draw(seed, stream, i, draw++));
              if (node2vec_accept(nw, nxt == prev, u,
                                  [&] { return pd > 0 && edge_in_row(ind, ip[prev], ip[prev] + pd, nxt, false); }))
                break;
            }
          }
        }
        o[i * (walk_length + 1) + s] = nxt;
        prev = cur;
        cur = nxt;
      }
    }
  });
  return out;
}

// ----------------------------------------------------------------------------
// Stitch per-partition one-hop results back into seed order (only needed by
// the RPC/CPU deployment mode; the P2P kernels write each seed's slot in
// place).  Reference: csrc/cpu/stitch_sample_results.cc:24-85.
// ----------------------------------------------------------------------------
std::tuple<Tensor, Tensor, Tensor> cpu_stitch(
    int64_t num_seeds, const std::vector<Tensor>& idx_list, const std::vector<Tensor>& nbrs_list,
    const std::vector<Tensor>& nbrs_num_list, const std::vector<Tensor>& eids_list) {
  const size_t P = idx_list.size();
  TORCH_CHECK(nbrs_list.size() == P && nbrs_num_list.size() == P, "partition list mismatch");
  const bool with_edge = eids_list.size() == P && P > 0;
  Tensor counts = torch::zeros({num_seeds}, torch::kInt64);
  int64_t* cnt = counts.data_ptr<int64_t>();
  for (size_t p = 0; p < P; ++p) {
    check_i64(idx_list[p], "idx");
    check_i64(nbrs_num_list[p], "nbrs_num");
    const int64_t* ix = idx_list[p].data_ptr<int64_t>();
    const int64_t* nn = nbrs_num_list[p].data_ptr<int64_t>();
    for (int64_t i = 0; i < idx_list[p].numel(); ++i) cnt[ix[i]] = nn[i];
  }
  std::vector<int64_t> offs(num_seeds + 1, 0);
  for (int64_t i = 0; i < num_seeds; ++i) offs[i + 1] = offs[i] + cnt[i];
  Tensor nbrs = torch::empty({offs[num_seeds]}, torch::kInt64);
  Tensor eids = with_edge ? torch::empty({offs[num_seeds]}, torch::kInt64) : Tensor();
  for (size_t p = 0; p < P; ++p) {
    const int64_t* ix = idx_list[p].data_ptr<int64_t>();
    const int64_t* nn = nbrs_num_list[p].data_ptr<int64_t>();
    const int64_t* nb = nbrs_list[p].data_ptr<int64_t>();
    const int64_t* ee = with_edge ? eids_list[p].data_ptr<int64_t>() : nullptr;
    int64_t src = 0;
    for (int64_t i = 0; i < idx_list[p].numel(); ++i) {
      std::memcpy(nbrs.data_ptr<int64_t>() + offs[ix[i]], nb + src, sizeof(int64_t) * nn[i]);
      if (ee) std::memcpy(eids.data_ptr<int64_t>() + offs[ix[i]], ee + src, sizeof(int64_t) * nn[i]);
      src += nn[i];
    }
  }
  return {nbrs, counts, eids};
}

// ----------------------------------------------------------------------------
// Hotness propagation used by the frequency partitioner / cache admission.
// Reference: csrc/cuda/random_sampler.cu:167-209 (CalNbrProbKernel):
//   cur[v] = 1 - (1 - last[v]) * prod_{u in N(v)} skip(u),
//   skip(u) = 1 - last[u]                       if deg(u) <= k
//           = 1 - last[u] * k / deg(u)           otherwise
// where N(v) are the rows that can reach v in one sampling step.
// ----------------------------------------------------------------------------
Tensor cpu_nbr_prob(const Tensor& indptr, const Tensor& indices, const Tensor& nbr_indptr,
                    const Tensor& last_prob, const Tensor& nbr_last_prob, int64_t k) {
  check_i64(indptr, "indptr");
  check_i64(indices, "indices");
  check_i64(nbr_indptr, "nbr_indptr");
  TORCH_CHECK(last_prob.scalar_type() == torch::kFloat32 && last_prob.is_contiguous());
  TORCH_CHECK(nbr_last_prob.scalar_type() == torch::kFloat32 && nbr_last_prob.is_contiguous());
  const int64_t n = last_prob.numel();
  const int64_t nn = nbr_last_prob.numel();
  const int64_t rows = indptr.numel() - 1;
  const int64_t nrows = nbr_indptr.numel() - 1;
  const int64_t* ip = indptr.data_ptr<int64_t>();
  const int64_t* ind = indices.data_ptr<int64_t>();
  const int64_t* nip = nbr_indptr.data_ptr<int64_t>();
  const float* lp = last_prob.data_ptr<float>();
  const float* nlp = nbr_last_prob.data_ptr<float>();
  Tensor cur = torch::zeros({n}, torch::kFloat32);
  float* cp = cur.data_ptr<float>();
  glt::parallel_for(0, std::min(n, rows), 2048, [&](int64_t b, int64_t e) {
    for (int64_t v = b; v < e; ++v) {
      if (ip[v + 1] == ip[v]) continue;  // isolated rows stay 0 (reference :181-185)
      double acc = 1.0;
      for (int64_t p = ip[v]; p < ip[v + 1]; ++p) {
        int64_t u = ind[p];
        if (u < 0 || u >= nn) continue;
        int64_t du = (u < nrows) ? nip[u + 1] - nip[u] : 0;
        if (du == 0) continue;
        acc *= (du <= k || k < 0) ? 1.0 - nlp[u] : 1.0 - nlp[u] * (double)k / (double)du;
      }
      cp[v] = (float)(1.0 - (1.0 - lp[v]) * acc);
    }
  });
  return cur;
}

}  // namespace glt
