// Python bindings: the only translation unit (besides cpu/*.cc) that sees torch
// headers.  Native surface parity with the reference's pybind module
// (python/py_export_glt.cc:47-222): Graph, samplers, negative sampler, inducer
// tables, subgraph op, SampleQueue, UnifiedTensor-style row tables -- plus the
// batch sampler arena and the GraphSAGE engine kernels that have no reference
// counterpart.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <pybind11/functional.h>
#include <pybind11/stl.h>
#include <torch/extension.h>

#include <cstdarg>
#include <cstdio>
#include <type_traits>

#include "cpu/cpu_ops.h"
#include "cpu/sample_queue.h"
#include "cuda/glt_cuda.h"

namespace py = pybind11;
using torch::Tensor;

namespace glt {

static cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

// Every TORCH_CHECK in this extension takes at most one message argument: a message assembled from several arguments
// crashes the process when it is thrown instead of raising.  A message that carries values is formatted first.
static std::string fmt(const char* f, ...) __attribute__((format(printf, 1, 2)));
static std::string fmt(const char* f, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, f);
  std::vsnprintf(buf, sizeof(buf), f, ap);
  va_end(ap);
  return buf;
}

static void check_cuda_err(const char* what) {
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, fmt("%s: %s", what, cudaGetErrorString(e)));
}

static const void* dev_ptr(const Tensor& t) {
  // CUDA tensors (local or peer device) and pinned host tensors are both
  // directly dereferenceable from a kernel under UVA.
  TORCH_CHECK(t.is_cuda() || t.is_pinned(), "tensor must be CUDA or pinned host memory");
  return t.data_ptr();
}

// Argument checks of the engine operands.  Unlike graph shards and row-table parts (dev_ptr), an operand must live on
// the device the binding launches on, the one its CUDAGuard made current.
static bool has(const c10::optional<Tensor>& t) { return t.has_value() && t->defined(); }

template <typename T = void>
static T* opt_ptr(const c10::optional<Tensor>& t) {
  if constexpr (std::is_void_v<T>) return has(t) ? t->data_ptr() : nullptr;
  else return has(t) ? t->data_ptr<T>() : nullptr;
}

static bool on_dev(const Tensor& t) { return t.is_cuda() && t.get_device() == c10::cuda::current_device(); }
static bool aligned16(const Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; }

// contiguous [rows, w], 16-byte aligned
static void check_rows(const Tensor& t, c10::ScalarType dt, int64_t w, const char* msg) {
  TORCH_CHECK(on_dev(t) && t.scalar_type() == dt && t.dim() == 2 && t.size(1) == w && t.is_contiguous() &&
              aligned16(t), msg);
}

// 2-D view with unit inner stride and 16-byte aligned rows whose columns [col, col + w) lie inside the row
static void check_block(const Tensor& t, c10::ScalarType dt, int64_t col, int64_t w, const char* msg) {
  TORCH_CHECK(on_dev(t) && t.scalar_type() == dt && t.dim() == 2 && t.stride(1) == 1 &&
              t.stride(0) * t.element_size() % 16 == 0 && aligned16(t) && col >= 0 &&
              col * t.element_size() % 16 == 0 && col + w <= t.size(1), msg);
}

// contiguous [n], 16-byte aligned
static void check_vec(const Tensor& t, c10::ScalarType dt, int64_t n, const char* msg) {
  TORCH_CHECK(on_dev(t) && t.scalar_type() == dt && t.numel() == n && t.is_contiguous() && aligned16(t), msg);
}

// int32 device counters with an entry at idx
static void check_counters(const Tensor& t, int64_t idx, const char* msg) {
  TORCH_CHECK(on_dev(t) && t.scalar_type() == torch::kInt32 && t.is_contiguous() && idx >= 0 && t.numel() > idx, msg);
}

// contiguous int64 ids
static void check_ids(const Tensor& t, const char* msg) {
  TORCH_CHECK(on_dev(t) && t.scalar_type() == torch::kInt64 && t.is_contiguous(), msg);
}

// ---------------------------------------------------------------------------
// GraphHandle: device view of a (possibly multi-GPU) CSR.
// ---------------------------------------------------------------------------
struct GraphHandle {
  GraphTable tbl{};
  std::vector<Tensor> keep;
  int device = 0;
  bool has_eids = true, has_weights = true;
  int64_t num_rows = 0;

  explicit GraphHandle(int dev) : device(dev) { tbl.num_parts = 0; tbl.idx_bytes = 8; }

  void add_shard(const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
                 const c10::optional<Tensor>& weights, int64_t row_begin, int64_t row_end) {
    TORCH_CHECK(tbl.num_parts < kMaxParts, "too many graph shards");
    TORCH_CHECK(indptr.scalar_type() == torch::kInt64 && indptr.is_contiguous(),
                "add_shard: indptr must be contiguous int64");
    TORCH_CHECK(indices.is_contiguous() &&
                (indices.scalar_type() == torch::kInt32 || indices.scalar_type() == torch::kInt64),
                "add_shard: indices must be contiguous int32 or int64");
    int ib = indices.scalar_type() == torch::kInt32 ? 4 : 8;
    if (tbl.num_parts == 0) tbl.idx_bytes = ib;
    TORCH_CHECK(tbl.idx_bytes == ib, "all shards must share the column id width");
    TORCH_CHECK(indptr.numel() == row_end - row_begin + 1, "indptr size != rows + 1");
    TORCH_CHECK(!has(eids) || (eids->scalar_type() == torch::kInt64 && eids->is_contiguous() &&
                               eids->numel() == indices.numel()),
                "add_shard: eids must be contiguous int64, one per column index");
    TORCH_CHECK(!has(weights) || (weights->scalar_type() == torch::kFloat32 && weights->is_contiguous() &&
                                  weights->numel() == indices.numel()),
                "add_shard: weights must be contiguous fp32, one per column index");
    CsrShard& s = tbl.parts[tbl.num_parts++];
    s.indptr = reinterpret_cast<const int64_t*>(dev_ptr(indptr));
    s.indices = dev_ptr(indices);
    s.eids = nullptr;
    s.weights = nullptr;
    keep.push_back(indptr);
    keep.push_back(indices);
    if (has(eids)) {
      s.eids = reinterpret_cast<const int64_t*>(dev_ptr(*eids));
      keep.push_back(*eids);
    } else {
      has_eids = false;
    }
    if (has(weights)) {
      s.weights = reinterpret_cast<const float*>(dev_ptr(*weights));
      keep.push_back(*weights);
    } else {
      has_weights = false;
    }
    s.row_begin = row_begin;
    s.row_end = row_end;
    num_rows = std::max(num_rows, row_end);
  }

  torch::TensorOptions opts(torch::ScalarType t) const {
    return torch::TensorOptions().dtype(t).device(torch::kCUDA, device);
  }

  // (nbrs [n,k] padded with -1, counts [n] int32, eids [n,k] | undefined)
  std::tuple<Tensor, Tensor, Tensor> sample_one_hop(const Tensor& seeds, int64_t k, bool with_edge,
                                                    bool weighted, bool replace, int64_t seed,
                                                    int64_t stream) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(seeds, "sample_one_hop: seeds must be contiguous int64 on the graph's device");
    TORCH_CHECK(k > 0 && k <= 512, "fanout must be in [1, 512] (use -1 for all neighbours)");
    TORCH_CHECK(!with_edge || has_eids, "graph has no edge ids");
    TORCH_CHECK(!weighted || has_weights, "graph has no edge weights on the device");
    const int64_t n = seeds.numel();
    Tensor nbrs = torch::empty({n, k}, opts(torch::kInt64));
    Tensor cnt = torch::empty({n}, opts(torch::kInt32));
    Tensor eids = with_edge ? torch::empty({n, k}, opts(torch::kInt64)) : Tensor();
    launch_sample_one_hop(tbl, seeds.data_ptr<int64_t>(), n, k, weighted, replace, seed, stream,
                          nbrs.data_ptr<int64_t>(), with_edge ? eids.data_ptr<int64_t>() : nullptr,
                          cnt.data_ptr<int32_t>(), cur_stream());
    check_cuda_err("sample_one_hop");
    return {nbrs, cnt, eids};
  }

  Tensor lookup_degree(const Tensor& ids) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(ids, "lookup_degree: ids must be contiguous int64 on the graph's device");
    Tensor out = torch::empty({ids.numel()}, opts(torch::kInt64));
    launch_lookup_degree(tbl, ids.data_ptr<int64_t>(), ids.numel(), out.data_ptr<int64_t>(), cur_stream());
    check_cuda_err("lookup_degree");
    return out;
  }

  // all neighbours; returns (nbrs [sum], counts [n] int64, eids)
  std::tuple<Tensor, Tensor, Tensor> full_neighbors(const Tensor& ids, bool with_edge) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(!with_edge || has_eids, "graph has no edge ids");
    Tensor deg = lookup_degree(ids);
    Tensor offs = torch::zeros({ids.numel() + 1}, opts(torch::kInt64));
    if (ids.numel() > 0) offs.narrow(0, 1, ids.numel()).copy_(deg.cumsum(0));
    const int64_t total = ids.numel() > 0 ? offs[ids.numel()].item<int64_t>() : 0;  // host sync
    Tensor nbrs = torch::empty({total}, opts(torch::kInt64));
    Tensor eids = with_edge ? torch::empty({total}, opts(torch::kInt64)) : Tensor();
    launch_copy_neighbors(tbl, ids.data_ptr<int64_t>(), ids.numel(), offs.data_ptr<int64_t>(),
                          nbrs.data_ptr<int64_t>(), with_edge ? eids.data_ptr<int64_t>() : nullptr,
                          cur_stream());
    check_cuda_err("full_neighbors");
    return {nbrs, deg, eids};
  }

  // (rows, cols, count) with rows/cols sized `req`; count stays on the device
  std::tuple<Tensor, Tensor, Tensor> negative_sample(int64_t num_rows_, int64_t num_cols, int64_t req,
                                                     int64_t trials, bool padding, int64_t seed,
                                                     int64_t stream) {
    c10::cuda::CUDAGuard guard(device);
    Tensor rows = torch::empty({req}, opts(torch::kInt64));
    Tensor cols = torch::empty({req}, opts(torch::kInt64));
    Tensor count = torch::zeros({1}, opts(torch::kInt32));
    launch_negative_sample(tbl, num_rows_, num_cols, req, trials, padding, seed, stream,
                           rows.data_ptr<int64_t>(), cols.data_ptr<int64_t>(),
                           count.data_ptr<int32_t>(), cur_stream());
    check_cuda_err("negative_sample");
    return {rows, cols, count};
  }

  Tensor random_walk(const Tensor& starts, int64_t walk_len, double p, double q, int64_t seed,
                     int64_t stream) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(starts, "random_walk: starts must be contiguous int64 on the graph's device");
    TORCH_CHECK(walk_len >= 0 && walk_len < INT32_MAX, "random_walk: walk_length must be in [0, 2^31 - 1)");
    Node2VecWeights w;
    const char* bad = node2vec_weights(p, q, &w);
    TORCH_CHECK(bad == nullptr, fmt("random_walk: %s", bad));
    Tensor out = torch::empty({starts.numel(), walk_len + 1}, opts(torch::kInt64));
    launch_random_walk(tbl, starts.data_ptr<int64_t>(), starts.numel(), static_cast<int>(walk_len),
                       !(p == 1.0 && q == 1.0), w, seed, stream, out.data_ptr<int64_t>(), cur_stream());
    check_cuda_err("random_walk");
    return out;
  }

  Tensor nbr_prob(GraphHandle& nbr_graph, const Tensor& last, const Tensor& nbr_last, int64_t k) {
    c10::cuda::CUDAGuard guard(device);
    for (const Tensor* t : {&last, &nbr_last})
      TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous(),
                  "nbr_prob: last and nbr_last must be contiguous fp32 on the graph's device");
    Tensor cur = torch::zeros_like(last);
    launch_nbr_prob(tbl, nbr_graph.tbl, last.data_ptr<float>(), nbr_last.data_ptr<float>(),
                    std::min<int64_t>(last.numel(), num_rows), nbr_last.numel(), k,
                    cur.data_ptr<float>(), cur_stream());
    check_cuda_err("nbr_prob");
    return cur;
  }
};

// ---------------------------------------------------------------------------
// DeviceTable: GPU id table (inducer state); one per node type for hetero.
// ---------------------------------------------------------------------------
struct DeviceTable {
  int device;
  int64_t cap_nodes;
  Tensor keys, vals, aux, nodes, cursor;
  HashTable ht{};

  DeviceTable(int dev, int64_t capacity) : device(dev), cap_nodes(std::max<int64_t>(capacity, 16)) {
    c10::cuda::CUDAGuard guard(device);
    int64_t slots = 64;
    while (slots < cap_nodes * 2) slots <<= 1;
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, device);
    keys = torch::full({slots}, -1, o64);
    vals = torch::zeros({slots}, o32);
    aux = torch::zeros({slots}, o32);
    nodes = torch::zeros({cap_nodes}, o64);
    cursor = torch::zeros({1}, o32);
    ht.keys = keys.data_ptr<int64_t>();
    ht.vals = vals.data_ptr<int32_t>();
    ht.aux = aux.data_ptr<int32_t>();
    ht.mask = static_cast<uint32_t>(slots - 1);
  }

  void clear() {
    c10::cuda::CUDAGuard guard(device);
    launch_table_clear(ht, cur_stream());
    cursor.zero_();
  }

  // unordered insert; returns local ids (int32).  New keys are appended to `nodes`.
  Tensor insert(const Tensor& k) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(k, "DeviceTable.insert: keys must be contiguous int64 on the table's device");
    Tensor out = torch::empty({k.numel()}, torch::TensorOptions().dtype(torch::kInt32).device(k.device()));
    launch_table_insert(ht, k.data_ptr<int64_t>(), k.numel(), nodes.data_ptr<int64_t>(),
                        cursor.data_ptr<int32_t>(), cap_nodes, out.data_ptr<int32_t>(), cur_stream());
    launch_table_resolve(ht, out.data_ptr<int32_t>(), k.numel(), cur_stream());
    check_cuda_err("table insert");
    return out;
  }

  // ordered (first-occurrence) insert into an empty table; returns local ids
  Tensor init_ordered(const Tensor& k) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(k, "DeviceTable.init_ordered: keys must be contiguous int64 on the table's device");
    TORCH_CHECK(k.numel() <= cap_nodes, "table capacity exceeded");
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(k.device());
    Tensor out = torch::empty({k.numel()}, o32);
    Tensor scratch = torch::empty({std::max<int64_t>(k.numel(), 1)}, o32);
    Tensor counters = torch::zeros({16}, o32);
    BatchCounters c{counters.data_ptr<int32_t>(), counters.data_ptr<int32_t>() + 6, cursor.data_ptr<int32_t>(), nullptr};
    launch_init_seeds(k.data_ptr<int64_t>(), k.numel(), nullptr, ht, nodes.data_ptr<int64_t>(),
                      out.data_ptr<int32_t>(), scratch.data_ptr<int32_t>(), c, nullptr, 0, cur_stream());
    check_cuda_err("table init_ordered");
    return out;
  }

  Tensor lookup(const Tensor& k) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(k, "DeviceTable.lookup: keys must be contiguous int64 on the table's device");
    Tensor out = torch::empty({k.numel()}, torch::TensorOptions().dtype(torch::kInt32).device(k.device()));
    launch_table_lookup(ht, k.data_ptr<int64_t>(), k.numel(), out.data_ptr<int32_t>(), cur_stream());
    check_cuda_err("table lookup");
    return out;
  }

  int64_t size() { return cursor.item<int32_t>(); }  // host sync

  // induced subgraph of `g` on the table's current node set (n = size())
  std::tuple<Tensor, Tensor, Tensor> subgraph(GraphHandle& g, int64_t n, bool with_edge) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(n >= 0 && n <= cap_nodes, "DeviceTable.subgraph: n must be in [0, capacity]");
    TORCH_CHECK(!with_edge || g.has_eids, "graph has no edge ids");
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    Tensor cnt = torch::zeros({n}, o64);
    launch_subgraph_count(g.tbl, ht, nodes.data_ptr<int64_t>(), n, cnt.data_ptr<int64_t>(), cur_stream());
    Tensor offs = torch::zeros({n + 1}, o64);
    if (n > 0) offs.narrow(0, 1, n).copy_(cnt.cumsum(0));
    const int64_t total = n > 0 ? offs[n].item<int64_t>() : 0;  // host sync
    Tensor rows = torch::empty({total}, o64), cols = torch::empty({total}, o64);
    Tensor eids = with_edge ? torch::empty({total}, o64) : Tensor();
    launch_subgraph_fill(g.tbl, ht, nodes.data_ptr<int64_t>(), n, offs.data_ptr<int64_t>(),
                         rows.data_ptr<int64_t>(), cols.data_ptr<int64_t>(),
                         with_edge ? eids.data_ptr<int64_t>() : nullptr, cur_stream());
    check_cuda_err("subgraph");
    return {rows, cols, eids};
  }
};

// ---------------------------------------------------------------------------
// SamplerArena: static-shape multi-hop sampling state (no host sync).
// ---------------------------------------------------------------------------
struct SamplerArena {
  int device;
  int max_seeds;
  std::vector<int64_t> fanouts;
  bool with_edge;
  std::vector<int64_t> cap_rows;  // frontier capacity per hop
  int64_t cap_nodes;
  Tensor nodes, deg, counters, seed_local, scratch, step;
  std::vector<Tensor> ell, ell_eids;
  std::unique_ptr<DeviceTable> table;
  // optional transposed adjacency (see cuda/transpose.cu): built after the hops of
  // every sample() once enable_transpose(n_hops) was called
  int tr_hops = 0;
  int64_t tr_cap_edges = 0;
  Tensor tr_cnt, tr_off, tr_cursor, tr_tgt, tr_block_sums, tr_meta, tr_meta_inv;

  // cap_override: optional calibrated frontier capacities per hop (+ one trailing entry for the
  // number of nodes the last hop may add); empty = worst case (max_seeds * prod(fanouts)).
  SamplerArena(int dev, int64_t max_seeds_, std::vector<int64_t> fanouts_, bool with_edge_,
               int64_t num_graph_nodes, std::vector<int64_t> cap_override = {})
      : device(dev), max_seeds(max_seeds_), fanouts(std::move(fanouts_)), with_edge(with_edge_) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(fanouts.size() >= 1 && fanouts.size() <= 4, "1..4 hops supported by the arena");
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, device);
    int64_t rows = max_seeds;
    cap_nodes = max_seeds;
    TORCH_CHECK(cap_override.empty() || cap_override.size() == fanouts.size() + 1,
                "cap_override needs len(fanouts)+1 entries");
    for (size_t h = 0; h < fanouts.size(); ++h) {
      TORCH_CHECK(fanouts[h] > 0 && fanouts[h] <= 512, "arena fanouts must be in [1,512]");
      if (!cap_override.empty()) rows = std::min(rows, std::max<int64_t>(cap_override[h], 1));
      cap_rows.push_back(rows);
      ell.push_back(torch::full({rows * fanouts[h]}, -1, o32));
      ell_eids.push_back(with_edge ? torch::full({rows * fanouts[h]}, -1, o64) : Tensor());
      rows = std::min<int64_t>(rows * fanouts[h], num_graph_nodes > 0 ? num_graph_nodes : INT64_MAX);
      if (!cap_override.empty()) rows = std::min(rows, std::max<int64_t>(cap_override[h + 1], 1));
      cap_nodes += rows;
    }
    cap_rows.push_back(rows);  // capacity of the nodes added by the last hop
    if (num_graph_nodes > 0) cap_nodes = std::min(cap_nodes, num_graph_nodes + max_seeds);
    TORCH_CHECK(cap_nodes < (1LL << 30), "sampler arena too large");
    table = std::make_unique<DeviceTable>(device, cap_nodes);
    nodes = table->nodes;
    deg = torch::zeros({cap_nodes}, o32);
    counters = torch::zeros({16}, o32);
    seed_local = torch::zeros({max_seeds}, o32);
    scratch = torch::zeros({max_seeds}, o32);
    step = torch::zeros({1}, o32);
  }

  void enable_transpose(int64_t n_hops) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(n_hops >= 1 && n_hops <= static_cast<int64_t>(fanouts.size()), "bad number of hops to transpose");
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, device);
    tr_hops = static_cast<int>(n_hops);
    tr_cap_edges = 0;
    for (int h = 0; h < tr_hops; ++h) tr_cap_edges += cap_rows[h] * fanouts[h];
    TORCH_CHECK(tr_cap_edges < (1LL << 31), "transposed adjacency too large");
    tr_cnt = torch::zeros({tr_hops, cap_nodes}, o32);
    tr_cursor = torch::zeros({tr_hops, cap_nodes}, o32);
    tr_off = torch::zeros({cap_nodes + 1}, o32);
    tr_tgt = torch::zeros({std::max<int64_t>(tr_cap_edges, 1)}, o32);
    tr_block_sums = torch::zeros({cap_nodes / 1024 + 2}, o32);
    tr_meta = torch::zeros({cap_nodes, 4}, o32);
    tr_meta_inv = torch::zeros({cap_nodes, 2}, o32.dtype(torch::kFloat32));
  }

  void build_transpose(cudaStream_t s) {
    TransposeArgs a{};
    a.cum = counters.data_ptr<int32_t>();
    a.deg = deg.data_ptr<int32_t>();
    for (int h = 0; h < 4; ++h) { a.ell[h] = nullptr; a.k[h] = 1; a.cap_rows[h] = 0; }
    for (int h = 0; h < tr_hops; ++h) {
      a.ell[h] = ell[h].data_ptr<int32_t>();
      a.k[h] = static_cast<int>(fanouts[h]);
      a.cap_rows[h] = static_cast<int>(cap_rows[h]);
    }
    a.n_hops = tr_hops;
    a.cap_nodes = static_cast<int>(cap_nodes);
    a.cap_edges = static_cast<int>(tr_cap_edges);
    a.cnt = tr_cnt.data_ptr<int32_t>();
    a.off = tr_off.data_ptr<int32_t>();
    a.cursor = tr_cursor.data_ptr<int32_t>();
    a.tgt = tr_tgt.data_ptr<int32_t>();
    a.block_sums = tr_block_sums.data_ptr<int32_t>();
    a.meta = tr_meta.data_ptr<int32_t>();
    a.meta_inv = tr_meta_inv.data_ptr<float>();
    launch_build_transpose(a, s);
  }

  BatchCounters bc() {
    int32_t* c = counters.data_ptr<int32_t>();
    return BatchCounters{c, c + 6, table->cursor.data_ptr<int32_t>(), c + 12};
  }

  bool deterministic = false;   // re-assign every hop's new local ids in ascending global-id order
  Tensor det_tmp;

  void sample(GraphHandle& g, const Tensor& seeds, const c10::optional<Tensor>& n_dev, int64_t seed,
              int64_t stream_base, bool weighted, bool replace, bool use_dev_step, int64_t step_inc) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(seeds, "SamplerArena.sample: seeds must be contiguous int64 on the arena's device");
    TORCH_CHECK(seeds.numel() <= max_seeds, "more seeds than the arena was built for");
    if (has(n_dev)) check_counters(*n_dev, 0, "SamplerArena.sample: n_dev must be int32 [>= 1] on the arena's device");
    TORCH_CHECK(!with_edge || g.has_eids, "graph has no edge ids");
    TORCH_CHECK(!weighted || g.has_weights, "graph has no device edge weights");
    cudaStream_t s = cur_stream();
    launch_table_clear(table->ht, s);
    launch_init_seeds(seeds.data_ptr<int64_t>(), seeds.numel(), opt_ptr<int32_t>(n_dev), table->ht, nodes.data_ptr<int64_t>(),
                      seed_local.data_ptr<int32_t>(), scratch.data_ptr<int32_t>(), bc(),
                      (use_dev_step && step_inc != 0) ? step.data_ptr<int32_t>() : nullptr,
                      static_cast<int>(step_inc), s);
    for (size_t h = 0; h < fanouts.size(); ++h) {
      HopArgs a{};
      a.g = g.tbl;
      a.t = table->ht;
      a.c = bc();
      a.nodes = nodes.data_ptr<int64_t>();
      a.ell = ell[h].data_ptr<int32_t>();
      a.ell_eids = with_edge ? ell_eids[h].data_ptr<int64_t>() : nullptr;
      a.deg = deg.data_ptr<int32_t>();
      a.hop = h;
      a.k = fanouts[h];
      a.cap_rows = cap_rows[h];
      a.cap_nodes = cap_nodes;
      a.cap_rows_next = cap_rows[h + 1];
      a.weighted = weighted;
      a.replace = replace;
      a.seed = seed;
      a.stream = static_cast<uint32_t>(stream_base + h);
      a.stream_dev = use_dev_step ? step.data_ptr<int32_t>() : nullptr;
      launch_sample_hop(a, s);
      if (deterministic) {
        if (!det_tmp.defined())
          det_tmp = torch::empty({cap_nodes}, torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device));
        launch_det_keys(a, det_tmp.data_ptr<int64_t>(), s);
        Tensor sorted = std::get<0>(torch::sort(det_tmp));
        launch_det_assign(a, sorted.data_ptr<int64_t>(), s);
      }
      launch_relabel_hop(a, s);
    }
    if (tr_hops > 0) build_transpose(s);
    check_cuda_err("arena sample");
  }

  // PyG-shaped COO (one host sync to learn the sizes):
  // returns (node [N], row [E], col [E], eids|undef, num_sampled_nodes, num_sampled_edges)
  std::tuple<Tensor, Tensor, Tensor, Tensor, std::vector<int64_t>, std::vector<int64_t>> to_coo() {
    c10::cuda::CUDAGuard guard(device);
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    Tensor host = counters.cpu();  // sync
    const int32_t* c = host.data_ptr<int32_t>();
    const int L = fanouts.size();
    std::vector<int64_t> nn, ne;
    for (int h = 0; h <= L; ++h) nn.push_back(c[h + 1] - c[h]);
    int64_t E = 0;
    for (int h = 0; h < L; ++h) { ne.push_back(c[6 + h]); E += c[6 + h]; }
    const int64_t N = c[L + 1], T = c[L];
    Tensor offs = torch::zeros({T + 1}, o64);
    if (T > 0) offs.narrow(0, 1, T).copy_(deg.narrow(0, 0, T).to(torch::kInt64).cumsum(0));
    Tensor rows = torch::empty({E}, o64), cols = torch::empty({E}, o64);
    Tensor eids = with_edge ? torch::empty({E}, o64) : Tensor();
    for (int h = 0; h < L; ++h) {
      launch_ell_to_coo(ell[h].data_ptr<int32_t>(), with_edge ? ell_eids[h].data_ptr<int64_t>() : nullptr,
                        deg.data_ptr<int32_t>(), offs.data_ptr<int64_t>(), counters.data_ptr<int32_t>(),
                        h, fanouts[h], cap_rows[h], rows.data_ptr<int64_t>(), cols.data_ptr<int64_t>(),
                        with_edge ? eids.data_ptr<int64_t>() : nullptr, cur_stream());
    }
    check_cuda_err("to_coo");
    return {nodes.narrow(0, 0, N).clone(), rows, cols, eids, nn, ne};
  }
};


// ---------------------------------------------------------------------------
// HeteroArena: device-resident multi-hop sampling + inducing over a heterogeneous graph (native counterpart of
// the reference's CUDAHeteroInducer, csrc/cuda/inducer.cu:194-338, plus the per-hop orchestration of
// python/sampler/neighbor_sampler.py:232-317).  Node types and relations are integer coded; every node type
// owns an id table / id list / hop counters, every relation owns fixed-stride ELL blocks per hop.  One hop =
// three launches for ALL relations together (grouped sample, per-type finalize, grouped relabel) and no host
// synchronisation; sizes stay in `counters` until a PyG-shaped COO is requested.
// ---------------------------------------------------------------------------
struct HeteroArena {
  int device, n_types, n_rel, hops;
  bool with_edge;
  std::vector<GraphHandle*> graphs;
  std::vector<int64_t> key_type, nbr_type;
  std::vector<std::vector<int64_t>> fanouts;       // [rel][hop]
  std::vector<std::vector<int64_t>> cap_rows;      // [type][hop + 1]
  std::vector<int64_t> cap_nodes, max_seeds;
  std::vector<std::unique_ptr<DeviceTable>> tables;
  Tensor all_keys;                                 // the tables' key arrays, contiguous: one memset clears them
  Tensor counters, step, descs, type_states, seed_scratch, seed_local, deg_all;
  std::vector<Tensor> deg;                         // [rel] views into deg_all
  std::vector<std::vector<Tensor>> ell, ell_eids;  // [rel][hop]
  std::vector<int> max_k, max_rows;                // per hop
  bool any_zero_fanout = false;
  int ctr_type_base(int t) const { return t * 8; }
  int ctr_rel_base(int r) const { return n_types * 8 + r * 4; }
  int ctr_overflow() const { return n_types * 8 + n_rel * 4; }

  HeteroArena(int dev, int64_t n_types_, std::vector<GraphHandle*> graphs_, std::vector<int64_t> key_type_,
              std::vector<int64_t> nbr_type_, std::vector<std::vector<int64_t>> fanouts_,
              std::vector<int64_t> num_nodes, std::vector<int64_t> max_seeds_, bool with_edge_, int64_t seed,
              bool weighted, bool replace, int64_t cap_limit, std::vector<std::vector<int64_t>> cap_override)
      : device(dev), n_types(n_types_), n_rel(graphs_.size()), with_edge(with_edge_), graphs(std::move(graphs_)),
        key_type(std::move(key_type_)), nbr_type(std::move(nbr_type_)), fanouts(std::move(fanouts_)),
        max_seeds(std::move(max_seeds_)) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(n_rel >= 1 && static_cast<int>(key_type.size()) == n_rel && static_cast<int>(nbr_type.size()) == n_rel &&
                static_cast<int>(fanouts.size()) == n_rel, "HeteroArena: one (graph, key type, nbr type, fanouts) per relation");
    TORCH_CHECK(static_cast<int>(num_nodes.size()) == n_types && static_cast<int>(max_seeds.size()) == n_types,
                "HeteroArena: num_nodes and max_seeds need one entry per node type");
    hops = fanouts[0].size();
    TORCH_CHECK(hops >= 1 && hops <= 4, "1..4 hops supported by the arena");
    for (int r = 0; r < n_rel; ++r) {
      TORCH_CHECK(static_cast<int>(fanouts[r].size()) == hops, "all relations need the same number of hops");
      TORCH_CHECK(key_type[r] >= 0 && key_type[r] < n_types && nbr_type[r] >= 0 && nbr_type[r] < n_types,
                  "HeteroArena: key and neighbour types must be in [0, n_types)");
      TORCH_CHECK(!with_edge || graphs[r]->has_eids, "graph has no edge ids");
      TORCH_CHECK(!weighted || graphs[r]->has_weights, "graph has no device edge weights");
      for (int h = 0; h < hops; ++h) {
        TORCH_CHECK(fanouts[r][h] >= 0 && fanouts[r][h] <= 512, "arena fanouts must be in [0,512]");
        if (fanouts[r][h] == 0) any_zero_fanout = true;
      }
    }
    if (cap_limit <= 0) cap_limit = INT64_MAX;
    // frontier capacities: worst case of the fan-out recursion, bounded by the type's node count and cap_limit
    cap_rows.assign(n_types, std::vector<int64_t>(hops + 1, 0));
    for (int t = 0; t < n_types; ++t) cap_rows[t][0] = max_seeds[t];
    for (int h = 0; h < hops; ++h)
      for (int t = 0; t < n_types; ++t) {
        int64_t rows = 0;
        for (int r = 0; r < n_rel; ++r)
          if (nbr_type[r] == t) rows += cap_rows[key_type[r]][h] * fanouts[r][h];
        rows = std::min(rows, std::min(num_nodes[t] > 0 ? num_nodes[t] : INT64_MAX, cap_limit));
        if (!cap_override.empty()) rows = std::min(rows, std::max<int64_t>(cap_override[t][h + 1], 0));
        cap_rows[t][h + 1] = rows;
      }
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, device);
    auto o8 = torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, device);
    counters = torch::zeros({n_types * 8 + n_rel * 4 + 8}, o32);   // [types | relations | overflow, scratch]
    step = torch::zeros({1}, o32);
    int32_t* cbase = counters.data_ptr<int32_t>();
    // id tables: key arrays carved out of one buffer so a batch starts with ONE memset
    int64_t total_slots = 0;
    std::vector<int64_t> slots(n_types);
    cap_nodes.assign(n_types, 0);
    int64_t max_seed_all = 1;
    for (int t = 0; t < n_types; ++t) {
      int64_t cn = 0;
      for (int h = 0; h <= hops; ++h) cn += cap_rows[t][h];
      if (num_nodes[t] > 0) cn = std::min(cn, num_nodes[t] + max_seeds[t]);
      cap_nodes[t] = std::max<int64_t>(cn, 16);
      TORCH_CHECK(cap_nodes[t] < (1LL << 30), "sampler arena too large");
      int64_t sl = 64;
      while (sl < cap_nodes[t] * 2) sl <<= 1;
      slots[t] = sl;
      total_slots += sl;
      max_seed_all = std::max(max_seed_all, max_seeds[t]);
    }
    all_keys = torch::full({total_slots}, -1, o64);
    int64_t off = 0;
    for (int t = 0; t < n_types; ++t) {
      auto tb = std::make_unique<DeviceTable>(device, 16);   // small placeholder, re-pointed below
      tb->cap_nodes = cap_nodes[t];
      tb->keys = all_keys.narrow(0, off, slots[t]);
      tb->vals = torch::zeros({slots[t]}, o32);
      tb->aux = torch::zeros({slots[t]}, o32);
      tb->nodes = torch::zeros({cap_nodes[t]}, o64);
      tb->cursor = counters.narrow(0, ctr_type_base(t) + 6, 1);
      tb->ht.keys = tb->keys.data_ptr<int64_t>();
      tb->ht.vals = tb->vals.data_ptr<int32_t>();
      tb->ht.aux = tb->aux.data_ptr<int32_t>();
      tb->ht.mask = static_cast<uint32_t>(slots[t] - 1);
      off += slots[t];
      tables.push_back(std::move(tb));
    }
    seed_scratch = torch::zeros({max_seed_all}, o32);
    seed_local = torch::zeros({n_types, max_seed_all}, o32);
    // per-relation degree arrays (indexed by the key type's local id), one contiguous buffer
    int64_t deg_total = 0;
    for (int r = 0; r < n_rel; ++r) deg_total += cap_nodes[key_type[r]];
    deg_all = torch::zeros({deg_total}, o32);
    off = 0;
    for (int r = 0; r < n_rel; ++r) {
      deg.push_back(deg_all.narrow(0, off, cap_nodes[key_type[r]]));
      off += cap_nodes[key_type[r]];
    }
    ell.resize(n_rel);
    ell_eids.resize(n_rel);
    for (int r = 0; r < n_rel; ++r)
      for (int h = 0; h < hops; ++h) {
        const int64_t n = cap_rows[key_type[r]][h] * fanouts[r][h];
        ell[r].push_back(torch::full({std::max<int64_t>(n, 1)}, -1, o32));
        ell_eids[r].push_back(with_edge ? torch::full({std::max<int64_t>(n, 1)}, -1, o64) : Tensor());
      }
    // static launch descriptors
    std::vector<HopArgs> hd(static_cast<size_t>(hops) * n_rel);
    max_k.assign(hops, 0);
    max_rows.assign(hops, 1);
    for (int h = 0; h < hops; ++h)
      for (int r = 0; r < n_rel; ++r) {
        HopArgs a{};
        const int kt = key_type[r], nt = nbr_type[r];
        a.g = graphs[r]->tbl;
        a.t = tables[nt]->ht;
        a.c.cum = cbase + ctr_type_base(kt);
        a.c.edges = cbase + ctr_rel_base(r);
        a.c.cursor = cbase + ctr_type_base(nt) + 6;
        a.c.overflow = cbase + ctr_overflow();
        a.nodes = tables[kt]->nodes.data_ptr<int64_t>();
        a.nodes_out = tables[nt]->nodes.data_ptr<int64_t>();
        a.ell = ell[r][h].data_ptr<int32_t>();
        a.ell_eids = with_edge ? ell_eids[r][h].data_ptr<int64_t>() : nullptr;
        a.deg = deg[r].data_ptr<int32_t>();
        a.hop = h;
        a.k = static_cast<int>(fanouts[r][h]);
        a.cap_rows = static_cast<int>(cap_rows[kt][h]);
        a.cap_nodes = static_cast<int>(cap_nodes[nt]);
        a.cap_rows_next = static_cast<int>(cap_rows[nt][h + 1]);
        a.weighted = weighted ? 1 : 0;
        a.replace = replace ? 1 : 0;
        a.seed = static_cast<uint64_t>(seed);
        a.stream = static_cast<uint32_t>(h * n_rel + r);
        a.stream_dev = step.data_ptr<int32_t>();
        a.stream_stride = 1;   // `step` holds the Philox stream base itself (callers add hops * n_rel per batch)
        a.bound_ptr = cbase + ctr_type_base(nt) + h + 2;
        hd[static_cast<size_t>(h) * n_rel + r] = a;
        if (a.k > 0) {
          max_k[h] = std::max(max_k[h], a.k);
          max_rows[h] = std::max(max_rows[h], a.cap_rows);
        }
      }
    descs = torch::empty({static_cast<int64_t>(hd.size() * sizeof(HopArgs))}, o8);
    cudaMemcpy(descs.data_ptr(), hd.data(), hd.size() * sizeof(HopArgs), cudaMemcpyHostToDevice);
    std::vector<HeteroTypeState> ts(n_types);
    for (int t = 0; t < n_types; ++t) {
      ts[t].cum = cbase + ctr_type_base(t);
      ts[t].cursor = cbase + ctr_type_base(t) + 6;
      ts[t].cap_nodes = static_cast<int>(cap_nodes[t]);
      for (int h = 0; h < 5; ++h) ts[t].cap_rows[h] = h <= hops ? static_cast<int>(cap_rows[t][h]) : 0;
    }
    type_states = torch::empty({static_cast<int64_t>(ts.size() * sizeof(HeteroTypeState))}, o8);
    cudaMemcpy(type_states.data_ptr(), ts.data(), ts.size() * sizeof(HeteroTypeState), cudaMemcpyHostToDevice);
    check_cuda_err("HeteroArena setup");
  }

  // seeds of one or more node types -> multi-hop sample of every relation; no host synchronisation
  void sample(const std::vector<int64_t>& seed_types, const std::vector<Tensor>& seeds, int64_t step_inc) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(seed_types.size() == seeds.size() && !seeds.empty(), "HeteroArena.sample: one seed type per seed tensor");
    cudaStream_t s = cur_stream();
    int32_t* cbase = counters.data_ptr<int32_t>();
    cudaMemsetAsync(cbase, 0, sizeof(int32_t) * ctr_overflow(), s);          // every cum / cursor / edge counter
    cudaMemsetAsync(all_keys.data_ptr(), 0xFF, all_keys.numel() * sizeof(int64_t), s);
    if (any_zero_fanout) cudaMemsetAsync(deg_all.data_ptr(), 0, deg_all.numel() * sizeof(int32_t), s);
    for (size_t i = 0; i < seeds.size(); ++i) {
      const int t = static_cast<int>(seed_types[i]);
      const Tensor& sd = seeds[i];
      TORCH_CHECK(t >= 0 && t < n_types, "HeteroArena.sample: seed type outside [0, n_types)");
      check_ids(sd, "HeteroArena.sample: seeds must be contiguous int64 on the arena's device");
      TORCH_CHECK(sd.numel() <= max_seeds[t], "more seeds than the arena was built for");
      BatchCounters c{cbase + ctr_type_base(t), cbase + ctr_overflow() + 1 /* scratch */, cbase + ctr_type_base(t) + 6,
                      cbase + ctr_overflow()};
      // init_seeds zeroes 4 "edge" counters: point them at scratch words that nothing else reads
      launch_init_seeds(sd.data_ptr<int64_t>(), sd.numel(), nullptr, tables[t]->ht, tables[t]->nodes.data_ptr<int64_t>(),
                        seed_local.data_ptr<int32_t>() + t * seed_local.size(1), seed_scratch.data_ptr<int32_t>(), c,
                        (i == 0 && step_inc != 0) ? step.data_ptr<int32_t>() : nullptr, static_cast<int>(step_inc), s);
    }
    const HopArgs* d = reinterpret_cast<const HopArgs*>(descs.data_ptr());
    const HeteroTypeState* ts = reinterpret_cast<const HeteroTypeState*>(type_states.data_ptr());
    for (int h = 0; h < hops; ++h) {
      launch_sample_hop_grouped(d + static_cast<size_t>(h) * n_rel, n_rel, max_k[h], max_rows[h], s);
      launch_hetero_finalize(ts, n_types, h, s);
      launch_relabel_hop_grouped(d + static_cast<size_t>(h) * n_rel, n_rel, max_k[h], max_rows[h], s);
    }
    check_cuda_err("hetero arena sample");
  }

  // PyG-shaped output (ONE host sync for the sizes):
  //   nodes[t] (global ids, hop-contiguous), per relation (rows = neighbour local ids, cols = key local ids, eids),
  //   num_sampled_nodes[t][hop], num_sampled_edges[rel][hop]
  std::tuple<std::vector<Tensor>, std::vector<Tensor>, std::vector<Tensor>, std::vector<Tensor>,
             std::vector<std::vector<int64_t>>, std::vector<std::vector<int64_t>>> to_coo() {
    c10::cuda::CUDAGuard guard(device);
    auto o64 = torch::TensorOptions().dtype(torch::kInt64).device(torch::kCUDA, device);
    Tensor host = counters.cpu();  // sync
    const int32_t* c = host.data_ptr<int32_t>();
    std::vector<Tensor> nodes_out, rows_out, cols_out, eids_out;
    std::vector<std::vector<int64_t>> nn(n_types), ne(n_rel);
    for (int t = 0; t < n_types; ++t) {
      const int32_t* cum = c + ctr_type_base(t);
      for (int h = 0; h <= hops; ++h) nn[t].push_back(cum[h + 1] - cum[h]);
      nodes_out.push_back(tables[t]->nodes.narrow(0, 0, cum[hops + 1]).clone());
    }
    for (int r = 0; r < n_rel; ++r) {
      const int32_t* cum = c + ctr_type_base(key_type[r]);
      int64_t E = 0;
      for (int h = 0; h < hops; ++h) { ne[r].push_back(c[ctr_rel_base(r) + h]); E += c[ctr_rel_base(r) + h]; }
      const int64_t T = cum[hops];
      Tensor rows = torch::empty({E}, o64), cols = torch::empty({E}, o64);
      Tensor eids = with_edge ? torch::empty({E}, o64) : Tensor();
      if (E > 0) {
        Tensor offs = torch::zeros({T + 1}, o64);
        offs.narrow(0, 1, T).copy_(deg[r].narrow(0, 0, T).to(torch::kInt64).cumsum(0));
        for (int h = 0; h < hops; ++h) {
          if (fanouts[r][h] <= 0) continue;
          launch_ell_to_coo(ell[r][h].data_ptr<int32_t>(), with_edge ? ell_eids[r][h].data_ptr<int64_t>() : nullptr,
                            deg[r].data_ptr<int32_t>(), offs.data_ptr<int64_t>(),
                            counters.data_ptr<int32_t>() + ctr_type_base(key_type[r]), h, fanouts[r][h],
                            cap_rows[key_type[r]][h], rows.data_ptr<int64_t>(), cols.data_ptr<int64_t>(),
                            with_edge ? eids.data_ptr<int64_t>() : nullptr, cur_stream());
        }
      }
      rows_out.push_back(rows); cols_out.push_back(cols); eids_out.push_back(eids);
    }
    check_cuda_err("hetero to_coo");
    return {nodes_out, rows_out, cols_out, eids_out, nn, ne};
  }

  int64_t overflow_index() const { return ctr_overflow(); }
  Tensor seed_local_of(int64_t t) { return seed_local[t]; }
  Tensor nodes_of(int64_t t) { return tables[t]->nodes; }
  Tensor deg_of(int64_t r) { return deg[r]; }
  Tensor ell_of(int64_t r, int64_t h) { return ell[r][h]; }
};

// Bytes of an MXFP8 row of d elements: d e4m3 bytes, d / 32 scale bytes, zero padding to 16 (data/quantize.py,
// mxfp8_row_bytes).
static int64_t mxfp8_row_bytes(int64_t d) { return (d + d / 32 + 15) / 16 * 16; }

// ---------------------------------------------------------------------------
// RowTableHandle: multi-source row store (UnifiedTensor).
// ---------------------------------------------------------------------------
struct RowTableHandle {
  RowTable tbl{};
  std::vector<Tensor> keep;
  unsigned local_mask = 0;   // bit p: part p is memory of `device` itself (not a peer GPU's HBM / pinned host)
  int device;
  torch::ScalarType dtype = torch::kFloat32;
  int64_t width = 0;

  explicit RowTableHandle(int dev) : device(dev) { tbl.num_parts = 0; tbl.row_begin[0] = 0; }

  // remote = true: the rows live in a PEER GPU's HBM (IPC-mapped); cudaPointerGetAttributes cannot tell -- it reports
  // the importing device for memory opened with cudaIpcOpenMemHandle -- so the caller says so (parallel/partitioned.py)
  void append(const Tensor& part, bool remote = false) {
    TORCH_CHECK(tbl.num_parts < kMaxParts, "too many row-table parts");
    TORCH_CHECK(part.dim() >= 1 && part.is_contiguous(), "parts must be contiguous [rows, ...]");
    const int64_t w = part.numel() / std::max<int64_t>(part.size(0), 1);
    if (tbl.num_parts == 0) {
      dtype = part.scalar_type();
      width = part.dim() > 1 ? w : 1;
      tbl.row_bytes = width * part.element_size();
    }
    TORCH_CHECK(part.scalar_type() == dtype, "dtype mismatch between parts");
    TORCH_CHECK((part.dim() > 1 ? w : 1) == width || part.size(0) == 0, "row width mismatch");
    tbl.base[tbl.num_parts] = part.size(0) > 0 ? dev_ptr(part) : nullptr;
    if (part.size(0) > 0 && part.is_cuda() && !remote) {
      cudaPointerAttributes at{};
      if (cudaPointerGetAttributes(&at, part.data_ptr()) == cudaSuccess && at.type == cudaMemoryTypeDevice &&
          at.device == device)
        local_mask |= 1u << tbl.num_parts;
      else
        cudaGetLastError();
    }
    tbl.row_begin[tbl.num_parts + 1] = tbl.row_begin[tbl.num_parts] + part.size(0);
    tbl.num_parts++;
    keep.push_back(part);
  }

  int64_t num_rows() const { return tbl.row_begin[tbl.num_parts]; }

  Tensor gather(const Tensor& idx, const c10::optional<Tensor>& id2index, int64_t out_width) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(idx, "gather: idx must be contiguous int64 on the table's device");
    if (has(id2index)) check_ids(*id2index, "gather: id2index must be contiguous int64 on the table's device");
    if (out_width <= 0) out_width = width;
    TORCH_CHECK(out_width >= width, "gather: out_width must be at least the table's width");
    auto o = torch::TensorOptions().dtype(dtype).device(torch::kCUDA, device);
    Tensor out = out_width == width ? torch::empty({idx.numel(), width}, o)
                                    : torch::zeros({idx.numel(), out_width}, o);
    launch_gather_rows(tbl, idx.data_ptr<int64_t>(), opt_ptr<int64_t>(id2index), idx.numel(), nullptr, out.data_ptr(),
                       out_width * out.element_size(), cur_stream(), has(id2index) ? id2index->numel() : 0);
    check_cuda_err("gather_rows");
    return out;
  }

  bool all_local() const { return local_mask == ((tbl.num_parts >= 32) ? ~0u : ((1u << tbl.num_parts) - 1u)); }

  // rows are MXFP8 (d e4m3 bytes + d/32 UE8M0 scales + padding to 16 bytes): dequantised bf16 [n, d]
  Tensor gather_mxfp8(const Tensor& idx, int64_t d) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(dtype == torch::kUInt8 && d % 128 == 0 && width >= d + d / 32 && width % 16 == 0,
                "gather_mxfp8: table must hold uint8 rows of d + d/32 (+pad) bytes, d a multiple of 128");
    check_ids(idx, "gather_mxfp8: idx must be contiguous int64 on the table's device");
    Tensor out = torch::empty({idx.numel(), d}, torch::TensorOptions().dtype(torch::kBFloat16).device(torch::kCUDA, device));
    launch_gather_mxfp8(tbl, idx.data_ptr<int64_t>(), idx.numel(), d, out.data_ptr(), cur_stream());
    check_cuda_err("gather_mxfp8");
    return out;
  }

  bool holds_mxfp8(int64_t d) const {
    return dtype == torch::kUInt8 && d % 32 == 0 && d >= 32 && d <= 1024 && width == mxfp8_row_bytes(d);
  }

  // gather_into for MXFP8 rows of d elements (any multiple of 32 up to 1024): out[i, :d] = bf16(dequantised row);
  // rows past *n_dev and rows with a negative (or unmapped) id are written as zeros; columns >= d are not touched
  void gather_mxfp8_into(const Tensor& idx, const c10::optional<Tensor>& id2index,
                         const c10::optional<Tensor>& n_dev, Tensor out, int64_t d) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(d % 32 == 0 && d >= 32 && d <= 1024, "gather_mxfp8_into: d must be a multiple of 32 in [32, 1024]");
    TORCH_CHECK(holds_mxfp8(d), "gather_mxfp8_into: the table must hold uint8 rows of mxfp8_row_bytes(d) bytes");
    check_ids(idx, "gather_mxfp8_into: idx must be a contiguous int64 CUDA tensor");
    if (has(id2index)) check_ids(*id2index, "gather_mxfp8_into: id2index must be contiguous int64 on the table's device");
    if (has(n_dev)) check_counters(*n_dev, 0, "gather_mxfp8_into: n_dev must be int32 [>= 1] on the table's device");
    check_block(out, torch::kBFloat16, 0, d,
                "gather_mxfp8_into: destination must be bf16 [>= rows, >= d] with unit inner stride and 16-byte aligned rows");
    TORCH_CHECK(out.size(0) >= idx.numel(), "gather_mxfp8_into: destination must be bf16 [>= rows, >= d]");
    launch_gather_mxfp8_rows(tbl, idx.data_ptr<int64_t>(), opt_ptr<int64_t>(id2index), idx.numel(),
                             opt_ptr<int32_t>(n_dev), static_cast<int>(d), out.data_ptr(), out.stride(0) * 2, cur_stream(),
                             has(id2index) ? id2index->numel() : 0);
    check_cuda_err("gather_mxfp8_into");
  }

  // static-shape gather into a caller-provided buffer with a device-side count
  void gather_into(const Tensor& idx, const c10::optional<Tensor>& id2index,
                   const c10::optional<Tensor>& n_dev, Tensor out) {
    c10::cuda::CUDAGuard guard(device);
    check_ids(idx, "gather_into: idx must be contiguous int64 on the table's device");
    if (has(id2index)) check_ids(*id2index, "gather_into: id2index must be contiguous int64 on the table's device");
    if (has(n_dev)) check_counters(*n_dev, 0, "gather_into: n_dev must be int32 [>= 1] on the table's device");
    check_block(out, dtype, 0, width, "gather_into: [rows, >= width] destination of the table's dtype with unit inner stride");
    TORCH_CHECK(out.size(0) >= idx.numel(), "gather_into: [rows, >= width] destination with a row per id");
    launch_gather_rows(tbl, idx.data_ptr<int64_t>(), opt_ptr<int64_t>(id2index), idx.numel(), opt_ptr<int32_t>(n_dev),
                       out.data_ptr(), out.stride(0) * out.element_size(), cur_stream(),
                       has(id2index) ? id2index->numel() : 0);
    check_cuda_err("gather_into");
  }
};

// ---------------------------------------------------------------------------
// GraphSAGE engine kernels
// ---------------------------------------------------------------------------
// The ELL blocks of the hops and the degree array: int32, contiguous, on the device.  Returns deg's pointer.
static const int32_t* fill_ell(const std::vector<Tensor>& ell, const std::vector<int64_t>& ks, const Tensor& deg,
                               const int32_t** out_ell, int* out_k) {
  TORCH_CHECK(ell.size() == ks.size() && ell.size() <= 4, "ell and ks need one entry per hop, at most 4");
  TORCH_CHECK(on_dev(deg) && deg.scalar_type() == torch::kInt32 && deg.is_contiguous(),
              "deg must be contiguous int32 on the device");
  for (size_t i = 0; i < 4; ++i) { out_ell[i] = nullptr; out_k[i] = 1; }
  for (size_t i = 0; i < ell.size(); ++i) {
    TORCH_CHECK(on_dev(ell[i]) && ell[i].scalar_type() == torch::kInt32 && ell[i].is_contiguous(),
                "ELL blocks must be contiguous int32 on the device");
    out_ell[i] = ell[i].data_ptr<int32_t>();
    out_k[i] = ks[i];
  }
  return deg.data_ptr<int32_t>();
}

// The aggregation / scatter kernels cover at most 128 16-byte vectors per row, i.e. 1024 bf16 columns (the lane-group
// dispatch, dispatch_lanes in csrc/cuda/launch_utils.h).
static void check_sage_width(int64_t d, const char* msg) {
  TORCH_CHECK(d % 8 == 0 && d >= 8 && d <= 1024, msg);
}

// A layer-1 feature table of width d: bf16 rows d wide, or MXFP8 rows of mxfp8_row_bytes(d) bytes.
static void check_feature_table(const RowTableHandle* feat, int64_t d) {
  TORCH_CHECK(feat->dtype == torch::kBFloat16 || feat->dtype == torch::kUInt8,
              "engine features must be bf16 rows or MXFP8 (uint8) rows");
  TORCH_CHECK(feat->dtype == torch::kBFloat16 ? feat->width == d : feat->holds_mxfp8(d),
              "feature width mismatch (bf16 rows are d wide; MXFP8 rows are mxfp8_row_bytes(d) bytes, d a multiple of 32 in [32, 1024])");
}

static SageAggArgs make_agg(RowTableHandle* feat, const c10::optional<Tensor>& nodes,
                            const c10::optional<Tensor>& src_local, int64_t d, const Tensor& counters,
                            int64_t n_hops_targets, int64_t cap_targets, const std::vector<Tensor>& ell,
                            const std::vector<int64_t>& ks, const Tensor& deg, void* out) {
  SageAggArgs a{};
  if (has(src_local)) {
    check_rows(*src_local, torch::kBFloat16, d, "aggregation: src_local must be contiguous bf16 [rows, d]");
    a.src_local = src_local->data_ptr();
  } else {
    TORCH_CHECK(feat != nullptr && has(nodes), "layer-1 aggregation needs a feature table + nodes");
    check_feature_table(feat, d);
    check_ids(*nodes, "aggregation: nodes must be contiguous int64 on the device");
    a.feat = feat->tbl;
    a.feat_fp8 = feat->dtype == torch::kUInt8 ? 1 : 0;
    a.nodes = nodes->data_ptr<int64_t>();
  }
  TORCH_CHECK(d % 8 == 0, "feature width must be a multiple of 8");
  check_counters(counters, n_hops_targets, "aggregation: counters must be int32 [> n_hops_targets] on the device");
  a.d = d;
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  a.cap_targets = cap_targets;
  a.deg = fill_ell(ell, ks, deg, a.ell, a.k);
  a.out = out;
  return a;
}

static void sage_aggregate(RowTableHandle* feat, const c10::optional<Tensor>& nodes,
                           const c10::optional<Tensor>& src_local, int64_t d, const Tensor& counters,
                           int64_t n_hops_targets, const std::vector<Tensor>& ell,
                           const std::vector<int64_t>& ks, const Tensor& deg, Tensor out) {
  c10::cuda::CUDAGuard guard(out.device());
  check_sage_width(d, "sage_aggregate: d must be a multiple of 8 in [8, 1024]");
  check_rows(out, torch::kBFloat16, 2 * d, "sage_aggregate: out must be contiguous bf16 [rows, 2d]");
  SageAggArgs a = make_agg(feat, nodes, src_local, d, counters, n_hops_targets, out.size(0), ell, ks,
                           deg, out.data_ptr());
  launch_sage_aggregate(a, cur_stream());
  check_cuda_err("sage_aggregate");
}

// ---- column-block variants used by the heterogeneous engine: A_t = [mean_rel1 | mean_rel2 | ... | self] ----
static void sage_aggregate_block(RowTableHandle* feat, const c10::optional<Tensor>& nodes,
                                 const c10::optional<Tensor>& src_local, int64_t d, const Tensor& counters,
                                 int64_t n_hops_targets, const std::vector<Tensor>& ell,
                                 const std::vector<int64_t>& ks, const Tensor& deg, Tensor out, int64_t mean_col) {
  c10::cuda::CUDAGuard guard(out.device());
  check_sage_width(d, "sage_aggregate_block: d must be a multiple of 8 in [8, 1024]");
  check_block(out, torch::kBFloat16, mean_col, d,
              "sage_aggregate_block: out must be a bf16 view with 16-byte aligned rows holding columns [mean_col, mean_col + d)");
  SageAggArgs a = make_agg(feat, nodes, src_local, d, counters, n_hops_targets, out.size(0), ell, ks,
                           deg, out.data_ptr());
  a.out_ld = static_cast<int>(out.stride(0));
  a.mean_col = static_cast<int>(mean_col);
  a.self_col = -1;
  launch_sage_aggregate(a, cur_stream());
  check_cuda_err("sage_aggregate_block");
}

static void sage_scatter_block(const Tensor& dA, int64_t d, int64_t mean_col, const Tensor& counters,
                               int64_t n_hops_targets, const std::vector<Tensor>& ell,
                               const std::vector<int64_t>& ks, const Tensor& deg, Tensor dH) {
  c10::cuda::CUDAGuard guard(dA.device());
  check_sage_width(d, "sage_scatter_block: d must be a multiple of 8 in [8, 1024]");
  check_block(dA, torch::kBFloat16, mean_col, d,
              "sage_scatter_block: dA must be a bf16 view with 16-byte aligned rows holding columns [mean_col, mean_col + d)");
  check_rows(dH, torch::kFloat32, d, "sage_scatter_block: dH must be contiguous fp32 [rows, d]");
  check_counters(counters, n_hops_targets, "sage_scatter_block: counters must be int32 [> n_hops_targets] on the device");
  SageScatterArgs a{};
  a.dA = dA.data_ptr();
  a.d = d;
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  a.cap_targets = dA.size(0);
  a.deg = fill_ell(ell, ks, deg, a.ell, a.k);
  a.dH = dH.data_ptr<float>();
  a.dA_ld = static_cast<int>(dA.stride(0));
  a.mean_col = static_cast<int>(mean_col);
  launch_sage_scatter_bwd(a, cur_stream());
  check_cuda_err("sage_scatter_block");
}

// Exact full-neighbourhood aggregation of the global rows [r0, r1) (csrc/cuda/sage_infer.cu).  `src` (bf16, indexed by
// global id) is the source of deeper layers; without it the rows come from `feat` (bf16 or MXFP8 rows, layer 1).
static void sage_full_aggregate(GraphHandle* graph, RowTableHandle* feat, const c10::optional<Tensor>& src,
                                int64_t src_col, int64_t self_col, int64_t d, int64_t r0, int64_t r1, bool combine,
                                const c10::optional<Tensor>& bias, bool relu, Tensor out, bool mean_only) {
  c10::cuda::CUDAGuard guard(out.device());
  TORCH_CHECK(graph != nullptr && graph->tbl.num_parts > 0, "sage_full_aggregate: graph has no shards");
  TORCH_CHECK(!(combine && mean_only), "sage_full_aggregate: mean_only writes the mean block of the concat mode, not combine");
  check_sage_width(d, "sage_full_aggregate: d must be a multiple of 8 in [8, 1024]");
  TORCH_CHECK(0 <= r0 && r0 <= r1 && r1 <= graph->num_rows, "sage_full_aggregate: rows [r0, r1) outside the graph");
  const char* out_msg = combine || mean_only
      ? "sage_full_aggregate: out must be bf16 [>= r1 - r0, >= d] with unit inner stride and 16-byte aligned rows"
      : "sage_full_aggregate: out must be bf16 [>= r1 - r0, >= 2d] with unit inner stride and 16-byte aligned rows";
  check_block(out, torch::kBFloat16, 0, combine || mean_only ? d : 2 * d, out_msg);
  TORCH_CHECK(out.size(0) >= r1 - r0, out_msg);
  SageFullAggArgs a{};
  a.g = graph->tbl;
  a.d = static_cast<int>(d);
  a.r0 = r0;
  a.r1 = r1;
  a.combine = combine ? 1 : 0;
  a.out = out.data_ptr();
  a.out_ld = out.stride(0);
  a.mean_only = mean_only ? 1 : 0;
  if (has(src)) {
    const char* src_msg = "sage_full_aggregate: src must be a bf16 CUDA table with unit inner stride and 16-byte aligned "
                          "rows, and column blocks [src_col, src_col + d), [self_col, self_col + d) inside them";
    check_block(*src, torch::kBFloat16, src_col, d, src_msg);
    check_block(*src, torch::kBFloat16, self_col, d, src_msg);
    // (mean only: src is the source type's table, read only at neighbour ids -- those outside it read as zero rows)
    TORCH_CHECK(mean_only || src->size(0) >= graph->num_rows, "sage_full_aggregate: src needs one row per graph node");
    a.src = src->data_ptr();
    a.n_src = src->size(0);
    a.src_ld = src->stride(0);
    a.src_col = static_cast<int>(src_col);
    a.self_col = static_cast<int>(self_col);
  } else {
    TORCH_CHECK(!combine, "sage_full_aggregate: combine reads a dense src table");
    TORCH_CHECK(feat != nullptr, "sage_full_aggregate: needs a feature table or a src table");
    check_feature_table(feat, d);
    a.feat = feat->tbl;
    a.feat_fp8 = feat->dtype == torch::kUInt8 ? 1 : 0;
  }
  if (combine && has(bias)) {
    check_vec(*bias, torch::kBFloat16, d, "sage_full_aggregate: bias must be a 16-byte aligned bf16 [d] CUDA tensor");
    a.bias = bias->data_ptr();
  }
  a.relu = relu ? 1 : 0;
  launch_sage_full_aggregate(a, cur_stream());
  check_cuda_err("sage_full_aggregate");
}

// num_layers iterations of label propagation over every row of the graph (csrc/cuda/label_prop.cu), from x_0 = base:
//   x_{k+1} = post(alpha * A_norm x_k + (1 - alpha) * base),  post = clamp to [lo, hi], then base on the rows of fixed
// A_norm is 'sym' (deg_i^-1/2 deg_j^-1/2) or 'row' (1 / deg_i) over the unweighted CSR.  base: fp32 [num_rows, cp]
// holding c classes, cp = c rounded up to 4.  Returns a new [num_rows, cp] tensor whose columns >= c are 0 (a copy of
// base when num_layers = 0).  The factors are computed once, two buffers ping-pong, and nothing waits for the device.
static Tensor label_prop(GraphHandle* graph, const Tensor& base, int64_t c, int64_t num_layers, double alpha,
                         const std::string& norm, double lo, double hi, const c10::optional<Tensor>& fixed) {
  TORCH_CHECK(graph != nullptr && graph->tbl.num_parts > 0, "label_prop: graph has no shards");
  c10::cuda::CUDAGuard guard(graph->device);
  TORCH_CHECK(c >= 1 && c <= 512, fmt("label_prop: %lld classes, the kernel takes 1 to 512", static_cast<long long>(c)));
  TORCH_CHECK(norm == "sym" || norm == "row", fmt("label_prop: norm must be 'sym' or 'row', not '%s'", norm.c_str()));
  TORCH_CHECK(std::isfinite(alpha), "label_prop: alpha must be finite");
  TORCH_CHECK(num_layers >= 0, "label_prop: num_layers must be >= 0");
  TORCH_CHECK(!(lo > hi), "label_prop: clamp bounds need lo <= hi");
  const int64_t n = graph->num_rows, cp = (c + 3) / 4 * 4;
  check_rows(base, torch::kFloat32, cp, "label_prop: base must be contiguous, 16-byte aligned fp32 [rows, c rounded up "
                                        "to 4] on the graph's device");
  TORCH_CHECK(base.size(0) == n, fmt("label_prop: base has %lld rows, the graph %lld",
                                     static_cast<long long>(base.size(0)), static_cast<long long>(n)));
  if (has(fixed))
    check_vec(*fixed, torch::kBool, n, "label_prop: fixed must be a contiguous bool [rows] mask on the graph's device");
  if (num_layers == 0) return base.clone();
  const auto f32 = base.options();
  Tensor s = torch::empty({n}, f32);
  Tensor t = norm == "sym" ? torch::empty({n}, f32) : Tensor();
  launch_label_prop_factors(graph->tbl, n, norm == "sym", s.data_ptr<float>(), t.defined() ? t.data_ptr<float>() : nullptr,
                            cur_stream());
  check_cuda_err("label_prop_factors");
  Tensor buf[2] = {torch::empty({n, cp}, f32), num_layers > 1 ? torch::empty({n, cp}, f32) : Tensor()};
  LabelPropArgs a{};
  a.g = graph->tbl;
  a.n = n;
  a.c = static_cast<int>(c);
  a.cp = static_cast<int>(cp);
  a.base = base.data_ptr<float>();
  a.s = s.data_ptr<float>();
  a.t = t.defined() ? t.data_ptr<float>() : nullptr;
  a.alpha = static_cast<float>(alpha);
  a.beta = static_cast<float>(1.0 - alpha);
  a.lo = static_cast<float>(lo);
  a.hi = static_cast<float>(hi);
  a.fixed = has(fixed) ? reinterpret_cast<const uint8_t*>(fixed->data_ptr()) : nullptr;
  for (int64_t k = 0; k < num_layers; ++k) {
    a.x = k == 0 ? a.base : buf[(k - 1) & 1].data_ptr<float>();
    a.out = buf[k & 1].data_ptr<float>();
    launch_label_prop(a, cur_stream());
    check_cuda_err("label_prop");
  }
  return buf[(num_layers - 1) & 1];
}

// Exact top-k of <emb[q], emb[c]> over the candidate ids c of [lo, hi) for every query q (csrc/cuda/link_topk.cu), with
// q itself and the columns of row q of `exclude` never returned.  emb: bf16 [N, d]; queries: int64 [n] in [0, N).
// Returns (ids int64 [n, k], scores fp32 [n, k]), (score desc, id asc), padded with (-1, -inf).  splits = 0 picks the
// candidate split count from n and the SM count; any count gives bitwise identical results.
static std::tuple<Tensor, Tensor> link_topk(const Tensor& emb, const Tensor& queries, int64_t k, int64_t lo, int64_t hi,
                                            GraphHandle* exclude, int64_t splits) {
  TORCH_CHECK(emb.is_cuda(), "link_topk: emb must be a CUDA tensor");
  c10::cuda::CUDAGuard guard(emb.device());
  TORCH_CHECK(emb.dim() == 2, "link_topk: emb must be 2-D [N, d]");
  const int64_t N = emb.size(0), d = emb.size(1);
  TORCH_CHECK(d % 8 == 0 && d >= 8 && d <= 512,
              fmt("link_topk: width %lld, the kernel takes a multiple of 8 in [8, 512]", static_cast<long long>(d)));
  check_rows(emb, torch::kBFloat16, d, "link_topk: emb must be contiguous, 16-byte aligned bf16 [N, d]");
  TORCH_CHECK(k >= 1 && k <= 128, fmt("link_topk: k = %lld, the kernel takes 1 to 128", static_cast<long long>(k)));
  TORCH_CHECK(lo >= 0 && lo <= hi && hi <= N,
              fmt("link_topk: candidate range [%lld, %lld) is not inside [0, %lld)", static_cast<long long>(lo),
                  static_cast<long long>(hi), static_cast<long long>(N)));
  TORCH_CHECK(hi - lo < (int64_t(1) << 31), "link_topk: at most 2^31 - 1 candidates");
  TORCH_CHECK(N < (int64_t(1) << 32) - 1, "link_topk: at most 2^32 - 2 nodes");
  TORCH_CHECK(queries.dim() == 1, "link_topk: queries must be 1-D");
  check_ids(queries, "link_topk: queries must be contiguous int64 on emb's device");
  TORCH_CHECK(splits >= 0, "link_topk: splits must be >= 0 (0: chosen from n)");
  if (exclude != nullptr)
    TORCH_CHECK(exclude->tbl.num_parts == 0 || exclude->device == emb.get_device(),
                "link_topk: the exclusion graph must live on emb's device");
  const int64_t n = queries.numel();
  const auto i64 = queries.options();
  Tensor ids = torch::full({n, k}, -1, i64);
  Tensor scores = torch::full({n, k}, -std::numeric_limits<float>::infinity(), emb.options().dtype(torch::kFloat32));
  if (n == 0) return {ids, scores};
  const int64_t qmin = queries.min().item<int64_t>(), qmax = queries.max().item<int64_t>();
  TORCH_CHECK(qmin >= 0 && qmax < N, fmt("link_topk: query ids must lie in [0, %lld), got [%lld, %lld]",
                                         static_cast<long long>(N), static_cast<long long>(qmin),
                                         static_cast<long long>(qmax)));
  if (hi == lo) return {ids, scores};

  int smem_optin = 0;
  cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, emb.get_device());
  const int stages = link_topk_stages(static_cast<int>(d), static_cast<int>(k), static_cast<size_t>(smem_optin));
  TORCH_CHECK(stages > 0, "link_topk: the device has too little shared memory for this width and k");
  const int64_t q_tiles = (n + 63) / 64, c_tiles = (hi - lo + 63) / 64;
  TORCH_CHECK(q_tiles < (int64_t(1) << 31), "link_topk: too many queries");
  if (splits == 0) {   // one wave: every resident CTA slot busy, as few splits as that takes
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, emb.get_device());
    const int64_t slots = static_cast<int64_t>(sms) * link_topk_ctas_per_sm(static_cast<int>(d), static_cast<int>(k), stages);
    splits = std::max<int64_t>(1, std::min<int64_t>(64, slots / q_tiles));
  }
  splits = std::min(splits, c_tiles);
  TORCH_CHECK(splits <= 65535, "link_topk: at most 65535 splits");
  const int64_t per = (c_tiles + splits - 1) / splits;
  splits = (c_tiles + per - 1) / per;   // no empty split

  Tensor qrows = emb.index_select(0, queries);
  Tensor part = torch::empty({splits, n, k}, i64);
  LinkTopkLaunch L{};
  int rc = make_tmap_bf16_2d(L.maps[0], qrows.data_ptr(), n, d, d, 64, 64);
  TORCH_CHECK(rc == 0, fmt("link_topk: cuTensorMapEncodeTiled failed for the query rows (rc=%d)", rc));
  rc = make_tmap_bf16_2d(L.maps[1], static_cast<const at::BFloat16*>(emb.data_ptr()) + lo * d, hi - lo, d, d, 64, 64);
  TORCH_CHECK(rc == 0, fmt("link_topk: cuTensorMapEncodeTiled failed for the candidate rows (rc=%d)", rc));
  LinkTopkArgs& a = L.args;
  if (exclude != nullptr) a.g = exclude->tbl;
  else a.g.num_parts = 0;
  a.queries = queries.data_ptr<int64_t>();
  a.n = n;
  a.lo = lo;
  a.hi = hi;
  a.d = static_cast<int>(d);
  a.k = static_cast<int>(k);
  a.part_keys = part.data_ptr<int64_t>();
  a.ids = ids.data_ptr<int64_t>();
  a.scores = scores.data_ptr<float>();
  L.splits = static_cast<int>(splits);
  L.tiles_per_split = static_cast<int>(per);
  L.stages = stages;
  launch_link_topk(L, cur_stream());
  check_cuda_err("link_topk");
  return {ids, scores};
}

static void add_block_f32(const Tensor& dA, int64_t col, int64_t d, const Tensor& counters, int64_t n_hops, Tensor dH) {
  c10::cuda::CUDAGuard guard(dA.device());
  TORCH_CHECK(d % 8 == 0, "add_block_f32: d must be a multiple of 8");
  check_block(dA, torch::kBFloat16, col, d,
              "add_block_f32: dA must be a bf16 view with 16-byte aligned rows holding columns [col, col + d)");
  check_rows(dH, torch::kFloat32, d, "add_block_f32: dH must be contiguous fp32 [rows, d]");
  check_counters(counters, n_hops, "add_block_f32: counters must be int32 [> n_hops] on the device");
  launch_add_block_f32(dA.data_ptr(), dA.stride(0), col, d, counters.data_ptr<int32_t>(), n_hops,
                       std::min<int64_t>(dA.size(0), dH.size(0)), dH.data_ptr<float>(), cur_stream());
  check_cuda_err("add_block_f32");
}

// Atomics-free backward of the mean aggregation over the arena's transposed adjacency
static void sage_gather_bwd(const Tensor& dA, int64_t d, SamplerArena& ar, int64_t n_hops_targets,
                            const c10::optional<Tensor>& Z, Tensor dPre, const c10::optional<Tensor>& colsum,
                            bool prezeroed, double gscale) {
  c10::cuda::CUDAGuard guard(dA.device());
  TORCH_CHECK(ar.tr_hops >= n_hops_targets && n_hops_targets >= 1, "enable_transpose(n_hops) covers too few hops");
  TORCH_CHECK(ar.device == dA.get_device(), "sage_gather_bwd: dA must be on the arena's device");
  check_sage_width(d, "sage_gather_bwd: d must be a multiple of 8 in [8, 1024]");
  check_rows(dA, torch::kBFloat16, 2 * d, "sage_gather_bwd: dA must be contiguous bf16 [rows, 2d]");
  check_rows(dPre, torch::kBFloat16, d, "sage_gather_bwd: dPre must be contiguous bf16 [rows, d]");
  TORCH_CHECK(dPre.size(0) <= ar.cap_nodes, "dPre has more rows than the arena has nodes");
  SageGatherBwdArgs a{};
  a.dA = dA.data_ptr();
  a.d = static_cast<int>(d);
  a.cum = ar.counters.data_ptr<int32_t>();
  a.n_hops_targets = static_cast<int>(n_hops_targets);
  a.cap_targets = static_cast<int>(dA.size(0));
  a.cap_src = static_cast<int>(dPre.size(0));
  a.deg = ar.deg.data_ptr<int32_t>();
  a.off = ar.tr_off.data_ptr<int32_t>();
  a.cnt_upto = ar.tr_cnt.data_ptr<int32_t>() + (n_hops_targets - 1) * ar.cap_nodes;
  a.tgt = ar.tr_tgt.data_ptr<int32_t>();
  a.meta = ar.tr_meta.data_ptr<int32_t>();
  a.meta_inv = ar.tr_meta_inv.data_ptr<float>();
  a.Z = nullptr;
  if (has(Z)) {
    check_rows(*Z, torch::kBFloat16, d, "sage_gather_bwd: Z must be contiguous bf16 [rows, d]");
    TORCH_CHECK(Z->size(0) >= dPre.size(0), "sage_gather_bwd: Z has fewer rows than dPre");
    a.Z = Z->data_ptr();
  }
  a.dPre = dPre.data_ptr();
  a.colsum = nullptr;
  if (has(colsum)) {
    TORCH_CHECK(d % 4 == 0 && colsum->numel() >= d, "colsum: fp32 [d], 16-byte aligned");
    check_vec(*colsum, torch::kFloat32, colsum->numel(), "colsum: fp32 [d], 16-byte aligned");
    a.colsum = colsum->data_ptr<float>();
  }
  a.colsum_prezeroed = prezeroed ? 1 : 0;
  a.gscale = static_cast<float>(gscale);
  launch_sage_gather_bwd(a, cur_stream());
  check_cuda_err("sage_gather_bwd");
}

static void relu_bwd_cast(const Tensor& dH, const Tensor& Z, const Tensor& counters, int64_t n_hops,
                          Tensor dPre, const c10::optional<Tensor>& colsum, bool prezeroed, double gscale, bool relu) {
  c10::cuda::CUDAGuard guard(dH.device());
  const int64_t d = dPre.dim() == 2 ? dPre.size(1) : 0;
  TORCH_CHECK(d % 8 == 0, "relu_bwd_cast: width must be a multiple of 8");
  check_rows(dH, torch::kFloat32, d, "relu_bwd_cast: dH must be contiguous fp32 [rows, d]");
  check_rows(Z, torch::kBFloat16, d, "relu_bwd_cast: Z must be contiguous bf16 [rows, d]");
  check_rows(dPre, torch::kBFloat16, d, "relu_bwd_cast: dPre must be contiguous bf16 [rows, d]");
  TORCH_CHECK(dPre.size(0) <= dH.size(0) && dPre.size(0) <= Z.size(0), "relu_bwd_cast: dH / Z have fewer rows than dPre");
  check_counters(counters, n_hops, "relu_bwd_cast: counters must be int32 [> n_hops] on the device");
  if (has(colsum)) check_vec(*colsum, torch::kFloat32, d, "relu_bwd_cast: colsum must be fp32 [d]");
  launch_relu_bwd_cast(dH.data_ptr<float>(), Z.data_ptr(), counters.data_ptr<int32_t>(), n_hops, dPre.size(0), d,
                       dPre.data_ptr(), opt_ptr<float>(colsum), cur_stream(), prezeroed, static_cast<float>(gscale), relu);
  check_cuda_err("relu_bwd_cast");
}

// ---- relational GAT (cuda/gat.cu) -------------------------------------------------------------------------------
// H = heads * C must be a multiple of 64 in [64, 1024] (the lane-group dispatch covers 1024 columns, see
// check_sage_width) with C a multiple of 8 (one 16-byte vector never straddles two heads).
static void check_gat_width(int64_t H, int64_t heads) {
  TORCH_CHECK(H % 64 == 0 && H >= 64 && H <= 1024 && heads >= 1 && H % heads == 0 && (H / heads) % 8 == 0,
              "gat: H must be a multiple of 64 in [64, 1024] and heads must divide H into head widths C with C % 8 == 0");
}

static void gat_fill_hops(const std::vector<Tensor>& ell, const std::vector<int64_t>& ks, const std::vector<Tensor>& bufs,
                          int64_t heads, float** out) {
  TORCH_CHECK(bufs.size() == ell.size(), "gat: one alpha buffer per hop");
  for (size_t h = 0; h < 4; ++h) out[h] = nullptr;
  for (size_t h = 0; h < bufs.size(); ++h) {
    TORCH_CHECK(on_dev(bufs[h]) && bufs[h].scalar_type() == torch::kFloat32 && bufs[h].is_contiguous() &&
                bufs[h].numel() >= ell[h].numel() * heads, "gat: alpha buffers must be fp32 [ELL slots of the hop, heads]");
    out[h] = bufs[h].data_ptr<float>();
  }
}

// scores of the source rows (P0, rows < counters0[idx0]) and, optionally, of the target rows (P1)
static void gat_scores(const Tensor& P0, const Tensor& att0, Tensor out0, const Tensor& counters0, int64_t idx0,
                       const c10::optional<Tensor>& P1, const c10::optional<Tensor>& att1,
                       const c10::optional<Tensor>& out1, const c10::optional<Tensor>& counters1, int64_t idx1,
                       const c10::optional<Tensor>& zero, int64_t heads) {
  c10::cuda::CUDAGuard guard(P0.device());
  const int64_t H = P0.size(1);
  check_gat_width(H, heads);
  GatScoreArgs a{};
  a.H = H; a.heads = heads;
  check_rows(P0, torch::kBFloat16, H, "gat_scores: P must be contiguous bf16 [rows, H]");
  check_rows(out0, torch::kFloat32, heads, "gat_scores: out must be contiguous fp32 [rows, heads]");
  check_vec(att0, torch::kBFloat16, H, "gat_scores: att must be 16-byte aligned bf16 [H]");
  TORCH_CHECK(out0.size(0) >= P0.size(0), "gat_scores: out has fewer rows than P");
  check_counters(counters0, idx0, "gat_scores: counters must be int32 [> idx] on the device");
  a.P[0] = P0.data_ptr(); a.att[0] = att0.data_ptr(); a.out[0] = out0.data_ptr<float>();
  a.cum[0] = counters0.data_ptr<int32_t>(); a.idx[0] = idx0; a.cap[0] = P0.size(0);
  if (has(P1)) {
    TORCH_CHECK(has(att1) && has(out1) && has(counters1), "gat_scores: the second set needs P, att, out and counters");
    check_rows(*P1, torch::kBFloat16, H, "gat_scores: P must be contiguous bf16 [rows, H]");
    check_rows(*out1, torch::kFloat32, heads, "gat_scores: out must be contiguous fp32 [rows, heads]");
    check_vec(*att1, torch::kBFloat16, H, "gat_scores: att must be 16-byte aligned bf16 [H]");
    TORCH_CHECK(out1->size(0) >= P1->size(0), "gat_scores: out has fewer rows than P");
    check_counters(*counters1, idx1, "gat_scores: counters must be int32 [> idx] on the device");
    a.P[1] = P1->data_ptr(); a.att[1] = att1->data_ptr(); a.out[1] = out1->data_ptr<float>();
    a.cum[1] = counters1->data_ptr<int32_t>(); a.idx[1] = idx1; a.cap[1] = P1->size(0);
  } else {
    a.cum[1] = a.cum[0];
  }
  if (has(zero)) {
    check_rows(*zero, torch::kFloat32, heads, "gat_scores: zero must be contiguous fp32 [rows, heads]");
    TORCH_CHECK(zero->size(0) >= P0.size(0), "gat_scores: zero has fewer rows than P");
    a.zero = zero->data_ptr<float>();
  }
  launch_gat_scores(a, cur_stream());
  check_cuda_err("gat_scores");
}

// Returns nothing; writes alpha, and acc (first/last false) or Z (last).
static void gat_aggregate(const Tensor& P, const Tensor& as, const Tensor& ad, int64_t heads, const Tensor& counters,
                          int64_t n_hops_targets, const std::vector<Tensor>& ell, const std::vector<int64_t>& ks,
                          const Tensor& deg, const std::vector<Tensor>& alpha, const c10::optional<Tensor>& acc,
                          bool first, bool last, const c10::optional<Tensor>& bias, bool act, double p, int64_t seed,
                          int64_t layer, const c10::optional<Tensor>& step_dev, const c10::optional<Tensor>& Z) {
  c10::cuda::CUDAGuard guard(P.device());
  const int64_t H = P.size(1);
  check_gat_width(H, heads);
  check_rows(P, torch::kBFloat16, H, "gat_aggregate: P must be contiguous bf16 [rows, H]");
  check_rows(as, torch::kFloat32, heads, "gat_aggregate: as must be contiguous fp32 [rows, heads]");
  check_rows(ad, torch::kFloat32, heads, "gat_aggregate: ad must be contiguous fp32 [rows, heads]");
  TORCH_CHECK(as.size(0) >= P.size(0), "gat_aggregate: as has fewer rows than P");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "gat_aggregate: dropout p must be in [0, 1)");
  check_counters(counters, n_hops_targets, "gat_aggregate: counters must be int32 [> n_hops_targets] on the device");
  GatAggArgs a{};
  a.P = P.data_ptr(); a.as = as.data_ptr<float>(); a.ad = ad.data_ptr<float>();
  a.H = H; a.heads = heads;
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  int64_t cap = ad.size(0);
  a.deg = fill_ell(ell, ks, deg, a.ell, a.k);
  gat_fill_hops(ell, ks, alpha, heads, a.alpha);
  a.first = first ? 1 : 0; a.last = last ? 1 : 0;
  if (!(first && last)) {
    TORCH_CHECK(has(acc), "gat_aggregate: a relation sum over several launches needs acc");
    check_rows(*acc, torch::kFloat32, H, "gat_aggregate: acc must be contiguous fp32 [rows, H]");
    cap = std::min<int64_t>(cap, acc->size(0));
    a.acc = acc->data_ptr<float>();
  }
  if (last) {
    TORCH_CHECK(has(Z), "gat_aggregate: the last relation writes Z");
    check_rows(*Z, torch::kBFloat16, H, "gat_aggregate: Z must be contiguous bf16 [rows, H]");
    cap = std::min<int64_t>(cap, Z->size(0));
    a.z = Z->data_ptr();
    if (has(bias)) {
      TORCH_CHECK(bias->numel() % H == 0, "gat_aggregate: bias must be 16-byte aligned bf16 [n_bias * H]");
      check_vec(*bias, torch::kBFloat16, bias->numel(), "gat_aggregate: bias must be 16-byte aligned bf16 [n_bias * H]");
      a.bias = bias->data_ptr();
      a.n_bias = bias->numel() / H;
    }
    a.act = act ? 1 : 0;
    a.thresh16 = static_cast<uint32_t>(std::min(std::max(p, 0.0), 1.0) * 65536.0);
    a.dscale = static_cast<float>(1.0 / (1.0 - p));
    a.seed = static_cast<uint64_t>(seed);
    a.layer = layer;
    if (has(step_dev)) {
      check_counters(*step_dev, 0, "gat_aggregate: int32 step_dev");
      a.step_dev = step_dev->data_ptr<int32_t>();
    }
  }
  a.cap_targets = cap;
  launch_gat_aggregate(a, cur_stream());
  check_cuda_err("gat_aggregate");
}

static void gat_backward(const Tensor& G, const Tensor& P, int64_t heads, const Tensor& counters, int64_t n_hops_targets,
                         const std::vector<Tensor>& ell, const std::vector<int64_t>& ks, const Tensor& deg,
                         const std::vector<Tensor>& alpha, const std::vector<Tensor>& dal, Tensor dP, Tensor da_src,
                         Tensor da_dst) {
  c10::cuda::CUDAGuard guard(G.device());
  const int64_t H = P.size(1);
  check_gat_width(H, heads);
  check_rows(G, torch::kBFloat16, H, "gat_backward: G must be contiguous bf16 [rows, H]");
  check_rows(P, torch::kBFloat16, H, "gat_backward: P must be contiguous bf16 [rows, H]");
  check_rows(dP, torch::kFloat32, H, "gat_backward: dP must be contiguous fp32 [rows, H]");
  check_rows(da_src, torch::kFloat32, heads, "gat_backward: da_src must be contiguous fp32 [rows, heads]");
  check_rows(da_dst, torch::kFloat32, heads, "gat_backward: da_dst must be contiguous fp32 [rows, heads]");
  TORCH_CHECK(dP.size(0) >= P.size(0) && da_src.size(0) >= P.size(0), "gat_backward: dP / da_src have fewer rows than P");
  check_counters(counters, n_hops_targets, "gat_backward: counters must be int32 [> n_hops_targets] on the device");
  GatBwdArgs a{};
  a.G = G.data_ptr(); a.P = P.data_ptr(); a.H = H; a.heads = heads;
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  a.cap_targets = std::min<int64_t>(G.size(0), da_dst.size(0));
  a.deg = fill_ell(ell, ks, deg, a.ell, a.k);
  float* al[4];
  gat_fill_hops(ell, ks, alpha, heads, al);
  for (int h = 0; h < 4; ++h) a.alpha[h] = al[h];
  gat_fill_hops(ell, ks, dal, heads, a.dal);
  a.dP = dP.data_ptr<float>(); a.da_src = da_src.data_ptr<float>(); a.da_dst = da_dst.data_ptr<float>();
  launch_gat_backward(a, cur_stream());
  check_cuda_err("gat_backward");
}

// Source segment: P_src / dP_src / da_src / att_src -> dPb_src (+ g_att_src).  Destination: a separate projection
// P_dst -> dPb_dst, or (P_dst None) folded into the source rows, which then start with the target rows.
static void gat_score_bwd(const Tensor& P_src, const Tensor& dP_src, const Tensor& da_src, const Tensor& att_src,
                          Tensor g_att_src, Tensor dPb_src, const Tensor& ctr_src, int64_t idx_src, const Tensor& da_dst,
                          const Tensor& att_dst, Tensor g_att_dst, const Tensor& ctr_dst, int64_t idx_dst,
                          const c10::optional<Tensor>& P_dst, const c10::optional<Tensor>& dPb_dst, int64_t heads) {
  c10::cuda::CUDAGuard guard(P_src.device());
  const int64_t H = P_src.size(1);
  check_gat_width(H, heads);
  check_rows(P_src, torch::kBFloat16, H, "gat_score_bwd: P must be contiguous bf16 [rows, H]");
  check_rows(dP_src, torch::kFloat32, H, "gat_score_bwd: dP must be contiguous fp32 [rows, H]");
  check_rows(dPb_src, torch::kBFloat16, H, "gat_score_bwd: dPb must be contiguous bf16 [rows, H]");
  check_rows(da_src, torch::kFloat32, heads, "gat_score_bwd: da must be contiguous fp32 [rows, heads]");
  check_rows(da_dst, torch::kFloat32, heads, "gat_score_bwd: da must be contiguous fp32 [rows, heads]");
  TORCH_CHECK(dP_src.size(0) >= P_src.size(0) && dPb_src.size(0) >= P_src.size(0) && da_src.size(0) >= P_src.size(0),
              "gat_score_bwd: source buffers have fewer rows than P");
  for (const Tensor* t : {&att_src, &att_dst})
    check_vec(*t, torch::kBFloat16, H, "gat_score_bwd: att must be 16-byte aligned bf16 [H]");
  for (const Tensor* t : {&g_att_src, &g_att_dst})
    check_vec(*t, torch::kFloat32, H, "gat_score_bwd: attention gradients must be fp32 [H]");
  check_counters(ctr_src, idx_src, "gat_score_bwd: ctr_src must be int32 [> idx_src] on the device");
  check_counters(ctr_dst, idx_dst, "gat_score_bwd: ctr_dst must be int32 [> idx_dst] on the device");
  GatScoreBwdArgs a{};
  a.H = H; a.heads = heads;
  auto& s = a.seg[0];
  s.P = P_src.data_ptr(); s.dP = dP_src.data_ptr<float>(); s.da0 = da_src.data_ptr<float>();
  s.att0 = att_src.data_ptr(); s.gatt0 = g_att_src.data_ptr<float>(); s.dPb = dPb_src.data_ptr();
  s.cum = ctr_src.data_ptr<int32_t>(); s.idx = idx_src; s.cap = P_src.size(0);
  if (has(P_dst)) {
    TORCH_CHECK(has(dPb_dst), "gat_score_bwd: a separate destination projection needs dPb_dst");
    check_rows(*P_dst, torch::kBFloat16, H, "gat_score_bwd: P must be contiguous bf16 [rows, H]");
    check_rows(*dPb_dst, torch::kBFloat16, H, "gat_score_bwd: dPb must be contiguous bf16 [rows, H]");
    TORCH_CHECK(dPb_dst->size(0) >= P_dst->size(0) && da_dst.size(0) >= P_dst->size(0),
                "gat_score_bwd: destination buffers have fewer rows than P");
    auto& d = a.seg[1];
    d.P = P_dst->data_ptr(); d.da0 = da_dst.data_ptr<float>(); d.att0 = att_dst.data_ptr();
    d.gatt0 = g_att_dst.data_ptr<float>(); d.dPb = dPb_dst->data_ptr();
    d.cum = ctr_dst.data_ptr<int32_t>(); d.idx = idx_dst; d.cap = P_dst->size(0);
  } else {
    s.da1 = da_dst.data_ptr<float>(); s.att1 = att_dst.data_ptr(); s.gatt1 = g_att_dst.data_ptr<float>();
    s.cum1 = ctr_dst.data_ptr<int32_t>(); s.idx1 = idx_dst;
  }
  launch_gat_score_bwd(a, cur_stream());
  check_cuda_err("gat_score_bwd");
}

static void gat_act_bwd(const c10::optional<Tensor>& dH, const c10::optional<Tensor>& Z, Tensor dPre,
                        const Tensor& counters, int64_t n_hops, double p, int64_t seed, int64_t layer,
                        const c10::optional<Tensor>& step_dev, const c10::optional<Tensor>& bias_g) {
  c10::cuda::CUDAGuard guard(dPre.device());
  const int64_t d = dPre.size(1);
  TORCH_CHECK(d % 64 == 0 && d >= 64 && d <= 1024, "gat_act_bwd: width must be a multiple of 64 in [64, 1024]");
  check_rows(dPre, torch::kBFloat16, d, "gat_act_bwd: dPre must be contiguous bf16 [rows, d]");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "gat_act_bwd: dropout p must be in [0, 1)");
  check_counters(counters, n_hops, "gat_act_bwd: counters must be int32 [> n_hops] on the device");
  GatActBwdArgs a{};
  a.dPre = dPre.data_ptr(); a.cum = counters.data_ptr<int32_t>(); a.n_hops = n_hops; a.cap = dPre.size(0); a.d = d;
  if (has(dH)) {
    TORCH_CHECK(has(Z), "gat_act_bwd: the activation backward needs Z");
    check_rows(*dH, torch::kFloat32, d, "gat_act_bwd: dH must be contiguous fp32 [rows, d]");
    check_rows(*Z, torch::kBFloat16, d, "gat_act_bwd: Z must be contiguous bf16 [rows, d]");
    TORCH_CHECK(dH->size(0) >= dPre.size(0) && Z->size(0) >= dPre.size(0), "gat_act_bwd: dH / Z have fewer rows than dPre");
    a.dH = dH->data_ptr<float>(); a.Z = Z->data_ptr();
  }
  a.slope = 0.01f;
  a.thresh16 = static_cast<uint32_t>(p * 65536.0);
  a.dscale = static_cast<float>(1.0 / (1.0 - p));
  a.seed = static_cast<uint64_t>(seed);
  a.layer = layer;
  if (has(step_dev)) {
    check_counters(*step_dev, 0, "gat_act_bwd: int32 step_dev");
    a.step_dev = step_dev->data_ptr<int32_t>();
  }
  if (has(bias_g)) {
    TORCH_CHECK(bias_g->numel() % d == 0 && bias_g->numel() > 0, "gat_act_bwd: bias_g must be fp32 [n_bias * d]");
    check_vec(*bias_g, torch::kFloat32, bias_g->numel(), "gat_act_bwd: bias_g must be fp32 [n_bias * d]");
    a.bias_g = bias_g->data_ptr<float>();
    a.n_bias = bias_g->numel() / d;
  }
  launch_gat_act_bwd(a, cur_stream());
  check_cuda_err("gat_act_bwd");
}

// ---- HGT (cuda/hgt.cu) ------------------------------------------------------------------------------------------
// Per relation into the destination type: kv = the source rows [K | Q | V] (bf16 [rows, 3H]), prior (fp32 [heads]),
// the per-hop ELL blocks and fan-outs, deg, and the per-hop alpha buffers.
template <typename RelT>
static void hgt_fill_rels(RelT* rel, int64_t H, int64_t heads, const std::vector<Tensor>& kv,
                          const std::vector<Tensor>& prior, const std::vector<std::vector<Tensor>>& ell,
                          const std::vector<std::vector<int64_t>>& ks, const std::vector<Tensor>& deg,
                          const std::vector<std::vector<Tensor>>& alpha, int64_t n_hops) {
  const size_t R = kv.size();
  TORCH_CHECK(R >= 1 && R <= static_cast<size_t>(kHgtMaxRel), "hgt: a destination type takes 1 to 8 relations");
  TORCH_CHECK(prior.size() == R && ell.size() == R && ks.size() == R && deg.size() == R && alpha.size() == R,
              "hgt: kv, prior, ell, ks, deg and alpha need one entry per relation");
  for (size_t r = 0; r < R; ++r) {
    check_rows(kv[r], torch::kBFloat16, 3 * H, "hgt: source rows must be contiguous bf16 [rows, 3H] = [K | Q | V]");
    check_vec(prior[r], torch::kFloat32, heads, "hgt: prior must be fp32 [heads]");
    TORCH_CHECK(static_cast<int64_t>(ell[r].size()) == n_hops, "hgt: one ELL block per target hop");
    rel[r].kv = kv[r].data_ptr();
    rel[r].prior = prior[r].data_ptr<float>();
    rel[r].deg = fill_ell(ell[r], ks[r], deg[r], rel[r].ell, rel[r].k);
    float* al[4];
    gat_fill_hops(ell[r], ks[r], alpha[r], heads, al);
    for (int h = 0; h < 4; ++h) rel[r].alpha[h] = al[h];
  }
}

static void check_hgt_width(int64_t H, int64_t heads) {
  TORCH_CHECK(H % 64 == 0 && H >= 64 && H <= 1024 && heads >= 1 && H % heads == 0 && (H / heads) % 8 == 0,
              "hgt: H must be a multiple of 64 in [64, 1024] and heads must divide H into head widths D with D % 8 == 0");
}

static void hgt_attention(const Tensor& qq, Tensor u, int64_t heads, const Tensor& counters, int64_t n_hops_targets,
                          const std::vector<Tensor>& kv, const std::vector<Tensor>& prior,
                          const std::vector<std::vector<Tensor>>& ell, const std::vector<std::vector<int64_t>>& ks,
                          const std::vector<Tensor>& deg, const std::vector<std::vector<Tensor>>& alpha) {
  c10::cuda::CUDAGuard guard(qq.device());
  const int64_t R = static_cast<int64_t>(kv.size());
  TORCH_CHECK(R >= 1 && R <= kHgtMaxRel, "hgt: a destination type takes 1 to 8 relations");
  TORCH_CHECK(qq.dim() == 2 && qq.size(1) % R == 0, "hgt_attention: qq must be [rows, n_rel * H]");
  const int64_t H = qq.size(1) / R;
  check_hgt_width(H, heads);
  check_rows(qq, torch::kBFloat16, R * H, "hgt_attention: qq must be contiguous bf16 [rows, n_rel * H]");
  check_rows(u, torch::kBFloat16, R * H, "hgt_attention: u must be contiguous bf16 [rows, n_rel * H]");
  check_counters(counters, n_hops_targets, "hgt_attention: counters must be int32 [> n_hops_targets] on the device");
  HgtAttnArgs a{};
  a.qq = qq.data_ptr(); a.u = u.data_ptr();
  a.H = H; a.heads = heads; a.n_rel = R; a.kv_ld = 3 * H; a.v_off = 2 * H;
  a.scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(H / heads)));
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  a.cap_targets = std::min<int64_t>(qq.size(0), u.size(0));
  hgt_fill_rels(a.rel, H, heads, kv, prior, ell, ks, deg, alpha, n_hops_targets);
  launch_hgt_attention(a, cur_stream());
  check_cuda_err("hgt_attention");
}

static void hgt_attention_bwd(const Tensor& du, const Tensor& qq, Tensor dqq, int64_t heads, const Tensor& counters,
                              int64_t n_hops_targets, const std::vector<Tensor>& kv, const std::vector<Tensor>& prior,
                              const std::vector<std::vector<Tensor>>& ell,
                              const std::vector<std::vector<int64_t>>& ks, const std::vector<Tensor>& deg,
                              const std::vector<std::vector<Tensor>>& alpha, const std::vector<std::vector<Tensor>>& dal,
                              const std::vector<Tensor>& dkv, const std::vector<Tensor>& dprior) {
  c10::cuda::CUDAGuard guard(qq.device());
  const int64_t R = static_cast<int64_t>(kv.size());
  TORCH_CHECK(R >= 1 && R <= kHgtMaxRel, "hgt: a destination type takes 1 to 8 relations");
  TORCH_CHECK(qq.dim() == 2 && qq.size(1) % R == 0, "hgt_attention_bwd: qq must be [rows, n_rel * H]");
  const int64_t H = qq.size(1) / R;
  check_hgt_width(H, heads);
  check_rows(qq, torch::kBFloat16, R * H, "hgt_attention_bwd: qq must be contiguous bf16 [rows, n_rel * H]");
  check_rows(du, torch::kBFloat16, R * H, "hgt_attention_bwd: du must be contiguous bf16 [rows, n_rel * H]");
  check_rows(dqq, torch::kBFloat16, R * H, "hgt_attention_bwd: dqq must be contiguous bf16 [rows, n_rel * H]");
  TORCH_CHECK(dal.size() == static_cast<size_t>(R) && dkv.size() == static_cast<size_t>(R) &&
              dprior.size() == static_cast<size_t>(R), "hgt_attention_bwd: dal, dkv and dprior need one entry per relation");
  check_counters(counters, n_hops_targets, "hgt_attention_bwd: counters must be int32 [> n_hops_targets] on the device");
  HgtAttnBwdArgs a{};
  a.du = du.data_ptr(); a.qq = qq.data_ptr(); a.dqq = dqq.data_ptr();
  a.H = H; a.heads = heads; a.n_rel = R; a.kv_ld = 3 * H; a.v_off = 2 * H;
  a.scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(H / heads)));
  a.cum = counters.data_ptr<int32_t>();
  a.n_hops_targets = n_hops_targets;
  a.cap_targets = std::min<int64_t>(std::min<int64_t>(qq.size(0), du.size(0)), dqq.size(0));
  hgt_fill_rels(a.rel, H, heads, kv, prior, ell, ks, deg, alpha, n_hops_targets);
  for (int64_t r = 0; r < R; ++r) {
    TORCH_CHECK(dal[r].size() == ell[r].size(), "hgt_attention_bwd: one dal buffer per hop");
    for (size_t h = 0; h < 4; ++h) a.rel[r].dal[h] = nullptr;
    for (size_t h = 0; h < dal[r].size(); ++h) {
      TORCH_CHECK(on_dev(dal[r][h]) && dal[r][h].scalar_type() == torch::kFloat32 && dal[r][h].is_contiguous() &&
                  dal[r][h].numel() >= 2 * ell[r][h].numel() * heads &&
                  reinterpret_cast<uintptr_t>(dal[r][h].data_ptr()) % 8 == 0,
                  "hgt_attention_bwd: dal buffers must be fp32 [ELL slots of the hop, heads, 2]");
      a.rel[r].dal[h] = dal[r][h].data_ptr<float>();
    }
    check_rows(dkv[r], torch::kFloat32, 2 * H, "hgt_attention_bwd: dkv must be contiguous fp32 [rows, 2H]");
    TORCH_CHECK(dkv[r].size(0) >= kv[r].size(0), "hgt_attention_bwd: dkv has fewer rows than the source rows");
    check_vec(dprior[r], torch::kFloat32, heads, "hgt_attention_bwd: dprior must be fp32 [heads]");
    a.rel[r].dkv = dkv[r].data_ptr<float>();
    a.rel[r].dprior = dprior[r].data_ptr<float>();
  }
  launch_hgt_attention_bwd(a, cur_stream());
  check_cuda_err("hgt_attention_bwd");
}

// ---- full-neighbourhood attention of the heterogeneous inference (cuda/hetero_infer.cu) ---------------------------
// R-GAT, one relation: targets are the global rows [r0, r1) of `graph` (its columns index P / as), acc and Z are
// chunk rows.  first / last / bias / act as in gat_aggregate, without dropout.
static void gat_full_aggregate(GraphHandle* graph, const Tensor& P, const Tensor& as, const Tensor& ad, int64_t heads,
                               int64_t r0, int64_t r1, const c10::optional<Tensor>& acc, bool first, bool last,
                               const c10::optional<Tensor>& bias, bool act, const c10::optional<Tensor>& Z) {
  c10::cuda::CUDAGuard guard(P.device());
  TORCH_CHECK(graph != nullptr && graph->tbl.num_parts > 0, "gat_full_aggregate: graph has no shards");
  TORCH_CHECK(0 <= r0 && r0 <= r1 && r1 <= graph->num_rows, "gat_full_aggregate: rows [r0, r1) outside the graph");
  const int64_t H = P.size(1);
  check_gat_width(H, heads);
  check_rows(P, torch::kBFloat16, H, "gat_full_aggregate: P must be contiguous bf16 [rows, H]");
  check_rows(as, torch::kFloat32, heads, "gat_full_aggregate: as must be contiguous fp32 [rows, heads]");
  check_rows(ad, torch::kFloat32, heads, "gat_full_aggregate: ad must be contiguous fp32 [rows, heads]");
  TORCH_CHECK(as.size(0) >= P.size(0), "gat_full_aggregate: as has fewer rows than P");
  TORCH_CHECK(ad.size(0) >= r1, "gat_full_aggregate: ad needs a row for every target id below r1");
  GatFullAggArgs a{};
  a.g = graph->tbl;
  a.P = P.data_ptr(); a.as = as.data_ptr<float>(); a.ad = ad.data_ptr<float>();
  a.n_src = P.size(0);
  a.H = H; a.heads = heads;
  a.r0 = r0; a.r1 = r1;
  a.first = first ? 1 : 0; a.last = last ? 1 : 0;
  if (!(first && last)) {
    TORCH_CHECK(has(acc), "gat_full_aggregate: a relation sum over several launches needs acc");
    check_rows(*acc, torch::kFloat32, H, "gat_full_aggregate: acc must be contiguous fp32 [rows, H]");
    TORCH_CHECK(acc->size(0) >= r1 - r0, "gat_full_aggregate: acc needs r1 - r0 rows");
    a.acc = acc->data_ptr<float>();
  }
  if (last) {
    TORCH_CHECK(has(Z), "gat_full_aggregate: the last relation writes Z");
    check_rows(*Z, torch::kBFloat16, H, "gat_full_aggregate: Z must be contiguous bf16 [rows, H]");
    TORCH_CHECK(Z->size(0) >= r1 - r0, "gat_full_aggregate: Z needs r1 - r0 rows");
    a.z = Z->data_ptr();
    if (has(bias)) {
      TORCH_CHECK(bias->numel() % H == 0, "gat_full_aggregate: bias must be 16-byte aligned bf16 [n_bias * H]");
      check_vec(*bias, torch::kBFloat16, bias->numel(), "gat_full_aggregate: bias must be 16-byte aligned bf16 [n_bias * H]");
      a.bias = bias->data_ptr();
      a.n_bias = bias->numel() / H;
    }
    a.act = act ? 1 : 0;
  }
  launch_gat_full_aggregate(a, cur_stream());
  check_cuda_err("gat_full_aggregate");
}

// HGT, one destination type: graphs[r] (targets [r0, r1) are its rows) with the source type's [K | Q | V] table kv[r]
// and prior[r]; qq / u are chunk rows [r1 - r0, n_rel * H].
static void hgt_full_attention(const std::vector<GraphHandle*>& graphs, const Tensor& qq, Tensor u, int64_t heads,
                               int64_t r0, int64_t r1, const std::vector<Tensor>& kv, const std::vector<Tensor>& prior) {
  c10::cuda::CUDAGuard guard(qq.device());
  const int64_t R = static_cast<int64_t>(kv.size());
  TORCH_CHECK(R >= 1 && R <= kHgtMaxRel, "hgt: a destination type takes 1 to 8 relations");
  TORCH_CHECK(graphs.size() == static_cast<size_t>(R) && prior.size() == static_cast<size_t>(R),
              "hgt_full_attention: graphs, kv and prior need one entry per relation");
  TORCH_CHECK(qq.dim() == 2 && qq.size(1) % R == 0, "hgt_full_attention: qq must be [rows, n_rel * H]");
  const int64_t H = qq.size(1) / R;
  check_hgt_width(H, heads);
  check_rows(qq, torch::kBFloat16, R * H, "hgt_full_attention: qq must be contiguous bf16 [rows, n_rel * H]");
  check_rows(u, torch::kBFloat16, R * H, "hgt_full_attention: u must be contiguous bf16 [rows, n_rel * H]");
  TORCH_CHECK(0 <= r0 && r0 <= r1 && qq.size(0) >= r1 - r0 && u.size(0) >= r1 - r0,
              "hgt_full_attention: qq and u need r1 - r0 rows");
  HgtFullAttnArgs a{};
  std::vector<GraphTable> tbl(R);
  for (int64_t r = 0; r < R; ++r) {
    TORCH_CHECK(graphs[r] != nullptr && graphs[r]->tbl.num_parts > 0, "hgt_full_attention: graph has no shards");
    TORCH_CHECK(r1 <= graphs[r]->num_rows, "hgt_full_attention: rows [r0, r1) outside a relation graph");
    check_rows(kv[r], torch::kBFloat16, 3 * H, "hgt_full_attention: kv must be contiguous bf16 [rows, 3H]");
    check_vec(prior[r], torch::kFloat32, heads, "hgt_full_attention: prior must be fp32 [heads]");
    tbl[r] = graphs[r]->tbl;
    a.kv[r] = kv[r].data_ptr();
    a.n_src[r] = kv[r].size(0);
    a.prior[r] = prior[r].data_ptr<float>();
  }
  // the relation tables (up to 8 x 776 bytes) go to the device in one stream-ordered copy
  Tensor host = torch::empty({static_cast<int64_t>(R * sizeof(GraphTable))},
                             torch::TensorOptions().dtype(torch::kUInt8).pinned_memory(true));
  std::memcpy(host.data_ptr(), tbl.data(), R * sizeof(GraphTable));
  Tensor dev_tbl = host.to(qq.device(), /*non_blocking=*/true);
  a.g = reinterpret_cast<const GraphTable*>(dev_tbl.data_ptr());
  a.n_rel = R; a.H = H; a.heads = heads; a.kv_ld = 3 * H; a.v_off = 2 * H;
  a.scale = static_cast<float>(1.0 / std::sqrt(static_cast<double>(H / heads)));
  a.qq = qq.data_ptr(); a.u = u.data_ptr();
  a.r0 = r0; a.r1 = r1;
  launch_hgt_full_attention(a, cur_stream());
  check_cuda_err("hgt_full_attention");
}

static void hgt_gelu(const Tensor& X, Tensor Y, const Tensor& counters, int64_t n_hops, const c10::optional<Tensor>& dY) {
  c10::cuda::CUDAGuard guard(X.device());
  const int64_t d = X.size(1);
  TORCH_CHECK(d % 8 == 0, "hgt_gelu: width must be a multiple of 8");
  check_rows(X, torch::kBFloat16, d, "hgt_gelu: X must be contiguous bf16 [rows, d]");
  check_rows(Y, torch::kBFloat16, d, "hgt_gelu: Y must be contiguous bf16 [rows, d]");
  check_counters(counters, n_hops, "hgt_gelu: counters must be int32 [> n_hops] on the device");
  int64_t cap = std::min<int64_t>(X.size(0), Y.size(0));
  if (has(dY)) {
    check_rows(*dY, torch::kBFloat16, d, "hgt_gelu: dY must be contiguous bf16 [rows, d]");
    cap = std::min<int64_t>(cap, dY->size(0));
  }
  launch_hgt_gelu(X.data_ptr(), Y.data_ptr(), counters.data_ptr<int32_t>(), n_hops, cap, d,
                  opt_ptr(dY), cur_stream());
  check_cuda_err("hgt_gelu");
}

static void hgt_gate(const Tensor& A, const Tensor& X, Tensor out, const Tensor& skip, const Tensor& counters,
                     int64_t n_hops, const c10::optional<Tensor>& dZ, const c10::optional<Tensor>& dX,
                     const c10::optional<Tensor>& skip_g) {
  c10::cuda::CUDAGuard guard(A.device());
  const int64_t d = A.size(1);
  TORCH_CHECK(d % 8 == 0, "hgt_gate: width must be a multiple of 8");
  check_rows(A, torch::kBFloat16, d, "hgt_gate: A must be contiguous bf16 [rows, d]");
  check_rows(X, torch::kBFloat16, d, "hgt_gate: X must be contiguous bf16 [rows, d]");
  check_rows(out, torch::kBFloat16, d, "hgt_gate: out must be contiguous bf16 [rows, d]");
  check_vec(skip, torch::kFloat32, 1, "hgt_gate: skip must be fp32 [1]");
  check_counters(counters, n_hops, "hgt_gate: counters must be int32 [> n_hops] on the device");
  HgtGateArgs a{};
  a.A = A.data_ptr(); a.X = X.data_ptr(); a.out = out.data_ptr(); a.skip = skip.data_ptr<float>();
  a.cum = counters.data_ptr<int32_t>(); a.n_hops = n_hops; a.d = d;
  int64_t cap = std::min<int64_t>(std::min<int64_t>(A.size(0), X.size(0)), out.size(0));
  if (has(dZ)) {
    TORCH_CHECK(on_dev(*dZ) && dZ->is_contiguous() && dZ->dim() == 2 && dZ->size(1) == d &&
                (dZ->scalar_type() == torch::kFloat32 || dZ->scalar_type() == torch::kBFloat16),
                "hgt_gate: dZ must be contiguous fp32 or bf16 [rows, d]");
    cap = std::min<int64_t>(cap, dZ->size(0));
    if (dZ->scalar_type() == torch::kFloat32) a.dZ32 = dZ->data_ptr<float>(); else a.dZ16 = dZ->data_ptr();
    if (has(dX)) {
      check_rows(*dX, torch::kFloat32, d, "hgt_gate: dX must be contiguous fp32 [rows, d]");
      cap = std::min<int64_t>(cap, dX->size(0));
      a.dX = dX->data_ptr<float>();
    }
    if (has(skip_g)) {
      check_vec(*skip_g, torch::kFloat32, 1, "hgt_gate: skip_g must be fp32 [1]");
      a.skip_g = skip_g->data_ptr<float>();
    }
  }
  a.cap = cap;
  launch_hgt_gate(a, cur_stream());
  check_cuda_err("hgt_gate");
}

// Block-diagonal images of a (layer, type)'s relation transforms (att, msg bf16 [n_rel, heads, D, D]); with the
// gradient arguments, the inverse map of the dense fp32 GEMM weight gradients into att_g / msg_g instead.
static void hgt_blocks(const Tensor& att, const Tensor& msg, Tensor att_img, Tensor msg_img,
                       const c10::optional<Tensor>& att_dense, const c10::optional<Tensor>& msg_dense,
                       const c10::optional<Tensor>& att_g, const c10::optional<Tensor>& msg_g) {
  c10::cuda::CUDAGuard guard(att.device());
  TORCH_CHECK(on_dev(att) && on_dev(msg) && att.dim() == 4 && att.size(2) == att.size(3) && msg.sizes() == att.sizes() && att.is_contiguous() &&
              msg.is_contiguous() && att.scalar_type() == torch::kBFloat16 && msg.scalar_type() == torch::kBFloat16,
              "hgt_blocks: att and msg must be contiguous bf16 [n_rel, heads, D, D]");
  const int64_t R = att.size(0), heads = att.size(1), D = att.size(2), H = heads * D;
  TORCH_CHECK(R >= 1 && R <= kHgtMaxRel, "hgt: a destination type takes 1 to 8 relations");
  check_hgt_width(H, heads);
  check_rows(att_img, torch::kBFloat16, H, "hgt_blocks: att_img must be contiguous bf16 [n_rel * H, H]");
  check_rows(msg_img, torch::kBFloat16, R * H, "hgt_blocks: msg_img must be contiguous bf16 [H, n_rel * H]");
  TORCH_CHECK(att_img.size(0) == R * H && msg_img.size(0) == H, "hgt_blocks: image shapes");
  HgtBlockArgs a{};
  a.att = att.data_ptr(); a.msg = msg.data_ptr(); a.att_img = att_img.data_ptr(); a.msg_img = msg_img.data_ptr();
  a.n_rel = R; a.heads = heads; a.D = D;
  if (has(att_g)) {
    TORCH_CHECK(has(msg_g) && has(att_dense) && has(msg_dense), "hgt_blocks: the gradient map needs all four buffers");
    for (const Tensor* t : {&*att_g, &*msg_g})
      TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && t->numel() == R * H * D,
                  "hgt_blocks: att_g / msg_g must be fp32 [n_rel, heads, D, D]");
    for (const Tensor* t : {&*att_dense, &*msg_dense})
      TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && t->numel() == R * H * H,
                  "hgt_blocks: the dense gradients must be fp32 [n_rel * H, H] / [H, n_rel * H]");
    a.att_dense = att_dense->data_ptr<float>(); a.msg_dense = msg_dense->data_ptr<float>();
    a.att_g = att_g->data_ptr<float>(); a.msg_g = msg_g->data_ptr<float>();
  }
  launch_hgt_blocks(a, cur_stream());
  check_cuda_err("hgt_blocks");
}

static void hgt_kqv_cast(Tensor dkv, const c10::optional<Tensor>& dq, Tensor out, const c10::optional<Tensor>& bias_g,
                         const Tensor& counters, int64_t idx, int64_t idx_q) {
  c10::cuda::CUDAGuard guard(dkv.device());
  TORCH_CHECK(out.dim() == 2 && out.size(1) % 3 == 0, "hgt_kqv_cast: out must be [rows, 3H]");
  const int64_t H = out.size(1) / 3;
  TORCH_CHECK(H % 64 == 0 && H >= 64 && H <= 1024, "hgt_kqv_cast: H must be a multiple of 64 in [64, 1024]");
  check_rows(out, torch::kBFloat16, 3 * H, "hgt_kqv_cast: out must be contiguous bf16 [rows, 3H]");
  check_rows(dkv, torch::kFloat32, 2 * H, "hgt_kqv_cast: dkv must be contiguous fp32 [rows, 2H]");
  check_counters(counters, idx, "hgt_kqv_cast: counters must be int32 [> idx] on the device");
  HgtKqvCastArgs a{};
  a.dkv = dkv.data_ptr<float>(); a.out = out.data_ptr(); a.cum = counters.data_ptr<int32_t>();
  a.idx = idx; a.idx_q = idx_q; a.H = H;
  a.cap = std::min<int64_t>(out.size(0), dkv.size(0));
  if (has(dq)) {
    check_rows(*dq, torch::kBFloat16, H, "hgt_kqv_cast: dq must be contiguous bf16 [rows, H]");
    check_counters(counters, idx_q, "hgt_kqv_cast: counters must be int32 [> idx_q] on the device");
    a.dq = dq->data_ptr();
    a.cap_q = dq->size(0);
  }
  if (has(bias_g)) {
    check_vec(*bias_g, torch::kFloat32, 3 * H, "hgt_kqv_cast: bias_g must be fp32 [3H]");
    a.bias_g = bias_g->data_ptr<float>();
  }
  launch_hgt_kqv_cast(a, cur_stream());
  check_cuda_err("hgt_kqv_cast");
}

// Link-prediction seeds of one batch (cuda/link.cu): pos int64 [2, B] -> seeds int64 [2 (1 + k) B], n_pairs int32.
// `step` is the arena's device step, read before the arena's sample() advances it.
static void link_seeds(GraphHandle* graph, const Tensor& pos, int64_t num_nodes, int64_t neg_ratio, int64_t seed,
                       const Tensor& step, Tensor seeds, Tensor n_pairs) {
  c10::cuda::CUDAGuard guard(seeds.device());
  TORCH_CHECK(graph != nullptr && graph->tbl.num_parts > 0, "link_seeds: graph has no shards");
  TORCH_CHECK(on_dev(pos) && pos.scalar_type() == torch::kInt64 && pos.is_contiguous() && pos.dim() == 2 &&
              pos.size(0) == 2, "link_seeds: pos must be a contiguous int64 [2, B] CUDA tensor");
  TORCH_CHECK(neg_ratio >= 1, "link_seeds: neg_ratio must be >= 1");
  TORCH_CHECK(num_nodes >= 1 && num_nodes <= graph->num_rows && num_nodes < (1LL << 32),
              "link_seeds: num_nodes must be in [1, graph rows] and < 2^32");
  const int64_t B = pos.size(1), P = (1 + neg_ratio) * B;
  TORCH_CHECK(P < (1LL << 30), "link_seeds: batch too large");
  check_ids(seeds, "link_seeds: seeds must be a contiguous int64 [2 (1 + k) B] CUDA tensor");
  TORCH_CHECK(seeds.numel() == 2 * P, "link_seeds: seeds must be a contiguous int64 [2 (1 + k) B] CUDA tensor");
  check_counters(step, 0, "link_seeds: int32 step");
  check_counters(n_pairs, 0, "link_seeds: int32 n_pairs");
  launch_link_seeds(graph->tbl, pos.data_ptr<int64_t>(), static_cast<int>(B), static_cast<int>(neg_ratio), num_nodes,
                    static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), seeds.data_ptr<int64_t>(),
                    n_pairs.data_ptr<int32_t>(), cur_stream());
  check_cuda_err("link_seeds");
}

// Fused edge loss of a link batch (cuda/link.cu) over the embeddings Z (bf16 [rows, ld], first C columns real).
static void link_bce(const Tensor& Z, int64_t C, const Tensor& seed_local, int64_t P, int64_t B, const Tensor& n_pairs,
                     Tensor loss, const c10::optional<Tensor>& correct, const c10::optional<Tensor>& dZ) {
  c10::cuda::CUDAGuard guard(Z.device());
  TORCH_CHECK(Z.scalar_type() == torch::kBFloat16 && Z.is_contiguous() && Z.dim() == 2,
              "link_bce: Z must be a contiguous bf16 [rows, ld] CUDA tensor");
  TORCH_CHECK(C % 8 == 0 && C >= 8 && C <= 512 && C <= Z.size(1) && Z.size(1) % 8 == 0,
              "link_bce: C must be a multiple of 8 in [8, 512] and <= Z's width");
  TORCH_CHECK(0 <= B && B <= P && on_dev(seed_local) && seed_local.scalar_type() == torch::kInt32 &&
              seed_local.is_contiguous() && seed_local.numel() >= 2 * P, "link_bce: seed_local must be int32 [>= 2P]");
  check_counters(n_pairs, 0, "link_bce: n_pairs must be int32 [>= 1] on the device");
  TORCH_CHECK(on_dev(loss) && loss.scalar_type() == torch::kFloat32 && loss.numel() >= 1,
              "link_bce: loss must be fp32 [>= 1] on the device");
  if (has(correct)) check_counters(*correct, 0, "link_bce: correct must be int32 [>= 1] on the device");
  if (has(dZ))
    TORCH_CHECK(on_dev(*dZ) && dZ->scalar_type() == torch::kFloat32 && dZ->is_contiguous() && dZ->sizes() == Z.sizes(),
                "link_bce: dZ must be a contiguous fp32 tensor of Z's shape");
  launch_link_bce(Z.data_ptr(), static_cast<int>(Z.size(1)), static_cast<int>(C), seed_local.data_ptr<int32_t>(),
                  static_cast<int>(P), static_cast<int>(B), n_pairs.data_ptr<int32_t>(), loss.data_ptr<float>(),
                  opt_ptr<int32_t>(correct), opt_ptr<float>(dZ), cur_stream());
  check_cuda_err("link_bce");
}

// ---------------------------------------------------------------------------
// MetaPath: device view of a metapath for the skip-gram kernels (cuda/skipgram.cu): the R relation graphs (CSR rows =
// source ids) as a device array of GraphTables, and the node type of every walk position slot as (first row in the
// concatenated embedding table, node count).  Slot 0 is the source type of relation 0, slot r + 1 the destination
// type of relation r.
// ---------------------------------------------------------------------------
struct MetaPath {
  int device, R;
  std::vector<GraphHandle*> graphs;
  MetaPathTypes types{};
  int64_t rows = 0;       // rows the embedding tables must have: max over slots of off + n
  Tensor tables;          // uint8 [R * sizeof(GraphTable)]

  MetaPath(int dev, std::vector<GraphHandle*> graphs_, std::vector<int64_t> slot_off, std::vector<int64_t> slot_n)
      : device(dev), R(static_cast<int>(graphs_.size())), graphs(std::move(graphs_)) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(R >= 1 && R <= kMaxMetaPath, fmt("MetaPath: 1 to %d relations", kMaxMetaPath));
    TORCH_CHECK(static_cast<int>(slot_off.size()) == R + 1 && static_cast<int>(slot_n.size()) == R + 1,
                "MetaPath: slot_off and slot_n need R + 1 entries");
    std::vector<GraphTable> t(R);
    for (int r = 0; r < R; ++r) {
      TORCH_CHECK(graphs[r] != nullptr && graphs[r]->tbl.num_parts > 0, "MetaPath: every relation needs a device graph");
      TORCH_CHECK(graphs[r]->device == device, "MetaPath: the relation graphs must live on the metapath's device");
      t[r] = graphs[r]->tbl;
    }
    for (int s = 0; s <= R; ++s) {
      TORCH_CHECK(slot_n[s] >= 1 && slot_n[s] < (1LL << 32) && slot_off[s] >= 0 && slot_off[s] + slot_n[s] < (1LL << 40),
                  "MetaPath: every slot needs 1 <= n < 2^32 nodes at a non-negative row offset");
      types.off[s] = slot_off[s];
      types.n[s] = slot_n[s];
      rows = std::max(rows, slot_off[s] + slot_n[s]);
    }
    tables = torch::empty({static_cast<int64_t>(R * sizeof(GraphTable))},
                          torch::TensorOptions().dtype(torch::kUInt8).device(torch::kCUDA, device));
    cudaMemcpy(tables.data_ptr(), t.data(), R * sizeof(GraphTable), cudaMemcpyHostToDevice);
    check_cuda_err("MetaPath setup");
  }
  const GraphTable* dev_tables() const { return reinterpret_cast<const GraphTable*>(tables.data_ptr()); }
};

// walks int64 [n_walks, L + 1] with L >= 1 and 2 <= C <= L + 1; returns (n_walks, L)
static std::pair<int64_t, int64_t> check_walks(const Tensor& walks, int64_t C, const char* msg) {
  TORCH_CHECK(on_dev(walks) && walks.scalar_type() == torch::kInt64 && walks.dim() == 2 && walks.is_contiguous() &&
              walks.size(1) >= 2 && walks.size(0) < (1LL << 31), msg);
  const int64_t L = walks.size(1) - 1;
  TORCH_CHECK(C >= 2 && C <= L + 1, fmt("context_size must be in [2, walk_length + 1 = %lld]", (long long)(L + 1)));
  return {walks.size(0), L};
}

// negatives int64 [n_walks (L + 2 - C) K, C]
static void check_negatives(const Tensor& neg, int64_t n_walks, int64_t L, int64_t C, int64_t K, const char* msg) {
  TORCH_CHECK(K >= 1, "num_negative_samples must be >= 1");
  const int64_t n = n_walks * (L + 2 - C) * K;
  TORCH_CHECK(n < (1LL << 31), "too many negative windows (>= 2^31)");
  TORCH_CHECK(on_dev(neg) && neg.scalar_type() == torch::kInt64 && neg.dim() == 2 && neg.is_contiguous() &&
              neg.size(0) == n && neg.size(1) == C, msg);
}

// Walks of one step: walk i starts at starts[i / walks_per_node]; n_valid = #windows of C valid entries.
static void metapath_walk(const MetaPath& mp, const Tensor& starts, int64_t walks_per_node, int64_t context_size,
                          int64_t seed, const Tensor& step, Tensor walks, Tensor n_valid) {
  c10::cuda::CUDAGuard guard(mp.device);
  check_ids(starts, "metapath_walk: starts must be contiguous int64 on the metapath's device");
  TORCH_CHECK(walks_per_node >= 1, "metapath_walk: walks_per_node must be >= 1");
  const auto [n_walks, L] = check_walks(walks, context_size,
                                        "metapath_walk: walks must be a contiguous int64 [n_walks, walk_length + 1] "
                                        "tensor on the metapath's device");
  TORCH_CHECK(n_walks == starts.numel() * walks_per_node, "metapath_walk: walks needs starts * walks_per_node rows");
  check_counters(step, 0, "metapath_walk: step must be int32 [>= 1] on the device");
  check_counters(n_valid, 0, "metapath_walk: n_valid must be int32 [>= 1] on the device");
  if (n_walks == 0) return;
  launch_metapath_walk(mp.dev_tables(), mp.R, mp.types, starts.data_ptr<int64_t>(), static_cast<int>(n_walks),
                       static_cast<int>(walks_per_node), static_cast<int>(L), static_cast<int>(context_size),
                       static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), walks.data_ptr<int64_t>(),
                       n_valid.data_ptr<int32_t>(), cur_stream());
  check_cuda_err("metapath_walk");
}

// node2vec's p / q walks of one step over a metapath of one relation from a type to itself; the same contract as
// metapath_walk.  p and q pass node2vec_weights (philox.h): r <= 64 bounds the rejection sampler's proposals.
static void node2vec_walk(const MetaPath& mp, const Tensor& starts, int64_t walks_per_node, int64_t context_size,
                          int64_t seed, const Tensor& step, Tensor walks, Tensor n_valid, double p, double q) {
  c10::cuda::CUDAGuard guard(mp.device);
  Node2VecWeights w;
  const char* bad = node2vec_weights(p, q, &w);
  TORCH_CHECK(bad == nullptr, fmt("node2vec_walk: %s", bad));
  TORCH_CHECK(mp.R == 1 && mp.types.off[0] == mp.types.off[1] && mp.types.n[0] == mp.types.n[1],
              "node2vec_walk: the metapath must be one relation from a node type to itself");
  check_ids(starts, "node2vec_walk: starts must be contiguous int64 on the metapath's device");
  TORCH_CHECK(walks_per_node >= 1, "node2vec_walk: walks_per_node must be >= 1");
  const auto [n_walks, L] = check_walks(walks, context_size,
                                        "node2vec_walk: walks must be a contiguous int64 [n_walks, walk_length + 1] "
                                        "tensor on the metapath's device");
  TORCH_CHECK(L <= kNode2VecMaxWalk, fmt("node2vec_walk: walk_length must be <= %d", kNode2VecMaxWalk));
  TORCH_CHECK(n_walks == starts.numel() * walks_per_node, "node2vec_walk: walks needs starts * walks_per_node rows");
  check_counters(step, 0, "node2vec_walk: step must be int32 [>= 1] on the device");
  check_counters(n_valid, 0, "node2vec_walk: n_valid must be int32 [>= 1] on the device");
  if (n_walks == 0) return;
  launch_node2vec_walk(mp.dev_tables(), mp.types, starts.data_ptr<int64_t>(), static_cast<int>(n_walks),
                       static_cast<int>(walks_per_node), static_cast<int>(L), static_cast<int>(context_size),
                       w.ret, w.in, w.out,
                       static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), walks.data_ptr<int64_t>(),
                       n_valid.data_ptr<int32_t>(), cur_stream());
  check_cuda_err("node2vec_walk");
}

static void sgns_negatives(const MetaPath& mp, const Tensor& walks, int64_t context_size, int64_t num_neg, int64_t seed,
                           const Tensor& step, Tensor neg) {
  c10::cuda::CUDAGuard guard(mp.device);
  const auto [n_walks, L] = check_walks(walks, context_size,
                                        "sgns_negatives: walks must be a contiguous int64 [n_walks, walk_length + 1] "
                                        "tensor on the metapath's device");
  check_negatives(neg, n_walks, L, context_size, num_neg,
                  "sgns_negatives: neg must be a contiguous int64 [n_walks * windows * K, C] tensor on the device");
  check_counters(step, 0, "sgns_negatives: step must be int32 [>= 1] on the device");
  if (neg.numel() == 0) return;
  launch_sgns_negatives(walks.data_ptr<int64_t>(), static_cast<int>(n_walks), static_cast<int>(L),
                        static_cast<int>(context_size), static_cast<int>(num_neg), mp.R, mp.types,
                        static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), neg.data_ptr<int64_t>(), cur_stream());
  check_cuda_err("sgns_negatives");
}

// emb / grad fp32 [rows >= mp.rows, D], D a multiple of 8 in [8, 512]; touched uint8 [rows]
static void check_sgns_tables(const MetaPath& mp, const Tensor& emb, const Tensor& grad, const Tensor& touched,
                              const char* who) {
  const int64_t D = emb.dim() == 2 ? emb.size(1) : 0;
  TORCH_CHECK(D % 8 == 0 && D >= 8 && D <= 512,
              fmt("%s: emb must be fp32 [rows, D] with D a multiple of 8 in [8, 512]", who));
  check_rows(emb, torch::kFloat32, D, fmt("%s: emb must be a contiguous fp32 [rows, D] tensor on the device", who).c_str());
  TORCH_CHECK(emb.size(0) >= mp.rows, fmt("%s: emb has fewer rows than the metapath's node types", who));
  check_rows(grad, torch::kFloat32, D, fmt("%s: grad must be a contiguous fp32 tensor of emb's shape", who).c_str());
  TORCH_CHECK(grad.size(0) == emb.size(0), fmt("%s: grad must be a contiguous fp32 tensor of emb's shape", who));
  TORCH_CHECK(on_dev(touched) && touched.scalar_type() == torch::kUInt8 && touched.is_contiguous() &&
              touched.numel() == emb.size(0), fmt("%s: touched must be contiguous uint8 [rows] on the device", who));
}

// SGNS loss of the walks' valid windows and their negatives (written to loss[0]); gradient red.added into grad and
// touched[row] = 1 for every row looked up.
static void sgns_loss_grad(const MetaPath& mp, const Tensor& walks, const Tensor& neg, int64_t context_size,
                           int64_t num_neg, const Tensor& emb, const Tensor& n_valid, Tensor grad, Tensor touched,
                           Tensor loss) {
  c10::cuda::CUDAGuard guard(mp.device);
  const auto [n_walks, L] = check_walks(walks, context_size,
                                        "sgns_loss_grad: walks must be a contiguous int64 [n_walks, walk_length + 1] "
                                        "tensor on the metapath's device");
  check_negatives(neg, n_walks, L, context_size, num_neg,
                  "sgns_loss_grad: neg must be a contiguous int64 [n_walks * windows * K, C] tensor on the device");
  check_sgns_tables(mp, emb, grad, touched, "sgns_loss_grad");
  check_counters(n_valid, 0, "sgns_loss_grad: n_valid must be int32 [>= 1] on the device");
  TORCH_CHECK(on_dev(loss) && loss.scalar_type() == torch::kFloat32 && loss.numel() >= 1,
              "sgns_loss_grad: loss must be fp32 [>= 1] on the device");
  launch_sgns_loss_grad(walks.data_ptr<int64_t>(), neg.data_ptr<int64_t>(), static_cast<int>(n_walks),
                        static_cast<int>(L), static_cast<int>(context_size), static_cast<int>(num_neg), mp.R, mp.types,
                        emb.data_ptr<float>(), static_cast<int>(emb.size(1)), n_valid.data_ptr<int32_t>(),
                        grad.data_ptr<float>(), touched.data_ptr<uint8_t>(), loss.data_ptr<float>(), cur_stream());
  check_cuda_err("sgns_loss_grad");
}

// torch.optim.SparseAdam step t = step[0] on the touched rows of emb / m / v; clears their grad rows and flags.
static void sparse_adam(const MetaPath& mp, Tensor emb, Tensor grad, Tensor m, Tensor v, Tensor touched,
                        const Tensor& step, double lr, double b1, double b2, double eps) {
  c10::cuda::CUDAGuard guard(mp.device);
  check_sgns_tables(mp, emb, grad, touched, "sparse_adam");
  for (const Tensor* t : {&m, &v})
    TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && aligned16(*t) &&
                t->sizes() == emb.sizes(), "sparse_adam: m and v must be contiguous fp32 tensors of emb's shape");
  check_counters(step, 0, "sparse_adam: step must be int32 [>= 1] on the device");
  TORCH_CHECK(lr > 0 && b1 >= 0 && b1 < 1 && b2 >= 0 && b2 < 1 && eps > 0,
              "sparse_adam: need lr > 0, 0 <= betas < 1 and eps > 0");
  launch_sparse_adam(emb.data_ptr<float>(), grad.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                     touched.data_ptr<uint8_t>(), emb.size(0), static_cast<int>(emb.size(1)), step.data_ptr<int32_t>(),
                     static_cast<float>(lr), static_cast<float>(b1), static_cast<float>(b2), static_cast<float>(eps),
                     cur_stream());
  check_cuda_err("sparse_adam");
}

// state int32 [3] = [next walk step, Adam step, walk step of the current step]
static void m2v_begin(Tensor state) {
  c10::cuda::CUDAGuard guard(state.device());
  check_counters(state, 2, "m2v_begin: state must be int32 [>= 3] on the device");
  launch_m2v_begin(state.data_ptr<int32_t>(), cur_stream());
  check_cuda_err("m2v_begin");
}

// ---------------------------------------------------------------------------
// Knowledge-graph embeddings (cuda/kge.cu, models/kge.py).  model: 0 TransE, 1 DistMult, 2 ComplEx, 3 RotatE.
// ---------------------------------------------------------------------------
// ent fp32 [N, D * entity parts], rel fp32 [R, D * relation parts], D a multiple of 8 in [8, 512]; returns D.
static int64_t check_kge_tables(int64_t model, const Tensor& ent, const Tensor& rel, const char* who) {
  TORCH_CHECK(model >= 0 && model <= 3, fmt("%s: model must be 0 (TransE), 1 (DistMult), 2 (ComplEx) or 3 (RotatE)", who));
  const int pe = kge_entity_parts(static_cast<int>(model)), pr = kge_relation_parts(static_cast<int>(model));
  TORCH_CHECK(ent.dim() == 2 && ent.size(1) % pe == 0, fmt("%s: ent must be fp32 [N, %d D]", who, pe));
  const int64_t D = ent.size(1) / pe;
  TORCH_CHECK(D % 8 == 0 && D >= 8 && D <= 512, fmt("%s: D must be a multiple of 8 in [8, 512]", who));
  check_rows(ent, torch::kFloat32, pe * D, fmt("%s: ent must be a contiguous fp32 [N, %d D] tensor on the device", who, pe).c_str());
  check_rows(rel, torch::kFloat32, pr * D, fmt("%s: rel must be a contiguous fp32 [R, %d D] tensor on the device", who, pr).c_str());
  TORCH_CHECK(ent.size(0) >= 1 && ent.size(0) < (int64_t(1) << 31) && rel.size(0) >= 1 &&
              rel.size(0) < (int64_t(1) << 31), fmt("%s: need 1 <= N, R < 2^31", who));
  return D;
}

// grad: a contiguous fp32 tensor of t's shape; touched: contiguous uint8 [rows of t]
static void check_kge_grad(const Tensor& t, const Tensor& grad, const Tensor& touched, const char* who) {
  check_rows(grad, torch::kFloat32, t.size(1), fmt("%s: gradients must be contiguous fp32 tensors of the tables' shapes", who).c_str());
  TORCH_CHECK(grad.size(0) == t.size(0), fmt("%s: gradients must be contiguous fp32 tensors of the tables' shapes", who));
  TORCH_CHECK(on_dev(touched) && touched.scalar_type() == torch::kUInt8 && touched.is_contiguous() &&
              touched.numel() == t.size(0), fmt("%s: touched flags must be contiguous uint8, one per table row", who));
}

// neg[i * K + j] of the first min(count[0], B) positives of a batch of B: uniform in [0, N).
static void kge_negatives(const Tensor& count, int64_t batch_size, int64_t num_neg, int64_t N, int64_t seed,
                          const Tensor& step, Tensor neg) {
  c10::cuda::CUDAGuard guard(neg.device());
  TORCH_CHECK(batch_size >= 1 && num_neg >= 1 && batch_size * num_neg < (int64_t(1) << 31),
              "kge_negatives: need batch_size, num_neg >= 1 and batch_size * num_neg < 2^31");
  TORCH_CHECK(N >= 1 && N < (int64_t(1) << 31), "kge_negatives: need 1 <= N < 2^31");
  check_counters(count, 0, "kge_negatives: count must be int32 [>= 1] on the device");
  check_counters(step, 0, "kge_negatives: step must be int32 [>= 1] on the device");
  TORCH_CHECK(neg.dim() == 2 && neg.size(0) == batch_size && neg.size(1) == num_neg,
              "kge_negatives: neg must be int64 [batch_size, num_neg]");
  check_ids(neg, "kge_negatives: neg must be contiguous int64 on the device");
  launch_kge_negatives(count.data_ptr<int32_t>(), static_cast<int>(batch_size), static_cast<int>(num_neg), N,
                       static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), neg.data_ptr<int64_t>(), cur_stream());
  check_cuda_err("kge_negatives");
}

// Loss of the first min(count[0], B) triples of trip (int64 [3, B]) and their negatives (written to loss[0]);
// gradients red.added into grad_ent / grad_rel, touched flags set for every row looked up.
static void kge_loss_grad(int64_t model, const Tensor& trip, const Tensor& count, const Tensor& neg, const Tensor& ent,
                          const Tensor& rel, double margin, int64_t p, Tensor grad_ent, Tensor grad_rel,
                          Tensor touched_ent, Tensor touched_rel, Tensor loss) {
  c10::cuda::CUDAGuard guard(ent.device());
  const int64_t D = check_kge_tables(model, ent, rel, "kge_loss_grad");
  TORCH_CHECK(trip.dim() == 2 && trip.size(0) == 3 && trip.size(1) >= 1, "kge_loss_grad: trip must be int64 [3, B]");
  check_ids(trip, "kge_loss_grad: trip must be contiguous int64 on the tables' device");
  const int64_t B = trip.size(1);
  TORCH_CHECK(neg.dim() == 2 && neg.size(0) == B && neg.size(1) >= 1 && B * neg.size(1) < (int64_t(1) << 31),
              "kge_loss_grad: neg must be int64 [B, K]");
  check_ids(neg, "kge_loss_grad: neg must be contiguous int64 on the tables' device");
  check_counters(count, 0, "kge_loss_grad: count must be int32 [>= 1] on the device");
  TORCH_CHECK(p == 1 || p == 2, "kge_loss_grad: p must be 1 or 2");
  check_kge_grad(ent, grad_ent, touched_ent, "kge_loss_grad");
  check_kge_grad(rel, grad_rel, touched_rel, "kge_loss_grad");
  TORCH_CHECK(on_dev(loss) && loss.scalar_type() == torch::kFloat32 && loss.numel() >= 1,
              "kge_loss_grad: loss must be fp32 [>= 1] on the device");
  launch_kge_loss_grad(static_cast<int>(model), trip.data_ptr<int64_t>(), static_cast<int>(B),
                       count.data_ptr<int32_t>(), neg.data_ptr<int64_t>(), static_cast<int>(neg.size(1)),
                       ent.data_ptr<float>(), rel.data_ptr<float>(), ent.size(0), rel.size(0), static_cast<int>(D),
                       static_cast<float>(margin), static_cast<int>(p), grad_ent.data_ptr<float>(),
                       grad_rel.data_ptr<float>(), touched_ent.data_ptr<uint8_t>(), touched_rel.data_ptr<uint8_t>(),
                       loss.data_ptr<float>(), cur_stream());
  check_cuda_err("kge_loss_grad");
}

// h, r, t: int64 [n] on the tables' device, every id in range (checked here, with one host sync)
static void check_kge_triples(const Tensor& h, const Tensor& r, const Tensor& t, int64_t N, int64_t R, const char* who) {
  for (const Tensor* x : {&h, &r, &t}) {
    TORCH_CHECK(x->dim() == 1 && x->numel() == h.numel(), fmt("%s: h, r and t must be 1-D of one length", who));
    check_ids(*x, fmt("%s: h, r and t must be contiguous int64 on the tables' device", who).c_str());
  }
  if (h.numel() == 0) return;
  const Tensor lo = torch::stack({h.min(), r.min(), t.min()}).cpu(), hi = torch::stack({h.max(), r.max(), t.max()}).cpu();
  const int64_t* l = lo.data_ptr<int64_t>();
  const int64_t* u = hi.data_ptr<int64_t>();
  TORCH_CHECK(l[0] >= 0 && u[0] < N && l[2] >= 0 && u[2] < N, fmt("%s: entity ids must lie in [0, %lld)", who, static_cast<long long>(N)));
  TORCH_CHECK(l[1] >= 0 && u[1] < R, fmt("%s: relation ids must lie in [0, %lld)", who, static_cast<long long>(R)));
}

// fp32 [n] scores of the triples (h[i], r[i], t[i]).
static Tensor kge_score(int64_t model, const Tensor& ent, const Tensor& rel, const Tensor& h, const Tensor& r,
                        const Tensor& t, double margin, int64_t p) {
  TORCH_CHECK(ent.is_cuda(), "kge_score: ent must be a CUDA tensor");
  c10::cuda::CUDAGuard guard(ent.device());
  const int64_t D = check_kge_tables(model, ent, rel, "kge_score");
  TORCH_CHECK(p == 1 || p == 2, "kge_score: p must be 1 or 2");
  check_kge_triples(h, r, t, ent.size(0), rel.size(0), "kge_score");
  Tensor out = torch::empty({h.numel()}, ent.options());
  if (h.numel() == 0) return out;
  launch_kge_score(static_cast<int>(model), h.data_ptr<int64_t>(), r.data_ptr<int64_t>(), t.data_ptr<int64_t>(),
                   h.numel(), ent.data_ptr<float>(), rel.data_ptr<float>(), static_cast<int>(D),
                   static_cast<float>(margin), static_cast<int>(p), out.data_ptr<float>(), cur_stream());
  check_cuda_err("kge_score");
  return out;
}

// float64 [n] ranks of the true tail (tail = true) or head among all N entities: 1 + #better + #tied / 2, with the
// true entity and the ids of the query's range of `keys` (sorted int64 (f R + r) N + c, f the fixed entity) left out.
// splits = 0 picks the candidate split count from n and the SM count; every count gives the same ranks.
static Tensor kge_rank(int64_t model, const Tensor& ent, const Tensor& rel, const Tensor& h, const Tensor& r,
                       const Tensor& t, bool tail, const c10::optional<Tensor>& keys, double margin, int64_t p,
                       int64_t splits) {
  TORCH_CHECK(ent.is_cuda(), "kge_rank: ent must be a CUDA tensor");
  c10::cuda::CUDAGuard guard(ent.device());
  const int64_t D = check_kge_tables(model, ent, rel, "kge_rank");
  TORCH_CHECK(p == 1 || p == 2, "kge_rank: p must be 1 or 2");
  TORCH_CHECK(splits >= 0, "kge_rank: splits must be >= 0 (0: chosen from n)");
  const int64_t N = ent.size(0), R = rel.size(0), n = h.numel();
  check_kge_triples(h, r, t, N, R, "kge_rank");
  if (has(keys)) {
    TORCH_CHECK(keys->dim() == 1, "kge_rank: keys must be 1-D");
    check_ids(*keys, "kge_rank: keys must be contiguous int64 on the tables' device");
  }
  if (n == 0) return torch::empty({0}, ent.options().dtype(torch::kFloat64));
  const int64_t q_tiles = (n + 63) / 64, c_tiles = (N + 63) / 64;
  TORCH_CHECK(q_tiles < (int64_t(1) << 31), "kge_rank: too many queries");
  if (splits == 0) {   // about two CTAs per SM, as few splits as that takes
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ent.get_device());
    splits = std::max<int64_t>(1, (2 * static_cast<int64_t>(sms) + q_tiles - 1) / q_tiles);
  }
  splits = std::min(splits, c_tiles);
  const int64_t per = (c_tiles + splits - 1) / splits;
  splits = (c_tiles + per - 1) / per;   // no empty split
  TORCH_CHECK(splits <= 65535, "kge_rank: at most 65535 splits");
  Tensor q = torch::empty({n, ent.size(1)}, ent.options());
  Tensor den = torch::empty({model == kKgeTransE ? N : 1}, ent.options());
  Tensor counts = torch::empty({n}, h.options());
  KgeRankArgs a{};
  a.model = static_cast<int>(model);
  a.D = static_cast<int>(D);
  a.p = static_cast<int>(p);
  a.margin = static_cast<float>(margin);
  a.tail = tail;
  a.h = h.data_ptr<int64_t>();
  a.r = r.data_ptr<int64_t>();
  a.t = t.data_ptr<int64_t>();
  a.n = n;
  a.N = N;
  a.R = R;
  a.ent = ent.data_ptr<float>();
  a.rel = rel.data_ptr<float>();
  a.keys = has(keys) && keys->numel() > 0 ? keys->data_ptr<int64_t>() : nullptr;
  a.n_keys = has(keys) ? keys->numel() : 0;
  a.den = den.data_ptr<float>();
  a.q = q.data_ptr<float>();
  a.counts = reinterpret_cast<unsigned long long*>(counts.data_ptr<int64_t>());
  a.splits = static_cast<int>(splits);
  a.tiles_per_split = static_cast<int>(per);
  launch_kge_rank(a, cur_stream());
  check_cuda_err("kge_rank");
  const Tensor better = counts.bitwise_right_shift(32), tied = counts.bitwise_and(0xFFFFFFFFLL);
  return better.to(torch::kFloat64) + 1.0 + tied.to(torch::kFloat64) * 0.5;
}

// torch.optim.SparseAdam step t = step[0] on the touched rows of one KGE table (entity or relation) and its moments;
// clears their gradient rows and flags.
static void kge_sparse_adam(Tensor w, Tensor grad, Tensor m, Tensor v, Tensor touched, const Tensor& step, double lr,
                            double b1, double b2, double eps) {
  c10::cuda::CUDAGuard guard(w.device());
  TORCH_CHECK(w.dim() == 2 && w.size(1) % 8 == 0 && w.size(1) >= 8 && w.size(1) <= 1024,
              "kge_sparse_adam: w must be fp32 [rows, W] with W a multiple of 8 in [8, 1024]");
  check_rows(w, torch::kFloat32, w.size(1), "kge_sparse_adam: w must be a contiguous fp32 [rows, W] tensor on the device");
  check_kge_grad(w, grad, touched, "kge_sparse_adam");
  for (const Tensor* t : {&m, &v})
    TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && aligned16(*t) &&
                t->sizes() == w.sizes(), "kge_sparse_adam: m and v must be contiguous fp32 tensors of w's shape");
  check_counters(step, 0, "kge_sparse_adam: step must be int32 [>= 1] on the device");
  TORCH_CHECK(lr > 0 && b1 >= 0 && b1 < 1 && b2 >= 0 && b2 < 1 && eps > 0,
              "kge_sparse_adam: need lr > 0, 0 <= betas < 1 and eps > 0");
  launch_sparse_adam(w.data_ptr<float>(), grad.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(),
                     touched.data_ptr<uint8_t>(), w.size(0), static_cast<int>(w.size(1)), step.data_ptr<int32_t>(),
                     static_cast<float>(lr), static_cast<float>(b1), static_cast<float>(b2), static_cast<float>(eps),
                     cur_stream());
  check_cuda_err("kge_sparse_adam");
}

// ---------------------------------------------------------------------------
// SealArena: the static per-link arena and parameter layout of SealEngine's step (cuda/seal.cu).
// ---------------------------------------------------------------------------
struct SealArena {
  int device;
  SealModel model{};
  SealArenaPtrs ptrs{};
  int cap_max;
  std::vector<std::tuple<std::string, int64_t, std::vector<int64_t>>> layout;
  Tensor nodes, z, meta, sptr, scol, dptr, dcol, X, XW, G, C1, flat, H1, mask, sel, logits, lossv, dlogit, samp, partials;

  SealArena(int dev, int64_t B, int64_t max_nodes, int64_t max_edges, int64_t hidden, int64_t num_layers, int64_t Z,
            int64_t k, int64_t cap_max_)
      : device(dev), cap_max(static_cast<int>(cap_max_)) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(B >= 1 && B <= (1 << 20), "SealArena: batch size must be in [1, 2^20]");
    TORCH_CHECK(max_nodes >= 2 && max_nodes <= kSealMaxNodes, fmt("SealArena: max_nodes must be in [2, %d]", kSealMaxNodes));
    TORCH_CHECK(max_edges >= 1 && max_edges <= (1 << 24), "SealArena: max_edges must be in [1, 2^24]");
    TORCH_CHECK(hidden >= 1 && hidden <= 256, "SealArena: hidden must be in [1, 256]");
    TORCH_CHECK(num_layers >= 1 && num_layers <= kSealMaxLayers, fmt("SealArena: num_layers must be in [1, %d]", kSealMaxLayers));
    TORCH_CHECK(Z >= 2 && Z <= (1 << 20), "SealArena: the label count max_z + 1 must be in [2, 2^20]");
    TORCH_CHECK(k >= 10 && k <= 2 * kSealMaxNodes, fmt("SealArena: sort-pool k must be in [10, %d]", 2 * kSealMaxNodes));
    TORCH_CHECK(cap_max_ >= 0 && cap_max_ <= max_nodes, "SealArena: neighbour caps must be in [0, max_nodes]");
    SealModel& m = model;
    m.H = static_cast<int>(hidden); m.L = static_cast<int>(num_layers); m.Z = static_cast<int>(Z);
    m.total = m.H * m.L + 1; m.k = static_cast<int>(k); m.dense = (m.k / 2 - 4) * 32;
    int64_t off = 0;
    auto add = [&](const std::string& name, std::vector<int64_t> shape) {
      int64_t n = 1;
      for (int64_t x : shape) n *= x;
      layout.emplace_back(name, off, shape);
      const int64_t at = off;
      off += n;
      return at;
    };
    for (int l = 0; l <= m.L; ++l) {
      const int64_t out = l < m.L ? m.H : 1, in = l == 0 ? m.Z : m.H;
      m.w[l] = add(fmt("convs.%d.lin.weight", l), {out, in});
      m.bias[l] = add(fmt("convs.%d.bias", l), {out});
    }
    m.c1w = add("conv1.weight", {16, 1, m.total});
    m.c1b = add("conv1.bias", {16});
    m.c2w = add("conv2.weight", {32, 16, 5});
    m.c2b = add("conv2.bias", {32});
    m.l1w = add("mlp.lins.0.weight", {128, m.dense});
    m.l1b = add("mlp.lins.0.bias", {128});
    m.l2w = add("mlp.lins.1.weight", {1, 128});
    m.l2b = add("mlp.lins.1.bias", {1});
    m.P = off;
    int optin = 0;
    cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
    const size_t need = std::max({seal_extract_smem(static_cast<int>(max_nodes)),
                                  seal_forward_smem(m, static_cast<int>(max_nodes)),
                                  seal_backward_smem(m, static_cast<int>(max_nodes))});
    TORCH_CHECK(need <= static_cast<size_t>(optin),
                fmt("SealArena: the per-link kernels need %zu bytes of shared memory (device limit %d); lower max_nodes, "
                    "hidden or k", need, optin));
    const auto f32 = torch::TensorOptions().dtype(torch::kFloat32).device(torch::kCUDA, device);
    const auto i32 = f32.dtype(torch::kInt32);
    nodes = torch::full({B, max_nodes}, -1, f32.dtype(torch::kInt64));
    z = torch::zeros({B, max_nodes}, i32);
    meta = torch::zeros({B, kSealMeta}, i32);
    sptr = torch::zeros({B, max_nodes + 1}, i32);
    dptr = torch::zeros({B, max_nodes + 1}, i32);
    scol = torch::zeros({B, max_edges}, f32.dtype(torch::kInt16));
    dcol = torch::zeros({B, max_edges}, f32.dtype(torch::kInt16));
    X = torch::zeros({B, max_nodes, m.total}, f32);
    XW = torch::zeros({B, max_nodes, m.H}, f32);
    G = torch::zeros({B, max_nodes, m.total}, f32);
    C1 = torch::zeros({B, 16, m.k}, f32);
    flat = torch::zeros({B, m.dense}, f32);
    H1 = torch::zeros({B, 128}, f32);
    mask = torch::zeros({B, 128}, f32);
    sel = torch::full({B, m.k}, -1, i32);
    logits = torch::zeros({B}, f32);
    lossv = torch::zeros({B}, f32);
    dlogit = torch::zeros({B}, f32);
    samp = torch::zeros({cap_max > 0 ? B * max_nodes * cap_max : 1}, i32);
    partials = torch::zeros({B, m.P}, f32);
    SealArenaPtrs& p = ptrs;
    p.B = static_cast<int>(B); p.max_nodes = static_cast<int>(max_nodes); p.max_edges = static_cast<int>(max_edges);
    p.nodes = nodes.data_ptr<int64_t>(); p.z = z.data_ptr<int32_t>(); p.meta = meta.data_ptr<int32_t>();
    p.sptr = sptr.data_ptr<int32_t>(); p.scol = scol.data_ptr<int16_t>();
    p.dptr = dptr.data_ptr<int32_t>(); p.dcol = dcol.data_ptr<int16_t>();
    p.X = X.data_ptr<float>(); p.XW = XW.data_ptr<float>(); p.G = G.data_ptr<float>(); p.C1 = C1.data_ptr<float>();
    p.flat = flat.data_ptr<float>(); p.H1 = H1.data_ptr<float>(); p.mask = mask.data_ptr<float>();
    p.sel = sel.data_ptr<int32_t>(); p.logits = logits.data_ptr<float>(); p.lossv = lossv.data_ptr<float>();
    p.dlogit = dlogit.data_ptr<float>();
    check_cuda_err("SealArena setup");
  }

  // links int64 [2, B] on the arena's device; caps: one entry per hop (<= 0: full rows), each <= cap_max.
  void extract(const GraphHandle& g, const Tensor& links, int64_t num_nodes, int64_t hops, std::vector<int64_t> caps,
               int64_t seed, const Tensor& step, int64_t max_z, Tensor truncated) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(g.tbl.num_parts > 0 && g.device == device, "SealArena.extract: graph must be a device graph on the arena's device");
    TORCH_CHECK(on_dev(links) && links.scalar_type() == torch::kInt64 && links.is_contiguous() && links.dim() == 2 &&
                links.size(0) == 2 && links.size(1) == ptrs.B,
                "SealArena.extract: links must be contiguous int64 [2, batch_size] on the arena's device");
    TORCH_CHECK(num_nodes >= 1, "SealArena.extract: num_nodes must be >= 1");
    TORCH_CHECK(hops >= 1 && hops <= kSealMaxHops, fmt("SealArena.extract: num_hops must be in [1, %d]", kSealMaxHops));
    TORCH_CHECK(static_cast<int64_t>(caps.size()) == hops, "SealArena.extract: caps needs one entry per hop");
    check_counters(step, 0, "SealArena.extract: step must be int32 [>= 1] on the device");
    check_counters(truncated, 0, "SealArena.extract: truncated must be int32 [>= 1] on the device");
    TORCH_CHECK(max_z < (1LL << 30), "SealArena.extract: max_z must be < 2^30");
    SealExtractArgs e{};
    e.g = g.tbl;
    e.links = links.data_ptr<int64_t>();
    e.num_nodes = num_nodes;
    e.hops = static_cast<int>(hops);
    e.cap_max = cap_max;
    for (int h = 0; h < hops; ++h) {
      TORCH_CHECK(caps[h] <= cap_max, "SealArena.extract: a neighbour cap exceeds the arena's cap_max");
      e.caps[h] = static_cast<int>(std::max<int64_t>(caps[h], 0));
    }
    e.seed = static_cast<uint64_t>(seed);
    e.step = step.data_ptr<int32_t>();
    e.max_z = static_cast<int>(max_z);
    e.samp = samp.data_ptr<int32_t>();
    e.truncated = truncated.data_ptr<int32_t>();
    launch_seal_extract(e, ptrs, cur_stream());
    check_cuda_err("SealArena.extract");
  }

  void check_params(const Tensor& params, const char* msg) const { check_vec(params, torch::kFloat32, model.P, msg); }

  // labels fp32 [B]; training = 0: no dropout
  void forward(const Tensor& params, const Tensor& labels, bool training, double p, int64_t seed, const Tensor& step) {
    c10::cuda::CUDAGuard guard(device);
    check_params(params, "SealArena.forward: params must be contiguous fp32 [num_params] on the arena's device");
    check_vec(labels, torch::kFloat32, ptrs.B, "SealArena.forward: labels must be contiguous fp32 [batch_size] on the device");
    TORCH_CHECK(p >= 0.0 && p < 1.0, "SealArena.forward: dropout must be in [0, 1)");
    check_counters(step, 0, "SealArena.forward: step must be int32 [>= 1] on the device");
    launch_seal_forward(model, ptrs, params.data_ptr<float>(), labels.data_ptr<float>(), training ? 1 : 0,
                        static_cast<float>(p), static_cast<uint64_t>(seed), step.data_ptr<int32_t>(), cur_stream());
    check_cuda_err("SealArena.forward");
  }

  void backward(const Tensor& params) {
    c10::cuda::CUDAGuard guard(device);
    check_params(params, "SealArena.backward: params must be contiguous fp32 [num_params] on the arena's device");
    launch_seal_backward(model, ptrs, params.data_ptr<float>(), partials.data_ptr<float>(), cur_stream());
    check_cuda_err("SealArena.backward");
  }

  void reduce(Tensor grad, Tensor loss) {
    c10::cuda::CUDAGuard guard(device);
    check_params(grad, "SealArena.reduce: grad must be contiguous fp32 [num_params] on the arena's device");
    check_vec(loss, torch::kFloat32, 1, "SealArena.reduce: loss must be fp32 [1] on the arena's device");
    launch_seal_reduce(model, ptrs, partials.data_ptr<float>(), grad.data_ptr<float>(), loss.data_ptr<float>(),
                       cur_stream());
    check_cuda_err("SealArena.reduce");
  }
};

static void dropout_bf16(Tensor Z, const Tensor& counters, int64_t n_hops, double p, int64_t seed, int64_t layer,
                         const c10::optional<Tensor>& step_dev) {
  c10::cuda::CUDAGuard guard(Z.device());
  TORCH_CHECK(Z.scalar_type() == torch::kBFloat16 && Z.is_contiguous() && Z.dim() == 2 && Z.size(1) % 8 == 0,
              "dropout_bf16: contiguous bf16 [rows, d], d % 8 == 0");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "dropout_bf16: p in [0, 1)");
  check_counters(counters, n_hops, "dropout_bf16: counters must be int32 [> n_hops] on the device");
  if (has(step_dev)) check_counters(*step_dev, 0, "dropout_bf16: step_dev must be int32 [>= 1] on the device");
  launch_dropout_bf16(Z.data_ptr(), counters.data_ptr<int32_t>(), n_hops, Z.size(0), Z.size(1),
                      static_cast<float>(p), static_cast<uint64_t>(seed), static_cast<int>(layer),
                      opt_ptr<int32_t>(step_dev), cur_stream());
  check_cuda_err("dropout_bf16");
}

static void softmax_nll(const Tensor& logits, int64_t C, const c10::optional<Tensor>& y,
                        const c10::optional<Tensor>& labels_all, const c10::optional<Tensor>& nodes,
                        const Tensor& counters, Tensor loss, Tensor dlogits,
                        const c10::optional<Tensor>& correct, const c10::optional<Tensor>& colsum, bool prezeroed) {
  c10::cuda::CUDAGuard guard(logits.device());
  TORCH_CHECK(logits.dim() == 2 && logits.size(1) % 8 == 0 && 1 <= C && C <= logits.size(1),
              "softmax_nll: logits must be [rows, ld] with ld a multiple of 8 and 1 <= C <= ld");
  check_rows(logits, torch::kBFloat16, logits.size(1), "softmax_nll: logits must be contiguous bf16 [rows, ld]");
  check_rows(dlogits, torch::kBFloat16, logits.size(1), "softmax_nll: dlogits must be contiguous bf16 of logits' shape");
  TORCH_CHECK(dlogits.size(0) == logits.size(0), "softmax_nll: dlogits must be contiguous bf16 of logits' shape");
  const bool direct = has(y);
  TORCH_CHECK(direct || (has(labels_all) && has(nodes)), "need y or (labels_all, nodes)");
  if (direct) {
    check_ids(*y, "softmax_nll: y must be contiguous int64 on the device");
  } else {
    check_ids(*labels_all, "softmax_nll: labels_all must be contiguous int64 on the device");
    check_ids(*nodes, "softmax_nll: nodes must be contiguous int64 on the device");
  }
  check_counters(counters, 1, "softmax_nll: counters must be int32 [> 1] on the device");
  TORCH_CHECK(on_dev(loss) && loss.scalar_type() == torch::kFloat32 && loss.numel() >= 1,
              "softmax_nll: loss must be fp32 [>= 1] on the device");
  if (has(correct)) check_counters(*correct, 0, "softmax_nll: correct must be int32 [>= 1] on the device");
  if (has(colsum)) check_vec(*colsum, torch::kFloat32, logits.size(1), "softmax_nll: colsum must be fp32 [ld]");
  launch_softmax_nll(logits.data_ptr(), logits.size(1), C, direct ? y->data_ptr<int64_t>() : nullptr,
                     direct ? nullptr : labels_all->data_ptr<int64_t>(), direct ? nullptr : nodes->data_ptr<int64_t>(),
                     counters.data_ptr<int32_t>(), logits.size(0), loss.data_ptr<float>(), dlogits.data_ptr(),
                     opt_ptr<int32_t>(correct), opt_ptr<float>(colsum), cur_stream(), prezeroed);
  check_cuda_err("softmax_nll");
}

static void sigmoid_bce(const Tensor& logits, int64_t T, const Tensor& label_bits, const Tensor& nodes,
                        const Tensor& counters, Tensor loss, Tensor dlogits, const c10::optional<Tensor>& counts,
                        const c10::optional<Tensor>& colsum, bool prezeroed) {
  c10::cuda::CUDAGuard guard(logits.device());
  TORCH_CHECK(logits.dim() == 2 && logits.size(1) % 8 == 0 && 1 <= T && T <= logits.size(1),
              "sigmoid_bce: logits must be [rows, ld] with ld a multiple of 8 and 1 <= T <= ld");
  check_rows(logits, torch::kBFloat16, logits.size(1), "sigmoid_bce: logits must be contiguous bf16 [rows, ld]");
  check_rows(dlogits, torch::kBFloat16, logits.size(1), "sigmoid_bce: dlogits must be contiguous bf16 of logits' shape");
  TORCH_CHECK(dlogits.size(0) == logits.size(0), "sigmoid_bce: dlogits must be contiguous bf16 of logits' shape");
  TORCH_CHECK(on_dev(label_bits) && label_bits.scalar_type() == torch::kUInt32 && label_bits.dim() == 2 &&
                  label_bits.size(1) == (T + 31) / 32 && label_bits.is_contiguous(),
              "sigmoid_bce: label_bits must be contiguous uint32 [num_nodes, ceil(T / 32)] on the device");
  check_ids(nodes, "sigmoid_bce: nodes must be contiguous int64 on the device");
  TORCH_CHECK(nodes.numel() >= logits.size(0), "sigmoid_bce: nodes must hold an id for every row of logits");
  check_counters(counters, 1, "sigmoid_bce: counters must be int32 [> 1] on the device");
  TORCH_CHECK(on_dev(loss) && loss.scalar_type() == torch::kFloat32 && loss.numel() >= 1,
              "sigmoid_bce: loss must be fp32 [>= 1] on the device");
  if (has(counts)) check_counters(*counts, 2, "sigmoid_bce: counts must be int32 [>= 3] on the device");
  if (has(colsum)) check_vec(*colsum, torch::kFloat32, logits.size(1), "sigmoid_bce: colsum must be fp32 [ld]");
  launch_sigmoid_bce(logits.data_ptr(), logits.size(1), T, static_cast<const uint32_t*>(label_bits.data_ptr()), label_bits.size(0),
                     nodes.data_ptr<int64_t>(), counters.data_ptr<int32_t>(), logits.size(0), loss.data_ptr<float>(),
                     dlogits.data_ptr(), opt_ptr<int32_t>(counts), opt_ptr<float>(colsum), cur_stream(), prezeroed);
  check_cuda_err("sigmoid_bce");
}

// (kernel, memset, memcpy) node counts of a captured CUDA graph: the launches one replay makes.  `raw_graph` is the
// cudaGraph_t of torch.cuda.CUDAGraph(keep_graph=True).raw_cuda_graph().
static std::tuple<int64_t, int64_t, int64_t> graph_node_counts(int64_t raw_graph) {
  TORCH_CHECK(raw_graph != 0, "graph_node_counts: null graph (capture with keep_graph=True)");
  cudaGraph_t graph = reinterpret_cast<cudaGraph_t>(static_cast<uintptr_t>(raw_graph));
  size_t n = 0;
  C10_CUDA_CHECK(cudaGraphGetNodes(graph, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  if (n > 0) C10_CUDA_CHECK(cudaGraphGetNodes(graph, nodes.data(), &n));
  int64_t kernels = 0, memsets = 0, memcpys = 0;
  for (cudaGraphNode_t node : nodes) {
    cudaGraphNodeType type;
    C10_CUDA_CHECK(cudaGraphNodeGetType(node, &type));
    kernels += type == cudaGraphNodeTypeKernel;
    memsets += type == cudaGraphNodeTypeMemset;
    memcpys += type == cudaGraphNodeTypeMemcpy;
  }
  return {kernels, memsets, memcpys};
}

static void zero_grads(Tensor g, const c10::optional<Tensor>& loss, const c10::optional<Tensor>& correct) {
  c10::cuda::CUDAGuard guard(g.device());
  TORCH_CHECK(g.scalar_type() == torch::kFloat32 && g.is_contiguous() && aligned16(g),
              "zero_grads: g must be contiguous 16-byte aligned fp32");
  if (has(loss))
    TORCH_CHECK(on_dev(*loss) && loss->scalar_type() == torch::kFloat32 && loss->numel() >= 1,
                "zero_grads: loss must be fp32 [>= 1] on the device");
  if (has(correct)) check_counters(*correct, 0, "zero_grads: correct must be int32 [>= 1] on the device");
  launch_zero_grads(g.data_ptr<float>(), g.numel(), opt_ptr<float>(loss), opt_ptr<int32_t>(correct), cur_stream());
  check_cuda_err("zero_grads");
}

static void colsum_bf16(const Tensor& X, const Tensor& counters, int64_t n_hops, Tensor out) {
  c10::cuda::CUDAGuard guard(X.device());
  const int64_t d = X.dim() == 2 ? X.size(1) : 0;
  TORCH_CHECK(d % 8 == 0 && d <= 2048, "colsum_bf16: width must be a multiple of 8 up to 2048");
  check_rows(X, torch::kBFloat16, d, "colsum_bf16: X must be contiguous bf16 [rows, d]");
  check_vec(out, torch::kFloat32, d, "colsum_bf16: out must be fp32 [d]");
  check_counters(counters, n_hops, "colsum_bf16: counters must be int32 [> n_hops] on the device");
  launch_colsum_bf16(X.data_ptr(), counters.data_ptr<int32_t>(), n_hops, X.size(0), d, out.data_ptr<float>(),
                     cur_stream());
  check_cuda_err("colsum_bf16");
}

static void zero_rows(Tensor p, const Tensor& counters, int64_t n_hops) {
  c10::cuda::CUDAGuard guard(p.device());
  const int64_t d = p.dim() == 2 ? p.size(1) : 0;
  TORCH_CHECK(d % 4 == 0, "zero_rows: width must be a multiple of 4");
  check_rows(p, torch::kFloat32, d, "zero_rows: p must be contiguous fp32 [rows, d]");
  check_counters(counters, n_hops, "zero_rows: counters must be int32 [> n_hops] on the device");
  launch_zero_rows(p.data_ptr<float>(), counters.data_ptr<int32_t>(), n_hops, p.size(0), d, cur_stream());
  check_cuda_err("zero_rows");
}

static void adam_step(Tensor p, const Tensor& g, Tensor m, Tensor v, const c10::optional<Tensor>& p_bf16,
                      double lr, double b1, double b2, double eps, double wd, const Tensor& step_dev,
                      double gscale) {
  c10::cuda::CUDAGuard guard(p.device());
  check_counters(step_dev, 1, "step_dev must be int32[2]: {steps taken, block ticket}");
  for (const Tensor* t : std::initializer_list<const Tensor*>{&p, &g, &m, &v})
    TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32, "adam: fp32 state");
  TORCH_CHECK(g.numel() >= p.numel() && m.numel() >= p.numel() && v.numel() >= p.numel() && p.is_contiguous() &&
              g.is_contiguous() && m.is_contiguous() && v.is_contiguous(), "adam: state size / layout mismatch");
  if (has(p_bf16))
    TORCH_CHECK(on_dev(*p_bf16) && p_bf16->scalar_type() == torch::kBFloat16 && p_bf16->is_contiguous() &&
                p_bf16->numel() >= p.numel(), "adam: p_bf16 must be a contiguous bf16 shadow of p on the device");
  launch_adam(p.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), opt_ptr(p_bf16),
              p.numel(), lr, b1, b2, eps, wd, step_dev.data_ptr<int32_t>(), gscale, cur_stream());
  check_cuda_err("adam");
}

static void sage_fused(RowTableHandle* feat, const c10::optional<Tensor>& nodes,
                       const c10::optional<Tensor>& src_local, int64_t d, const Tensor& counters,
                       int64_t n_hops_targets, const std::vector<Tensor>& ell,
                       const std::vector<int64_t>& ks, const Tensor& deg, const Tensor& w_packed,
                       const Tensor& bias, bool relu, Tensor z, const c10::optional<Tensor>& a_save) {
  c10::cuda::CUDAGuard guard(z.device());
  const bool local = has(src_local);
  const bool fp8 = feat != nullptr && !local && feat->dtype == torch::kUInt8;
  TORCH_CHECK(!fp8 || d == 128, "the MXFP8 loader of the fused kernel supports d = 128");
  const int64_t n_out = z.dim() == 2 ? z.size(1) : 0;
  check_rows(z, torch::kBFloat16, n_out, "sage_fused: z must be contiguous bf16 [rows, n_out]");
  TORCH_CHECK(sage_fused_supported(d, n_out),
              fmt("unsupported fused shape d=%lld n_out=%lld", static_cast<long long>(d), static_cast<long long>(n_out)));
  TORCH_CHECK(local || feat == nullptr || sage_fused_supported(d, n_out, &feat->tbl),
              "sage_fused: the fused kernel's 32-bit row handles cannot address this feature table "
              "(more than 16 parts, or a part of 2^28 rows or more)");
  check_vec(w_packed, torch::kBFloat16, 2 * d * n_out, "sage_fused: w_packed must be packed bf16 [n_out * 2d]");
  check_vec(bias, torch::kBFloat16, n_out, "sage_fused: bias must be bf16 [n_out]");
  SageFusedArgs f{};
  f.agg = make_agg(feat, nodes, src_local, d, counters, n_hops_targets, z.size(0), ell, ks, deg, nullptr);
  f.w_packed = w_packed.data_ptr();
  f.bias = bias.data_ptr();
  f.n_out = n_out;
  f.relu = relu;
  f.z = z.data_ptr();
  f.feat_fp8 = fp8 ? 1 : 0;
  f.a_save = nullptr;
  if (has(a_save)) {
    check_rows(*a_save, torch::kBFloat16, 2 * d, "sage_fused: a_save must be contiguous bf16 [>= rows of z, 2d]");
    TORCH_CHECK(a_save->size(0) >= z.size(0), "sage_fused: a_save must be contiguous bf16 [>= rows of z, 2d]");
    f.a_save = a_save->data_ptr();
  }
  launch_sage_fused(f, at::cuda::getCurrentDeviceProperties()->multiProcessorCount, cur_stream());
  check_cuda_err("sage_fused");
}

// ---------------------------------------------------------------------------
// TcGemm: a cached launch of the TMA-fed wgmma GEMM kernel (csrc/cuda/tc_gemm.cu) over fixed engine buffers.
// Tensor maps are encoded once; the batch-dependent extent is read from the sampler's device counters, so
// run() is a single static launch (CUDA-graph capturable).  Up to two problems share a launch.  The plan owns the
// kernel's 8-byte work ticket, which the kernel leaves zeroed: launches of one plan must therefore be ordered (never
// two in flight at once; every engine runs a plan on one stream).
// ---------------------------------------------------------------------------
struct TcGemm {
  TcGemmLaunch L;
  int device;
  std::vector<Tensor> keep;   // keeps every operand alive
  Tensor tickets;
  explicit TcGemm(int dev) : device(dev) {
    std::memset(&L, 0, sizeof(L));
    tickets = torch::zeros({2}, torch::dtype(torch::kInt32).device(torch::kCUDA, dev));
    L.args.tickets = tickets.data_ptr<int32_t>();
  }
  static int pick_bn(int64_t n) { return n % 256 == 0 ? 256 : (n % 128 == 0 ? 128 : 64); }
  void check_bf16(const Tensor& t, const char* what) {
    TORCH_CHECK(on_dev(t) && t.scalar_type() == torch::kBFloat16 && t.dim() == 2 && t.stride(1) == 1 &&
                (t.stride(0) * 2) % 16 == 0 && aligned16(t),
                fmt("TcGemm: %s must be a 2-D bf16 CUDA tensor with unit inner stride and 16-byte aligned rows", what));
  }
  void tmap(int slot, const Tensor& t, int box_cols, int box_rows) {
    const int rc = make_tmap_bf16_2d(L.maps[slot], t.data_ptr(), t.size(0), t.size(1), t.stride(0), box_cols, box_rows);
    TORCH_CHECK(rc == 0, fmt("TcGemm: cuTensorMapEncodeTiled failed (rc=%d)", rc));
    keep.push_back(t);
  }
  TcProblem& next() {
    TORCH_CHECK(L.args.n_prob < 2, "TcGemm: at most two problems per launch");
    return L.args.p[L.args.n_prob];
  }
  void set_dyn(TcProblem& p, const Tensor& counters, int64_t idx, int64_t cap, bool is_k) {
    check_counters(counters, idx, "TcGemm: counters must be int32 [> dyn_idx] on the device");
    p.dyn = counters.data_ptr<int32_t>();
    p.dyn_idx = static_cast<int>(idx);
    p.dyn_cap = static_cast<int>(cap);
    p.dyn_is_k = is_k ? 1 : 0;
    keep.push_back(counters);
  }
  // Z[rows, N] = act(A[rows, K] . W[N, K]^T + bias); rows = min(counters[dyn_idx], A.size(0))
  void add_forward(const Tensor& A, const Tensor& W, const c10::optional<Tensor>& bias, bool relu, Tensor Z,
                   const Tensor& counters, int64_t dyn_idx) {
    c10::cuda::CUDAGuard guard(A.device());
    check_bf16(A, "A"); check_bf16(W, "W"); check_bf16(Z, "Z");
    const int64_t K = A.size(1), N = W.size(0);
    TORCH_CHECK(W.size(1) == K && Z.size(1) == N && Z.size(0) >= A.size(0) && N % 64 == 0 && K % 8 == 0,
                "TcGemm.add_forward: A [rows, K], W [N, K], Z [>= rows, N] with N a multiple of 64 and K of 8");
    const int slot = 3 * L.args.n_prob;
    TcProblem& p = next();
    p.a_mn = 0; p.b_mn = 0; p.epi = 0; p.bn = pick_bn(N);
    p.m = A.size(0); p.n = N; p.k = K;
    set_dyn(p, counters, dyn_idx, A.size(0), false);
    p.bias = nullptr;
    if (has(bias)) {
      check_vec(*bias, torch::kBFloat16, N, "TcGemm.add_forward: bias must be 16-byte aligned bf16 [N]");
      p.bias = bias->data_ptr();
      keep.push_back(*bias);
    }
    p.relu = relu ? 1 : 0;
    tmap(slot + 0, A, 64, 128);
    tmap(slot + 1, W, 64, p.bn);
    tmap(slot + 2, Z, 64, 128);
    L.max_items += static_cast<int>((A.size(0) + 127) / 128 * (N / p.bn));
    ++L.args.n_prob;
  }
  // dA[rows, N] = dPre[rows, Kd] . W[Kd, N]  (W row-major = N contiguous: the MN-major B operand)
  void add_dgrad(const Tensor& dPre, const Tensor& W, Tensor dA, const Tensor& counters, int64_t dyn_idx) {
    c10::cuda::CUDAGuard guard(dPre.device());
    check_bf16(dPre, "dPre"); check_bf16(W, "W"); check_bf16(dA, "dA");
    const int64_t Kd = dPre.size(1), N = W.size(1);
    TORCH_CHECK(W.size(0) == Kd && dA.size(1) == N && dA.size(0) >= dPre.size(0) && N % 64 == 0 && Kd % 8 == 0,
                "TcGemm.add_dgrad: dPre [rows, Kd], W [Kd, N], dA [>= rows, N] with N a multiple of 64 and Kd of 8");
    const int slot = 3 * L.args.n_prob;
    TcProblem& p = next();
    p.a_mn = 0; p.b_mn = 1; p.epi = 0; p.bn = pick_bn(N);
    p.m = dPre.size(0); p.n = N; p.k = Kd;
    set_dyn(p, counters, dyn_idx, dPre.size(0), false);
    p.bias = nullptr; p.relu = 0;
    tmap(slot + 0, dPre, 64, 128);
    tmap(slot + 1, W, 64, 64);
    tmap(slot + 2, dA, 64, 128);
    L.max_items += static_cast<int>((dPre.size(0) + 127) / 128 * (N / p.bn));
    ++L.args.n_prob;
  }
  // gW[M, N] += dPre[rows, M]^T . A[rows, N], rows = min(counters[dyn_idx], dPre.size(0)); fp32 split-K red-add
  // (gW must be zeroed by the caller; dPre rows beyond the batch must be zero up to its capacity)
  void add_wgrad(const Tensor& dPre, const Tensor& A, Tensor gW, const Tensor& counters, int64_t dyn_idx) {
    c10::cuda::CUDAGuard guard(dPre.device());
    check_bf16(dPre, "dPre"); check_bf16(A, "A");
    const int64_t M = dPre.size(1), N = A.size(1);
    TORCH_CHECK(A.size(0) >= dPre.size(0) && N % 64 == 0 && M % 8 == 0,
                "TcGemm.add_wgrad: dPre [rows, M], A [>= rows, N] with N a multiple of 64 and M of 8");
    TORCH_CHECK(on_dev(gW) && gW.scalar_type() == torch::kFloat32 && gW.dim() == 2 && gW.size(0) == M &&
                gW.size(1) == N && gW.stride(1) == 1 && gW.stride(0) % 4 == 0 &&
                reinterpret_cast<uintptr_t>(gW.data_ptr()) % 16 == 0, "TcGemm: gW must be fp32 [M, N], 16-byte aligned");
    const int slot = 3 * L.args.n_prob;
    TcProblem& p = next();
    p.a_mn = 1; p.b_mn = 1; p.epi = 1; p.bn = pick_bn(N);
    p.m = M; p.n = N; p.k = dPre.size(0);
    set_dyn(p, counters, dyn_idx, dPre.size(0), true);
    p.bias = nullptr; p.relu = 0;
    p.out32 = gW.data_ptr<float>(); p.ld32 = static_cast<int>(gW.stride(0)); p.m_valid = static_cast<int>(M);
    keep.push_back(gW);
    tmap(slot + 0, dPre, 64, 64);
    tmap(slot + 1, A, 64, 64);
    L.max_items += 1 << 20;   // split-K fills the grid
    ++L.args.n_prob;
  }
  void run() {
    TORCH_CHECK(L.args.n_prob >= 1, "TcGemm: no problem added");
    c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
    launch_tc_gemm(L, at::cuda::getCurrentDeviceProperties()->multiProcessorCount, cur_stream());
    check_cuda_err("tc_gemm");
  }
};


static void enable_peer_access(int dev, int peer) {
  if (dev == peer) return;
  c10::cuda::CUDAGuard guard(dev);
  int can = 0;
  cudaDeviceCanAccessPeer(&can, dev, peer);
  TORCH_CHECK(can, fmt("GPU %d cannot access peer GPU %d", dev, peer));
  cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return; }
  TORCH_CHECK(e == cudaSuccess, fmt("cudaDeviceEnablePeerAccess: %s", cudaGetErrorString(e)));
}

// ---------------------------------------------------------------------------
// PeerBuffer: cudaMalloc'ed shard that other processes map with CUDA IPC *on their own
// device* (cudaIpcMemLazyEnablePeerAccess), so their kernels can dereference it over
// NVLink.  (Memory imported through torch's own IPC path is opened in the exporter
// device's context and is not reachable from kernels running on the importer's GPU.)
// ---------------------------------------------------------------------------
struct PeerBuffer : public std::enable_shared_from_this<PeerBuffer> {
  void* ptr = nullptr;
  size_t bytes = 0;
  int device = 0;       // device whose kernels may use `ptr`
  bool imported = false;

  ~PeerBuffer() {
    if (ptr == nullptr) return;
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    if (imported) cudaIpcCloseMemHandle(ptr); else cudaFree(ptr);
    cudaSetDevice(cur);
  }

  static std::shared_ptr<PeerBuffer> allocate(int device, int64_t nbytes) {
    c10::cuda::CUDAGuard guard(device);
    auto b = std::make_shared<PeerBuffer>();
    b->device = device;
    b->bytes = std::max<int64_t>(nbytes, 256);
    cudaError_t e = cudaMalloc(&b->ptr, b->bytes);
    TORCH_CHECK(e == cudaSuccess, fmt("cudaMalloc(%zu) failed: %s", b->bytes, cudaGetErrorString(e)));
    return b;
  }

  py::bytes handle() const {
    TORCH_CHECK(!imported, "only the owner can export a handle");
    c10::cuda::CUDAGuard guard(device);
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, ptr);
    TORCH_CHECK(e == cudaSuccess, fmt("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e)));
    return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
  }

  static std::shared_ptr<PeerBuffer> open(const std::string& handle_bytes, int my_device, int64_t nbytes) {
    TORCH_CHECK(handle_bytes.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
    c10::cuda::CUDAGuard guard(my_device);
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle_bytes.data(), sizeof(h));
    auto b = std::make_shared<PeerBuffer>();
    b->device = my_device;
    b->bytes = nbytes;
    b->imported = true;
    cudaError_t e = cudaIpcOpenMemHandle(&b->ptr, h, cudaIpcMemLazyEnablePeerAccess);
    TORCH_CHECK(e == cudaSuccess, fmt("cudaIpcOpenMemHandle failed: %s", cudaGetErrorString(e)));
    return b;
  }

  // non-owning tensor view (keeps the buffer alive through the deleter)
  Tensor as_tensor(torch::ScalarType dtype, std::vector<int64_t> sizes) {
    int64_t n = 1;
    for (auto v : sizes) n *= v;
    TORCH_CHECK(static_cast<size_t>(n) * c10::elementSize(dtype) <= bytes, "view exceeds the peer buffer");
    std::shared_ptr<PeerBuffer> keep = shared_from_this();
    auto opts = torch::TensorOptions().dtype(dtype).device(torch::kCUDA, device);
    return torch::from_blob(ptr, sizes, [keep](void*) mutable { keep.reset(); }, opts);
  }
};

// PeerGroup: the per-rank view of all ranks' gradient buffers + barrier flags.
struct PeerGroup {
  PeerPtrs p{};
  std::vector<Tensor> keep;
  Tensor epoch, err;
  int device;

  PeerGroup(int dev, int rank, std::vector<Tensor> grads, std::vector<Tensor> flags) : device(dev) {
    c10::cuda::CUDAGuard guard(dev);
    TORCH_CHECK(grads.size() == flags.size() && grads.size() <= kMaxParts,
                "PeerGroup: one gradient buffer and one flag array per rank, at most 16 ranks");
    p.world = grads.size();
    p.rank = rank;
    for (size_t r = 0; r < grads.size(); ++r) {
      TORCH_CHECK(grads[r].is_cuda() && grads[r].scalar_type() == torch::kFloat32 && grads[r].is_contiguous(),
                  "PeerGroup: gradient buffers must be contiguous fp32 CUDA tensors");
      TORCH_CHECK(flags[r].is_cuda() && flags[r].scalar_type() == torch::kInt32 && flags[r].is_contiguous() &&
                  flags[r].numel() >= 2 * p.world, "PeerGroup: flags must be contiguous int32 [2 * world] CUDA tensors");
      p.g[r] = grads[r].data_ptr<float>();
      p.flags[r] = flags[r].data_ptr<int32_t>();
      keep.push_back(grads[r]);
      keep.push_back(flags[r]);
    }
    auto o32 = torch::TensorOptions().dtype(torch::kInt32).device(torch::kCUDA, dev);
    epoch = torch::zeros({2}, o32);
    err = torch::zeros({1}, o32);
  }

  void barrier(int64_t which) {
    c10::cuda::CUDAGuard guard(device);
    launch_peer_barrier(p, which, epoch.data_ptr<int32_t>(), err.data_ptr<int32_t>(), cur_stream());
    check_cuda_err("peer_barrier");
  }

  void adam(Tensor param, Tensor m, Tensor v, const c10::optional<Tensor>& p_bf16, double lr, double b1, double b2,
            double eps, double wd, const Tensor& step_dev, double gscale) {
    c10::cuda::CUDAGuard guard(device);
    TORCH_CHECK(param.numel() % 4 == 0, "flat parameter buffer must be padded to a multiple of 4");
    check_counters(step_dev, 1, "step_dev must be int32[2]: {steps taken, block ticket}");
    for (const Tensor* t : {&param, &m, &v})
      TORCH_CHECK(on_dev(*t) && t->scalar_type() == torch::kFloat32 && t->is_contiguous() && t->numel() == param.numel(),
                  "PeerGroup.adam: param, m and v must be contiguous fp32 of one size on the group's device");
    if (has(p_bf16))
      TORCH_CHECK(on_dev(*p_bf16) && p_bf16->scalar_type() == torch::kBFloat16 && p_bf16->is_contiguous() &&
                  p_bf16->numel() >= param.numel(), "PeerGroup.adam: p_bf16 must be a contiguous bf16 shadow of param");
    launch_adam_peer(p, param.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), opt_ptr(p_bf16),
                     param.numel(), lr, b1, b2, eps, wd, step_dev.data_ptr<int32_t>(), gscale, cur_stream(),
                     err.data_ptr<int32_t>());
    check_cuda_err("adam_peer");
  }
};

static void multimem_copy(const Tensor& src, int64_t mc_ptr, int64_t dst_byte_offset) {
  c10::cuda::CUDAGuard guard(src.device());
  TORCH_CHECK(src.is_contiguous() && aligned16(src), "multimem_copy: src must be contiguous and 16-byte aligned");
  const int64_t nbytes = src.numel() * src.element_size();
  TORCH_CHECK(nbytes % 16 == 0 && dst_byte_offset % 16 == 0 && mc_ptr != 0,
              "multimem_copy: size and destination offset must be multiples of 16 bytes, mc_ptr non-null");
  launch_multimem_copy(src.data_ptr(), reinterpret_cast<void*>(mc_ptr + dst_byte_offset), nbytes, cur_stream());
  check_cuda_err("multimem_copy");
}

static Tensor pack_weight(const Tensor& w) {
  c10::cuda::CUDAGuard guard(w.device());
  TORCH_CHECK(w.scalar_type() == torch::kBFloat16 && w.is_contiguous() && w.dim() == 2,
              "pack_weight: w must be contiguous bf16 [N, K]");
  TORCH_CHECK(w.size(1) % 64 == 0 && w.size(0) % 16 == 0, "W must be [N%16, K%64]");
  Tensor out = torch::empty_like(w);
  launch_pack_weight(w.data_ptr(), w.size(0), w.size(1), out.data_ptr(), cur_stream());
  check_cuda_err("pack_weight");
  return out;
}

static void pack_weight_into(const Tensor& w, Tensor out) {
  c10::cuda::CUDAGuard guard(w.device());
  TORCH_CHECK(w.scalar_type() == torch::kBFloat16 && w.is_contiguous() && w.dim() == 2,
              "pack_weight_into: w must be contiguous bf16 [N, K]");
  check_vec(out, torch::kBFloat16, w.numel(), "pack_weight_into: out must be contiguous bf16 of w's size");
  launch_pack_weight(w.data_ptr(), w.size(0), w.size(1), out.data_ptr(), cur_stream());
  check_cuda_err("pack_weight");
}

}  // namespace glt

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  using namespace glt;
  m.doc() = "graphlearn_for_pytorch_b200 native core (CPU reference ops + sm_90a kernels)";

  // ---- CPU ops ----
  m.def("coo_to_csr", &coo_to_csr);
  m.def("cpu_sample_neighbors", &cpu_sample_neighbors);
  m.def("cpu_sample_neighbors_weighted", &cpu_sample_neighbors_weighted, py::arg("indptr"), py::arg("indices"),
        py::arg("eids"), py::arg("weights"), py::arg("seeds"), py::arg("k"), py::arg("with_edge"), py::arg("seed"),
        py::arg("stream"), py::arg("replace") = false);
  m.def("cpu_negative_sample", &cpu_negative_sample);
  m.def("cpu_node_subgraph", &cpu_node_subgraph);
  m.def("cpu_random_walk", &cpu_random_walk);
  m.def("cpu_stitch", &cpu_stitch);
  m.def("cpu_nbr_prob", &cpu_nbr_prob);
  m.def("cpu_gather_rows", &cpu_gather_rows, py::arg("table"), py::arg("ids"), py::arg("id2index"), py::arg("offset"),
        py::arg("out"), py::arg("pos"));
  py::class_<CpuIdTable>(m, "CpuIdTable")
      .def(py::init<int64_t>())
      .def("reset", &CpuIdTable::reset)
      .def("insert", &CpuIdTable::insert)
      .def("lookup", &CpuIdTable::lookup)
      .def("keys", &CpuIdTable::keys, py::arg("start") = 0)
      .def("size", &CpuIdTable::size);

  // ---- shm sample queue ----
  py::register_exception<QueueTimeoutError>(m, "QueueTimeoutError");
  py::register_exception<QueueClosedError>(m, "QueueClosedError");
  py::class_<SampleQueue>(m, "SampleQueue")
      .def(py::init<size_t, size_t>(), py::arg("max_msgs"), py::arg("buf_bytes"))
      .def(py::init<const std::string&>(), py::arg("name"))
      .def_property_readonly("name", &SampleQueue::name)
      .def("send", &SampleQueue::send, py::call_guard<py::gil_scoped_release>())
      .def("recv", &SampleQueue::recv, py::arg("timeout_ms") = 0, py::call_guard<py::gil_scoped_release>())
      .def("empty", &SampleQueue::empty)
      .def("size", &SampleQueue::size)
      .def("close", &SampleQueue::close)
      .def("pin_memory", &SampleQueue::pin_memory);

  // ---- CUDA graph / tables ----
  py::class_<GraphHandle>(m, "GraphHandle")
      .def(py::init<int>())
      .def("add_shard", &GraphHandle::add_shard)
      .def_readonly("num_rows", &GraphHandle::num_rows)
      .def_readonly("has_eids", &GraphHandle::has_eids)
      .def_readonly("has_weights", &GraphHandle::has_weights)
      .def_property_readonly("num_parts", [](const GraphHandle& g) { return g.tbl.num_parts; })
      .def("sample_one_hop", &GraphHandle::sample_one_hop)
      .def("lookup_degree", &GraphHandle::lookup_degree)
      .def("full_neighbors", &GraphHandle::full_neighbors)
      .def("negative_sample", &GraphHandle::negative_sample)
      .def("random_walk", &GraphHandle::random_walk)
      .def("nbr_prob", &GraphHandle::nbr_prob);
  py::class_<DeviceTable>(m, "DeviceTable")
      .def(py::init<int, int64_t>())
      .def("clear", &DeviceTable::clear)
      .def("insert", &DeviceTable::insert)
      .def("init_ordered", &DeviceTable::init_ordered)
      .def("lookup", &DeviceTable::lookup)
      .def("size", &DeviceTable::size)
      .def("subgraph", &DeviceTable::subgraph)
      .def_readonly("nodes", &DeviceTable::nodes)
      .def_readonly("cursor", &DeviceTable::cursor)
      .def_readonly("capacity", &DeviceTable::cap_nodes);
  py::class_<SamplerArena>(m, "SamplerArena")
      .def(py::init<int, int64_t, std::vector<int64_t>, bool, int64_t, std::vector<int64_t>>(), py::arg("device"),
           py::arg("max_seeds"), py::arg("fanouts"), py::arg("with_edge"), py::arg("num_graph_nodes"),
           py::arg("cap_override") = std::vector<int64_t>{})
      .def("sample", &SamplerArena::sample, py::arg("graph"), py::arg("seeds"), py::arg("n_dev"), py::arg("seed"),
           py::arg("stream_base"), py::arg("weighted"), py::arg("replace"), py::arg("use_dev_step"),
           py::arg("step_inc") = 0)
      .def("to_coo", &SamplerArena::to_coo)
      .def_readonly("nodes", &SamplerArena::nodes)
      .def_readonly("deg", &SamplerArena::deg)
      .def_readonly("counters", &SamplerArena::counters)
      .def_readonly("seed_local", &SamplerArena::seed_local)
      .def_readonly("step", &SamplerArena::step)
      .def("enable_transpose", &SamplerArena::enable_transpose)
      // rebuilds the transposed adjacency from `counters`, `deg` and `ell` as they stand (sample() builds it itself);
      // lets a batch laid out by hand be transposed
      .def("build_transpose", [](SamplerArena& a) {
        c10::cuda::CUDAGuard guard(a.device);
        TORCH_CHECK(a.tr_hops > 0, "call enable_transpose(n_hops) first");
        a.build_transpose(cur_stream());
        check_cuda_err("build_transpose");
      })
      .def_readwrite("deterministic", &SamplerArena::deterministic)
      .def_readonly("tr_hops", &SamplerArena::tr_hops)
      .def_readonly("tr_off", &SamplerArena::tr_off)
      .def_readonly("tr_cnt", &SamplerArena::tr_cnt)
      .def_readonly("tr_tgt", &SamplerArena::tr_tgt)
      .def_readonly("tr_meta", &SamplerArena::tr_meta)
      .def_readonly("tr_meta_inv", &SamplerArena::tr_meta_inv)
      .def_readonly("ell", &SamplerArena::ell)
      .def_readonly("ell_eids", &SamplerArena::ell_eids)
      .def_readonly("cap_rows", &SamplerArena::cap_rows)
      .def_readonly("cap_nodes", &SamplerArena::cap_nodes)
      .def_readonly("fanouts", &SamplerArena::fanouts);
  py::class_<HeteroArena>(m, "HeteroArena")
      .def(py::init<int, int64_t, std::vector<GraphHandle*>, std::vector<int64_t>, std::vector<int64_t>,
                    std::vector<std::vector<int64_t>>, std::vector<int64_t>, std::vector<int64_t>, bool, int64_t, bool,
                    bool, int64_t, std::vector<std::vector<int64_t>>>(),
           py::arg("device"), py::arg("n_types"), py::arg("graphs"), py::arg("key_type"), py::arg("nbr_type"),
           py::arg("fanouts"), py::arg("num_nodes"), py::arg("max_seeds"), py::arg("with_edge") = false,
           py::arg("seed") = 0, py::arg("weighted") = false, py::arg("replace") = false, py::arg("cap_limit") = 0,
           py::arg("cap_override") = std::vector<std::vector<int64_t>>{}, py::keep_alive<1, 4>())
      .def("sample", &HeteroArena::sample, py::arg("seed_types"), py::arg("seeds"), py::arg("step_inc") = 1)
      .def("to_coo", &HeteroArena::to_coo)
      .def("seed_local_of", &HeteroArena::seed_local_of)
      .def("overflow_index", &HeteroArena::overflow_index)
      .def("nodes_of", &HeteroArena::nodes_of)
      .def("deg_of", &HeteroArena::deg_of)
      .def("ell_of", &HeteroArena::ell_of)
      .def_readonly("counters", &HeteroArena::counters)
      .def_readonly("step", &HeteroArena::step)
      .def_readonly("cap_rows", &HeteroArena::cap_rows)
      .def_readonly("cap_nodes", &HeteroArena::cap_nodes)
      .def_readonly("hops", &HeteroArena::hops)
      .def_readonly("n_types", &HeteroArena::n_types)
      .def_readonly("n_rel", &HeteroArena::n_rel);
  py::class_<RowTableHandle>(m, "RowTableHandle")
      .def(py::init<int>())
      .def("append", &RowTableHandle::append, py::arg("part"), py::arg("remote") = false)
      .def("num_rows", &RowTableHandle::num_rows)
      .def_readonly("width", &RowTableHandle::width)
      .def_property_readonly("is_uint8", [](const RowTableHandle& t) { return t.dtype == torch::kUInt8; })
      .def_property_readonly("num_parts", [](const RowTableHandle& t) { return t.tbl.num_parts; })
      .def("gather", &RowTableHandle::gather, py::arg("idx"), py::arg("id2index") = py::none(),
           py::arg("out_width") = 0)
      .def("gather_into", &RowTableHandle::gather_into)
      .def("gather_mxfp8", &RowTableHandle::gather_mxfp8)
      .def("gather_mxfp8_into", &RowTableHandle::gather_mxfp8_into)
      .def("all_local", &RowTableHandle::all_local);

  // ---- GraphSAGE engine ----
  m.def("sage_aggregate", &sage_aggregate);
  m.def("sage_full_aggregate", &sage_full_aggregate, py::arg("graph"), py::arg("feat"), py::arg("src"),
        py::arg("src_col"), py::arg("self_col"), py::arg("d"), py::arg("r0"), py::arg("r1"), py::arg("combine"),
        py::arg("bias"), py::arg("relu"), py::arg("out"), py::arg("mean_only") = false);
  m.def("label_prop", &label_prop, py::arg("graph"), py::arg("base"), py::arg("c"), py::arg("num_layers"),
        py::arg("alpha"), py::arg("norm"), py::arg("lo"), py::arg("hi"), py::arg("fixed") = py::none());
  m.def("link_topk", &link_topk, py::arg("emb"), py::arg("queries"), py::arg("k"), py::arg("lo"), py::arg("hi"),
        py::arg("exclude") = nullptr, py::arg("splits") = 0);
  m.def("sage_aggregate_block", &sage_aggregate_block);
  m.def("sage_scatter_block", &sage_scatter_block);
  m.def("add_block_f32", &add_block_f32);
  m.def("relu_bwd_cast", &relu_bwd_cast, py::arg("dH"), py::arg("Z"), py::arg("counters"), py::arg("n_hops"),
        py::arg("dPre"), py::arg("colsum"), py::arg("prezeroed") = false, py::arg("gscale") = 1.0,
        py::arg("relu") = true);
  m.def("link_seeds", &link_seeds, py::arg("graph"), py::arg("pos"), py::arg("num_nodes"), py::arg("neg_ratio"),
        py::arg("seed"), py::arg("step"), py::arg("seeds"), py::arg("n_pairs"));
  m.def("link_bce", &link_bce, py::arg("Z"), py::arg("C"), py::arg("seed_local"), py::arg("P"), py::arg("B"),
        py::arg("n_pairs"), py::arg("loss"), py::arg("correct"), py::arg("dZ"));
  py::class_<MetaPath>(m, "MetaPath")
      .def(py::init<int, std::vector<GraphHandle*>, std::vector<int64_t>, std::vector<int64_t>>(), py::arg("device"),
           py::arg("graphs"), py::arg("slot_off"), py::arg("slot_n"), py::keep_alive<1, 3>())
      .def_readonly("R", &MetaPath::R)
      .def_readonly("rows", &MetaPath::rows);
  py::class_<SealArena>(m, "SealArena")
      .def(py::init<int, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t>(), py::arg("device"),
           py::arg("batch_size"), py::arg("max_nodes"), py::arg("max_edges"), py::arg("hidden"), py::arg("num_layers"),
           py::arg("num_labels"), py::arg("k"), py::arg("cap_max") = 0)
      .def("extract", &SealArena::extract, py::arg("graph"), py::arg("links"), py::arg("num_nodes"), py::arg("hops"),
           py::arg("caps"), py::arg("seed"), py::arg("step"), py::arg("max_z"), py::arg("truncated"))
      .def("forward", &SealArena::forward, py::arg("params"), py::arg("labels"), py::arg("training"), py::arg("p"),
           py::arg("seed"), py::arg("step"))
      .def("backward", &SealArena::backward, py::arg("params"))
      .def("reduce", &SealArena::reduce, py::arg("grad"), py::arg("loss"))
      .def_property_readonly("num_params", [](const SealArena& a) { return a.model.P; })
      .def_property_readonly("dense", [](const SealArena& a) { return a.model.dense; })
      .def_readonly("layout", &SealArena::layout)
      .def_readonly("nodes", &SealArena::nodes).def_readonly("z", &SealArena::z)
      .def_readonly("meta", &SealArena::meta).def_readonly("sptr", &SealArena::sptr)
      .def_readonly("scol", &SealArena::scol).def_readonly("dptr", &SealArena::dptr)
      .def_readonly("dcol", &SealArena::dcol).def_readonly("X", &SealArena::X)
      .def_readonly("C1", &SealArena::C1).def_readonly("flat", &SealArena::flat)
      .def_readonly("H1", &SealArena::H1).def_readonly("mask", &SealArena::mask)
      .def_readonly("sel", &SealArena::sel).def_readonly("logits", &SealArena::logits)
      .def_readonly("lossv", &SealArena::lossv).def_readonly("partials", &SealArena::partials);
  m.def("metapath_walk", &metapath_walk, py::arg("metapath"), py::arg("starts"), py::arg("walks_per_node"),
        py::arg("context_size"), py::arg("seed"), py::arg("step"), py::arg("walks"), py::arg("n_valid"));
  m.def("node2vec_walk", &node2vec_walk, py::arg("metapath"), py::arg("starts"), py::arg("walks_per_node"),
        py::arg("context_size"), py::arg("seed"), py::arg("step"), py::arg("walks"), py::arg("n_valid"), py::arg("p"),
        py::arg("q"));
  m.def("sgns_negatives", &sgns_negatives, py::arg("metapath"), py::arg("walks"), py::arg("context_size"),
        py::arg("num_neg"), py::arg("seed"), py::arg("step"), py::arg("neg"));
  m.def("sgns_loss_grad", &sgns_loss_grad, py::arg("metapath"), py::arg("walks"), py::arg("neg"),
        py::arg("context_size"), py::arg("num_neg"), py::arg("emb"), py::arg("n_valid"), py::arg("grad"),
        py::arg("touched"), py::arg("loss"));
  m.def("sparse_adam", &sparse_adam, py::arg("metapath"), py::arg("emb"), py::arg("grad"), py::arg("m"), py::arg("v"),
        py::arg("touched"), py::arg("step"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"));
  m.def("m2v_begin", &m2v_begin, py::arg("state"));
  m.def("kge_negatives", &kge_negatives, py::arg("count"), py::arg("batch_size"), py::arg("num_neg"), py::arg("N"),
        py::arg("seed"), py::arg("step"), py::arg("neg"));
  m.def("kge_loss_grad", &kge_loss_grad, py::arg("model"), py::arg("trip"), py::arg("count"), py::arg("neg"),
        py::arg("ent"), py::arg("rel"), py::arg("margin"), py::arg("p"), py::arg("grad_ent"), py::arg("grad_rel"),
        py::arg("touched_ent"), py::arg("touched_rel"), py::arg("loss"));
  m.def("kge_score", &kge_score, py::arg("model"), py::arg("ent"), py::arg("rel"), py::arg("h"), py::arg("r"),
        py::arg("t"), py::arg("margin"), py::arg("p"));
  m.def("kge_rank", &kge_rank, py::arg("model"), py::arg("ent"), py::arg("rel"), py::arg("h"), py::arg("r"),
        py::arg("t"), py::arg("tail"), py::arg("keys"), py::arg("margin"), py::arg("p"), py::arg("splits") = 0);
  m.def("kge_sparse_adam", &kge_sparse_adam, py::arg("w"), py::arg("grad"), py::arg("m"), py::arg("v"),
        py::arg("touched"), py::arg("step"), py::arg("lr"), py::arg("b1"), py::arg("b2"), py::arg("eps"));
  m.def("dropout_bf16", &dropout_bf16, py::arg("Z"), py::arg("counters"), py::arg("n_hops"), py::arg("p"),
        py::arg("seed"), py::arg("layer"), py::arg("step_dev") = py::none());
  m.def("zero_grads", &zero_grads);
  m.def("set_pdl", [](bool on) { return set_pdl(on ? 1 : 0) != 0; });
  m.def("graph_node_counts", &graph_node_counts, py::arg("raw_graph"));
  m.def("sage_gather_bwd", &sage_gather_bwd, py::arg("dA"), py::arg("d"), py::arg("arena"), py::arg("n_hops_targets"),
        py::arg("Z"), py::arg("dPre"), py::arg("colsum"), py::arg("prezeroed") = false, py::arg("gscale") = 1.0);
  m.def("gat_scores", &gat_scores, py::arg("P0"), py::arg("att0"), py::arg("out0"), py::arg("counters0"),
        py::arg("idx0"), py::arg("P1") = py::none(), py::arg("att1") = py::none(), py::arg("out1") = py::none(),
        py::arg("counters1") = py::none(), py::arg("idx1") = 0, py::arg("zero") = py::none(), py::arg("heads") = 1);
  m.def("gat_aggregate", &gat_aggregate, py::arg("P"), py::arg("as_"), py::arg("ad"), py::arg("heads"),
        py::arg("counters"), py::arg("n_hops_targets"), py::arg("ell"), py::arg("ks"), py::arg("deg"), py::arg("alpha"),
        py::arg("acc") = py::none(), py::arg("first") = true, py::arg("last") = true, py::arg("bias") = py::none(),
        py::arg("act") = false, py::arg("p") = 0.0, py::arg("seed") = 0, py::arg("layer") = 0,
        py::arg("step_dev") = py::none(), py::arg("Z") = py::none());
  m.def("gat_backward", &gat_backward, py::arg("G"), py::arg("P"), py::arg("heads"), py::arg("counters"),
        py::arg("n_hops_targets"), py::arg("ell"), py::arg("ks"), py::arg("deg"), py::arg("alpha"), py::arg("dal"),
        py::arg("dP"), py::arg("da_src"), py::arg("da_dst"));
  m.def("gat_score_bwd", &gat_score_bwd, py::arg("P_src"), py::arg("dP_src"), py::arg("da_src"), py::arg("att_src"),
        py::arg("g_att_src"), py::arg("dPb_src"), py::arg("ctr_src"), py::arg("idx_src"), py::arg("da_dst"),
        py::arg("att_dst"), py::arg("g_att_dst"), py::arg("ctr_dst"), py::arg("idx_dst"), py::arg("P_dst") = py::none(),
        py::arg("dPb_dst") = py::none(), py::arg("heads") = 1);
  m.def("gat_act_bwd", &gat_act_bwd, py::arg("dH"), py::arg("Z"), py::arg("dPre"), py::arg("counters"),
        py::arg("n_hops"), py::arg("p") = 0.0, py::arg("seed") = 0, py::arg("layer") = 0,
        py::arg("step_dev") = py::none(), py::arg("bias_g") = py::none());
  m.def("gat_full_aggregate", &gat_full_aggregate, py::arg("graph"), py::arg("P"), py::arg("as_"), py::arg("ad"),
        py::arg("heads"), py::arg("r0"), py::arg("r1"), py::arg("acc") = py::none(), py::arg("first") = true,
        py::arg("last") = true, py::arg("bias") = py::none(), py::arg("act") = false, py::arg("Z") = py::none());
  m.def("hgt_full_attention", &hgt_full_attention, py::arg("graphs"), py::arg("qq"), py::arg("u"), py::arg("heads"),
        py::arg("r0"), py::arg("r1"), py::arg("kv"), py::arg("prior"));
  m.def("hgt_attention", &hgt_attention, py::arg("qq"), py::arg("u"), py::arg("heads"), py::arg("counters"),
        py::arg("n_hops_targets"), py::arg("kv"), py::arg("prior"), py::arg("ell"), py::arg("ks"), py::arg("deg"),
        py::arg("alpha"));
  m.def("hgt_attention_bwd", &hgt_attention_bwd, py::arg("du"), py::arg("qq"), py::arg("dqq"), py::arg("heads"),
        py::arg("counters"), py::arg("n_hops_targets"), py::arg("kv"), py::arg("prior"), py::arg("ell"), py::arg("ks"),
        py::arg("deg"), py::arg("alpha"), py::arg("dal"), py::arg("dkv"), py::arg("dprior"));
  m.def("hgt_gelu", &hgt_gelu, py::arg("X"), py::arg("Y"), py::arg("counters"), py::arg("n_hops"),
        py::arg("dY") = py::none());
  m.def("hgt_gate", &hgt_gate, py::arg("A"), py::arg("X"), py::arg("out"), py::arg("skip"), py::arg("counters"),
        py::arg("n_hops"), py::arg("dZ") = py::none(), py::arg("dX") = py::none(), py::arg("skip_g") = py::none());
  m.def("hgt_blocks", &hgt_blocks, py::arg("att"), py::arg("msg"), py::arg("att_img"), py::arg("msg_img"),
        py::arg("att_dense") = py::none(), py::arg("msg_dense") = py::none(), py::arg("att_g") = py::none(),
        py::arg("msg_g") = py::none());
  m.def("hgt_kqv_cast", &hgt_kqv_cast, py::arg("dkv"), py::arg("dq"), py::arg("out"), py::arg("bias_g"),
        py::arg("counters"), py::arg("idx"), py::arg("idx_q"));
  m.def("softmax_nll", &softmax_nll, py::arg("logits"), py::arg("C"), py::arg("y"), py::arg("labels_all"),
        py::arg("nodes"), py::arg("counters"), py::arg("loss"), py::arg("dlogits"), py::arg("correct"),
        py::arg("colsum"), py::arg("prezeroed") = false);
  m.def("sigmoid_bce", &sigmoid_bce, py::arg("logits"), py::arg("T"), py::arg("label_bits"), py::arg("nodes"),
        py::arg("counters"), py::arg("loss"), py::arg("dlogits"), py::arg("counts") = py::none(),
        py::arg("colsum") = py::none(), py::arg("prezeroed") = false);
  m.def("adam_step", &adam_step);
  m.def("colsum_bf16", &colsum_bf16);
  m.def("zero_rows", &zero_rows);
  m.def("sage_fused", &sage_fused, py::arg("feat"), py::arg("nodes"), py::arg("src_local"), py::arg("d"),
        py::arg("counters"), py::arg("n_hops_targets"), py::arg("ell"), py::arg("ks"), py::arg("deg"),
        py::arg("w_packed"), py::arg("bias"), py::arg("relu"), py::arg("z"), py::arg("a_save") = py::none());
  m.def("sage_fused_supported",
        [](int64_t d, int64_t n_out, const RowTableHandle* feat) {
          return sage_fused_supported(static_cast<int>(d), static_cast<int>(n_out), feat ? &feat->tbl : nullptr);
        },
        py::arg("d"), py::arg("n_out"), py::arg("feat") = py::none());
  py::class_<PeerBuffer, std::shared_ptr<PeerBuffer>>(m, "PeerBuffer")
      .def_static("allocate", &PeerBuffer::allocate)
      .def_static("open", &PeerBuffer::open)
      .def("handle", &PeerBuffer::handle)
      .def("as_tensor", &PeerBuffer::as_tensor)
      .def_readonly("bytes", &PeerBuffer::bytes)
      .def_readonly("device", &PeerBuffer::device)
      .def_readonly("imported", &PeerBuffer::imported);
  py::class_<PeerGroup>(m, "PeerGroup")
      .def(py::init<int, int, std::vector<Tensor>, std::vector<Tensor>>())
      .def("barrier", &PeerGroup::barrier)
      .def("adam", &PeerGroup::adam)
      .def_readonly("err", &PeerGroup::err)
      .def_readonly("epoch", &PeerGroup::epoch);
  py::class_<TcGemm>(m, "TcGemm")
      .def(py::init<int>())
      .def("add_forward", &TcGemm::add_forward)
      .def("add_dgrad", &TcGemm::add_dgrad)
      .def("add_wgrad", &TcGemm::add_wgrad)
      .def("run", &TcGemm::run);
  m.def("enable_peer_access", &enable_peer_access);
  m.def("multimem_copy", &multimem_copy);
  m.def("pack_weight", &pack_weight);
  m.def("pack_weight_into", &pack_weight_into);
}
