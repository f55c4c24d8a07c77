// Declarations of the CPU reference ops (see cpu_ops.cc).
#pragma once
#include <torch/extension.h>

#include <tuple>
#include <vector>

namespace glt {

using torch::Tensor;

std::tuple<Tensor, Tensor, Tensor, Tensor> coo_to_csr(
    const Tensor& rows, const Tensor& cols, const c10::optional<Tensor>& eids,
    const c10::optional<Tensor>& weights, int64_t num_rows, bool sort_cols);

std::tuple<Tensor, Tensor, Tensor> cpu_sample_neighbors(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& seeds, int64_t k, bool with_edge, bool replace, int64_t seed, int64_t stream);

std::tuple<Tensor, Tensor, Tensor> cpu_sample_neighbors_weighted(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& weights, const Tensor& seeds, int64_t k, bool with_edge, int64_t seed,
    int64_t stream, bool replace);

class CpuIdTable {
 public:
  explicit CpuIdTable(int64_t capacity_hint);
  void reset();
  Tensor insert(const Tensor& keys);        // local ids, new keys appended in first-seen order
  Tensor lookup(const Tensor& keys) const;  // -1 when absent
  Tensor keys(int64_t from) const;          // keys[from:]
  int64_t size() const { return (int64_t)keys_.size(); }
  int64_t insert_one(int64_t key);
  int64_t find_one(int64_t key) const;

 private:
  struct Slot { int64_t key; int32_t val; uint32_t gen; };
  void rehash(int64_t min_slots);
  std::vector<Slot> slots_;
  std::vector<int64_t> keys_;
  uint64_t mask_ = 0;
  uint32_t gen_ = 1;
};

std::tuple<Tensor, Tensor> cpu_negative_sample(
    const Tensor& indptr, const Tensor& indices, int64_t num_rows, int64_t num_cols, int64_t req,
    int64_t trials, bool padding, bool sorted, int64_t seed, int64_t stream);

std::tuple<Tensor, Tensor, Tensor, Tensor> cpu_node_subgraph(
    const Tensor& indptr, const Tensor& indices, const c10::optional<Tensor>& eids,
    const Tensor& srcs, bool with_edge);

Tensor cpu_random_walk(const Tensor& indptr, const Tensor& indices, const Tensor& starts,
                       int64_t walk_length, double p, double q, int64_t seed, int64_t stream);

std::tuple<Tensor, Tensor, Tensor> cpu_stitch(
    int64_t num_seeds, const std::vector<Tensor>& idx_list, const std::vector<Tensor>& nbrs_list,
    const std::vector<Tensor>& nbrs_num_list, const std::vector<Tensor>& eids_list);

// out[pos[i]] (or out[i]) = table[id2index[ids[i]] - 0] (or table[ids[i] - offset]); rows are copied as raw bytes by
// all intra-op threads.  Host tier of Feature / RPC feature callee / DistFeature stitch.
void cpu_gather_rows(const Tensor& table, const Tensor& ids, const c10::optional<Tensor>& id2index, int64_t offset,
                     Tensor out, const c10::optional<Tensor>& pos);

Tensor cpu_nbr_prob(const Tensor& indptr, const Tensor& indices, const Tensor& nbr_indptr,
                    const Tensor& last_prob, const Tensor& nbr_last_prob, int64_t k);

}  // namespace glt
