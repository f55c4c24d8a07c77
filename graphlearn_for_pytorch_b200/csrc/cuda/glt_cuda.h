// Host-visible declarations of the sm_90a kernels (torch-free: raw pointers and
// a cudaStream_t) so the .cu files compile in seconds and the binding layer is
// the only translation unit that sees torch headers.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../philox.h"

namespace glt {

constexpr int kMaxParts = 16;  // 8 GPUs of one NVSwitch box + optional host tiers

// One CSR shard of a range-partitioned graph.  Pointers may live in local HBM,
// in a peer GPU's HBM (mapped over NVLink via CUDA IPC) or in pinned host
// memory; the kernels dereference them directly -- this is the generalisation
// of the reference's pointer-table gather (csrc/cuda/unified_tensor.cu:35-81)
// to graph topology.
struct CsrShard {
  const int64_t* indptr;   // [row_end - row_begin + 1], shard-local offsets
  const void* indices;     // int32 or int64 global column ids
  const int64_t* eids;     // optional global edge ids
  const float* weights;    // optional edge weights
  int64_t row_begin;       // first global row id owned by this shard
  int64_t row_end;         // one past the last owned row
};

struct GraphTable {
  int num_parts;
  int idx_bytes;  // 4: int32 column ids, 8: int64
  CsrShard parts[kMaxParts];
};

// Range-partitioned row store (features / labels).  Part p holds rows
// [row_begin[p], row_begin[p+1]).
struct RowTable {
  int num_parts;
  int64_t row_bytes;
  const void* base[kMaxParts];
  int64_t row_begin[kMaxParts + 1];
};

// Device-resident id -> local-id hash table (open addressing, linear probe).
struct HashTable {
  int64_t* keys;   // capacity slots, empty = -1
  int32_t* vals;   // dense local id of the key in this slot
  int32_t* aux;    // first-occurrence index (ordered insert only)
  uint32_t mask;   // capacity - 1
};

// Per-batch device-side bookkeeping; the host never reads it on the hot path.
//   cum[h]      : number of local nodes after hop h-1 (cum[0] = 0, cum[1] = #seeds)
//   edges[h]    : number of sampled edges of hop h
struct BatchCounters {
  int32_t* cum;     // [max_hops + 2]
  int32_t* edges;   // [max_hops]
  int32_t* cursor;  // running number of local nodes
  int32_t* overflow;  // optional: neighbours dropped by the capacity guard (cumulative)
};

// ---- sampling.cu -----------------------------------------------------------
void launch_table_clear(HashTable t, cudaStream_t s);

// Ordered (first-occurrence) insertion of the seed ids.  Writes nodes[0..n0),
// seed_local[i] (local id of seeds[i]), cum[0]=0, cum[1]=n0, cursor=n0.
void launch_init_seeds(const int64_t* seeds, int n_seeds, const int32_t* n_seeds_dev,
                       HashTable t, int64_t* nodes, int32_t* seed_local, int32_t* scratch,
                       BatchCounters c, int32_t* step_dev, int step_inc, cudaStream_t s);

struct HopArgs {
  GraphTable g;
  HashTable t;
  BatchCounters c;
  int64_t* nodes;       // local -> global id, appended by this hop
  int32_t* ell;         // [cap_rows * k] slot ids -> local ids after relabel; -1 = empty
  int64_t* ell_eids;    // optional [cap_rows * k]
  int32_t* deg;         // [cap_nodes] sampled degree per target local id
  int hop;              // reads frontier [cum[hop], cum[hop+1])
  int k;                // fanout (>0)
  int cap_rows;         // worst-case frontier size
  int cap_nodes;        // node arena capacity (overflow guard)
  int cap_rows_next;    // capacity of the next hop's frontier
  int weighted;         // 1: exponential-race weighted sampling
  int replace;          // 1: with replacement
  uint64_t seed;
  uint32_t stream;
  const int32_t* stream_dev;  // optional device step counter mixed into the Philox stream
  // --- heterogeneous graphs: frontier and neighbours belong to different node types -----------------
  int64_t* nodes_out;         // id list of the NEIGHBOUR type (appended); nullptr = same list as `nodes`
  const int32_t* bound_ptr;   // precomputed id bound of the neighbour type for this hop (k_hetero_finalize);
                              // nullptr = derive it from c.cum / c.cursor (single node type)
  uint32_t stream_stride;     // Philox stream ids consumed per device step (0 = 8, the homogeneous arena)
};
void launch_sample_hop(const HopArgs& a, cudaStream_t s);
void launch_relabel_hop(const HopArgs& a, cudaStream_t s);
// deterministic local-id order of a hop's new nodes (see sampling.cu): keys -> (caller sorts tmp) -> assign
void launch_det_keys(const HopArgs& a, int64_t* tmp, cudaStream_t s);
void launch_det_assign(const HopArgs& a, const int64_t* sorted, cudaStream_t s);

// Heterogeneous sampling (native hetero inducer; reference csrc/cuda/inducer.cu:194-338 CUDAHeteroInducer +
// python/sampler/neighbor_sampler.py:232-317): one GROUPED launch per hop over all relations.  `descs` is a
// device array of `n_rel` HopArgs (blockIdx.y selects the relation; relations with k <= 0 are skipped);
// `max_k` / `max_rows` are the maxima over the relations (template / grid selection).
void launch_sample_hop_grouped(const HopArgs* descs, int n_rel, int max_k, int max_rows, cudaStream_t s);
void launch_relabel_hop_grouped(const HopArgs* descs, int n_rel, int max_k, int max_rows, cudaStream_t s);
struct HeteroTypeState {
  int32_t* cum;       // [6] of this node type
  int32_t* cursor;
  int cap_nodes;
  int cap_rows[5];    // frontier capacity per hop (+ trailing entry)
};
// cum[hop + 2] = cursor = min(cursor, cap_nodes, cum[hop + 1] + cap_rows[hop + 1]) for every node type
void launch_hetero_finalize(const HeteroTypeState* types, int n_types, int hop, cudaStream_t s);

// One-hop API sampler (NeighborOutput): fixed-stride output, no dedup.
void launch_sample_one_hop(GraphTable g, const int64_t* seeds, int n, int k, int weighted,
                           int replace, uint64_t seed, uint32_t stream, int64_t* out_nbrs,
                           int64_t* out_eids, int32_t* out_cnt, cudaStream_t s);
// Degrees of arbitrary rows (all-neighbour fanout sizing).
void launch_lookup_degree(GraphTable g, const int64_t* ids, int n, int64_t* out, cudaStream_t s);
// Full-neighbourhood copy: out[offs[i] .. offs[i+1]) = N(ids[i]).
void launch_copy_neighbors(GraphTable g, const int64_t* ids, int n, const int64_t* offs,
                           int64_t* out_nbrs, int64_t* out_eids, cudaStream_t s);

// ELL -> COO of one hop with exact offsets (exclusive scan of deg over the frontier).
void launch_ell_to_coo(const int32_t* ell, const int64_t* ell_eids, const int32_t* deg,
                       const int64_t* offs, const int32_t* cum, int hop, int k, int cap_rows,
                       int64_t* rows, int64_t* cols, int64_t* eids, cudaStream_t s);

// Generic table ops for the inducer API (unordered insert + lookup).
void launch_table_insert(HashTable t, const int64_t* keys, int64_t n, int64_t* nodes,
                         int32_t* cursor, int cap_nodes, int32_t* out_slots, cudaStream_t s);
void launch_table_resolve(HashTable t, int32_t* slots_inout, int64_t n, cudaStream_t s);
void launch_table_lookup(HashTable t, const int64_t* keys, int64_t n, int32_t* out, cudaStream_t s);

// ---- negative / subgraph / walk / prob (graph_ops.cu) ------------------------
void launch_negative_sample(GraphTable g, int64_t num_rows, int64_t num_cols, int req, int trials,
                            int padding, uint64_t seed, uint32_t stream, int64_t* out_rows,
                            int64_t* out_cols, int32_t* out_count, cudaStream_t s);
void launch_subgraph_count(GraphTable g, HashTable t, const int64_t* nodes, int n, int64_t* cnt,
                           cudaStream_t s);
void launch_subgraph_fill(GraphTable g, HashTable t, const int64_t* nodes, int n,
                          const int64_t* offs, int64_t* rows, int64_t* cols, int64_t* eids,
                          cudaStream_t s);
// uniform steps when !biased, otherwise node2vec's second-order rule with weights w (philox.h)
void launch_random_walk(GraphTable g, const int64_t* starts, int n, int walk_len, bool biased, Node2VecWeights w,
                        uint64_t seed, uint32_t stream, int64_t* out, cudaStream_t s);
void launch_nbr_prob(GraphTable g, GraphTable nbr_g, const float* last, const float* nbr_last,
                     int64_t n, int64_t n_nbr, int k, float* cur, cudaStream_t s);

// ---- gather.cu ---------------------------------------------------------------
// out[i, :] = table[idx[i]] (idx optionally remapped through id2index); rows
// with idx < 0 or i >= *n_dev (when n_dev != nullptr) are zero-filled.
// id2index_len > 0: ids outside [0, id2index_len) produce zero rows instead of an out-of-bounds read
void launch_gather_rows(RowTable t, const int64_t* idx, const int64_t* id2index, int64_t n,
                        const int32_t* n_dev, void* out, int64_t out_row_bytes, cudaStream_t s,
                        int64_t id2index_len = 0);
// copy `nbytes` (multiple of 16) from local memory to an NVSwitch multicast address
void launch_multimem_copy(const void* src, void* mc_dst, int64_t nbytes, cudaStream_t s);
// out[i, 0..d) (bf16) = dequantised MXFP8 row idx[i] of `t` (see data/quantize.py), d a multiple of 128
void launch_gather_mxfp8(RowTable t, const int64_t* idx, int64_t n, int d, void* out, cudaStream_t s);
// launch_gather_rows for MXFP8 rows of any d that is a multiple of 32 up to 1024: the same idx / id2index / n_dev
// contract, de-quantised into bf16 rows of pitch out_row_bytes (a multiple of 16; `out` 16-byte aligned)
void launch_gather_mxfp8_rows(RowTable t, const int64_t* idx, const int64_t* id2index, int64_t n, const int32_t* n_dev,
                              int d, void* out, int64_t out_row_bytes, cudaStream_t s, int64_t id2index_len = 0);

// ---- sage.cu (GraphSAGE engine kernels) ---------------------------------------
struct SageAggArgs {
  // source rows: either a RowTable indexed by global id (layer 1) or a dense
  // local matrix (deeper layers, src_local != nullptr).
  RowTable feat;
  const int64_t* nodes;         // local -> global id (layer 1)
  const void* src_local;        // bf16 [n_src, d] (deeper layers)
  int d;                        // feature width (elements, multiple of 8)
  const int32_t* cum;           // device node counts
  int n_hops_targets;           // targets = cum[n_hops_targets]
  int cap_targets;
  // ELL blocks per hop (targets of hop h use ell[h] with stride k[h])
  const int32_t* ell[4];
  int k[4];
  const int32_t* deg;
  void* out;                    // bf16 [cap_targets, 2d] = [mean | self]
  // column-block output (heterogeneous layers: A_t = [mean_rel1 | mean_rel2 | ... | self]); out_ld == 0 keeps
  // the homogeneous layout above (out_ld = 2d, mean_col = 0, self_col = d)
  int out_ld;                   // row pitch of `out` in elements
  int mean_col;                 // first column of this relation's mean block
  int self_col;                 // first column of the self block, -1 = do not write it
  int feat_fp8;                 // 1: `feat` rows are MXFP8 (data/quantize.py), d a multiple of 32; src_local is always bf16
};
void launch_sage_aggregate(const SageAggArgs& a, cudaStream_t s);

// ---- sage_infer.cu (exact layer-wise inference over the full CSR) ---------------
// For every global row r in [r0, r1) the mean over ALL of r's CSR neighbours (multi-edges counted with their
// multiplicity, degree 0 -> 0), accumulated in fp32 in a fixed order and rounded once:
//   concat  (combine = 0): out[r - r0] = bf16([mean_u x_u | x_r])                       (out width >= 2d)
//   combine (combine = 1): out[r - r0] = bf16(act(mean_u src[u, src_col:] + src[r, self_col:] + bias))
//   mean only (combine = 0, mean_only = 1): out[r - r0, :d] = bf16(mean_u x_u), nothing else is written (one relation's
//                                           column block of a heterogeneous layer's wider A operand)
// Sources: the dense bf16 table `src` (row u at src + u * src_ld, ids outside [0, n_src) read as zero rows), or,
// when src == nullptr, the feature table `feat` (bf16 rows of d elements, or MXFP8 rows with feat_fp8 = 1, d a multiple
// of 32).
struct SageFullAggArgs {
  GraphTable g;
  RowTable feat;
  int feat_fp8;
  const void* src;              // bf16 [n_src, src_ld] indexed by global id, or nullptr
  int64_t n_src, src_ld;
  int src_col;                  // first column of the neighbour block in src
  int self_col;                 // first column of the self block in src
  int d;                        // width of the aggregated block (multiple of 8, <= 1024)
  int64_t r0, r1;
  int combine;
  const void* bias;             // combine: bf16 [d] or nullptr
  int relu;                     // combine: ReLU after the bias
  void* out;                    // bf16 [r1 - r0, out_ld]
  int64_t out_ld;
  int mean_only;                // concat without the self block
};
void launch_sage_full_aggregate(const SageFullAggArgs& a, cudaStream_t s);

// ---- label_prop.cu (label propagation / Correct & Smooth over the full CSR) ------
// One iteration over every row i of [0, n) (row i lists the nodes whose values flow into i; multi-edges count with
// their multiplicity):
//   out_i = alpha * s_i * sum_{j in row(i)} t_j x_j + beta * base_i, clamped to [lo, hi]; out_i = base_i where fixed[i]
// x, base, out: fp32 [n, cp], cp a multiple of 4 in [4, 512], 16-byte aligned; columns >= c of out are written as 0.
// Columns outside [0, n) read as zero rows.  t == nullptr: t_j = 1.
struct LabelPropArgs {
  GraphTable g;
  int64_t n;
  int c, cp;
  const float* x;
  const float* base;
  const float* s;               // [n]
  const float* t;               // [n] or nullptr
  float alpha, beta;
  float lo, hi;
  const uint8_t* fixed;         // bool [n] or nullptr
  float* out;
  int64_t r0, r1;               // set by launch_label_prop: all rows [0, n)
};
void launch_label_prop(const LabelPropArgs& a, cudaStream_t s);
// The per-row factors from row lengths: s = t = deg^-1/2 (sym), or s = 1 / deg (row; t not written); 0 where deg = 0.
void launch_label_prop_factors(const GraphTable& g, int64_t n, bool sym, float* s, float* t, cudaStream_t st);

// dH[s, :] += dA[t, mean_col : mean_col + d] / deg[t] for every sampled edge t <- s of the targets t < cum[n_hops]
// (the mean block of one relation of a heterogeneous layer; its self block is added by launch_add_block_f32)
struct SageScatterArgs {
  const void* dA;               // bf16 [cap_targets, dA_ld]
  int d;
  const int32_t* cum;
  int n_hops_targets;
  int cap_targets;
  const int32_t* ell[4];
  int k[4];
  const int32_t* deg;
  float* dH;                    // fp32 [cap_src, d]
  int dA_ld, mean_col;          // row pitch of dA and first column of the mean block (elements)
};
void launch_sage_scatter_bwd(const SageScatterArgs& a, cudaStream_t s);
// dH[t, :] += dA[t, col : col + d] for t < cum[n_hops] (self block of a heterogeneous layer)
void launch_add_block_f32(const void* dA, int dA_ld, int col, int d, const int32_t* cum, int n_hops, int cap,
                          float* dH, cudaStream_t s);

// ---- transpose.cu: per-batch transposed adjacency + atomics-free backward ----------
// The forward ELL blocks are keyed by TARGET (row t lists its sampled sources).  The backward of the
// mean aggregation needs the opposite view (for a source s: all targets that sampled it).  It is
// built once per batch on the sampling stream as a CSR over local source ids, ordered by hop inside
// every segment, so that one structure serves every layer (layer l uses the hops 0..L-l prefix).
struct TransposeArgs {
  const int32_t* cum;        // device counters (cum[h] = nodes before hop h's new nodes)
  const int32_t* deg;        // [cap_nodes] valid ELL entries per target
  const int32_t* ell[4];
  int k[4];
  int cap_rows[4];
  int n_hops;                // hops 0..n_hops-1 are transposed
  int cap_nodes;             // capacity of the local id space
  int cap_edges;             // capacity of tgt
  int32_t* cnt;              // [n_hops][cap_nodes]: in-counts per hop, then cumulative over hops
  int32_t* off;              // [cap_nodes + 1]: segment start per source
  int32_t* cursor;           // [n_hops][cap_nodes]: fill cursor per hop
  int32_t* tgt;              // [cap_edges]: target local ids
  int32_t* block_sums;       // [>= cap_nodes / 1024 + 2]
  int32_t* meta;             // [cap_nodes][4] = {segment start, first in-neighbour, second in-neighbour, total in-edges}
  float* meta_inv;           // [cap_nodes][2] = 1/deg of those two (the backward gather reads one record per source
                             // instead of walking off -> tgt -> deg)
};
void launch_build_transpose(const TransposeArgs& a, cudaStream_t s);

struct SageGatherBwdArgs {
  const void* dA;            // bf16 [cap_targets, 2d] = gradient of [mean | self]
  int d;
  const int32_t* cum;
  int n_hops_targets;        // targets = cum[n_hops_targets], sources = cum[n_hops_targets + 1]
  int cap_targets;
  int cap_src;               // rows of dPre / Z
  const int32_t* deg;
  const int32_t* off;        // transposed CSR
  const int32_t* cnt_upto;   // [cap_nodes] in-edges of the hops used by this layer (prefix of the segment)
  const int32_t* tgt;
  const int32_t* meta;       // TransposeArgs::meta / meta_inv
  const float* meta_inv;
  const void* Z;             // bf16 [cap_src, d] activations of the previous layer (ReLU mask) or nullptr
  void* dPre;                // bf16 [cap_src, d]
  float* colsum;             // optional fp32 [d]: bias gradient (16-byte aligned: accumulated with red.v4)
  int colsum_prezeroed;      // the caller already zeroed colsum (no memset node in the launch chain)
  float gscale;              // 1/(1-p) when Z is a post-dropout activation, else 1
};
// dPre[s] = relu'(Z[s]) * (dA_self[s] + sum_{t in in(s)} dA_mean[t] / deg[t]); rows >= sources are zero-filled.
void launch_sage_gather_bwd(const SageGatherBwdArgs& a, cudaStream_t s);

// dPre = (Z > 0) ? bf16(dH) : 0 for rows < cum[n_hops]; 0 beyond.  relu = false: dPre = bf16(dH), Z is not read.
// colsum (optional, fp32 [d]): bias gradient = column sums of the bf16 dPre, any d (multiple of 8): fused into the
// cast when d divides 2048, a second column-sum kernel otherwise.
void launch_relu_bwd_cast(const float* dH, const void* Z, const int32_t* cum, int n_hops, int cap,
                          int d, void* dPre, float* colsum, cudaStream_t s, bool prezeroed = false,
                          float gscale = 1.f, bool relu = true);
// In-place inverted dropout (keep prob 1-p, kept values scaled by 1/(1-p)) on rows < cum[n_hops] of bf16 Z[cap, d];
// mask = Philox(seed, layer, *step_dev, element).  Backward: launch_relu_bwd_cast(..., gscale = 1/(1-p)) on the
// post-dropout Z.
void launch_dropout_bf16(void* Z, const int32_t* cum, int n_hops, int cap, int d, float p, uint64_t seed, int layer,
                         const int32_t* step_dev, cudaStream_t s);
// g[0..n) = 0, *loss = 0, *correct = 0 (one launch at the start of the gradient phase; the *_prezeroed variants of
// the kernels below then skip their own memsets, which keeps the step a pure kernel chain)
void launch_zero_grads(float* g, int64_t n, float* loss, int32_t* correct, cudaStream_t s);
// loss = mean NLL(log_softmax(logits[:n0, :C]), y); dlogits = (softmax - onehot)/n0
// labels come from y[r], or (labels_all != nullptr) from labels_all[nodes[r]].
// colsum (optional, fp32 [ld]): bias gradient = column sums of the bf16 dlogits, any ld (multiple of 8): fused into
// the loss kernel for ld <= 256, a second column-sum kernel otherwise.
void launch_softmax_nll(const void* logits, int ld, int C, const int64_t* y, const int64_t* labels_all,
                        const int64_t* nodes, const int32_t* cum, int cap, float* loss, void* dlogits,
                        int32_t* correct, float* colsum, cudaStream_t s, bool prezeroed = false);
// out[c] = sum over valid rows of X[:, c]  (d multiple of 8)
void launch_colsum_bf16(const void* X, const int32_t* cum, int n_hops, int cap, int d, float* out,
                        cudaStream_t s);
// launch_colsum_bf16 without the memset: accumulates onto `out`
void launch_colsum_accum(const void* X, const int32_t* cum, int n_hops, int cap, int d, float* out,
                         cudaStream_t s);
void launch_zero_rows(float* p, const int32_t* cum, int n_hops, int cap, int d, cudaStream_t s);
// flat fp32 Adam over [n] with bf16 shadow copy refresh.
void launch_adam(float* p, const float* g, float* m, float* v, void* p_bf16, int64_t n, float lr,
                 float b1, float b2, float eps, float wd, int32_t* step_dev, float gscale,
                 cudaStream_t s);

// ---- multilabel.cu (multi-label node classification loss) --------------------------------------------------------
// loss = mean over rows r < n0 = min(cum[1], cap) and tasks c < T of BCE-with-logits(logits[r, c], y[r, c]), with
// y[r, c] = bit c & 31 of bits[nodes[r] * W + (c >> 5)], W = ceil(T / 32) (an id outside [0, n_nodes): all zeros);
// dlogits = (sigmoid - y) / (n0 T), zero in columns [T, ld) and rows [n0, cap).  counts (optional, int32 [3]) +=
// (TP, FP, FN) at logit 0.  colsum (optional, fp32 [ld]): bias gradient = column sums of the bf16 dlogits, fused for
// ld <= 256, a second column-sum kernel otherwise.  prezeroed: loss, counts and colsum were zeroed by the caller.
void launch_sigmoid_bce(const void* logits, int ld, int T, const uint32_t* bits, int64_t n_nodes,
                        const int64_t* nodes, const int32_t* cum, int cap, float* loss, void* dlogits,
                        int32_t* counts, float* colsum, cudaStream_t s, bool prezeroed = false);

// ---- link.cu (link-prediction step: in-graph negatives + fused edge loss) --------
// pos: int64 [2, B] positive pairs (-1 = padding).  Writes seeds [2P], P = (1 + k) B: seeds[p] = source and
// seeds[P + p] = destination of pair p; pairs [0, B) are pos, pair B + i k + j is the j-th negative of positive i,
// uniform over [0, num_nodes)^2 and redrawn (up to 5 draws) while it is an edge of g, keyed by Philox
// (seed, a stream no sampling kernel uses, *step_dev, p).  *n_pairs = (1 + k) x #valid positives.
void launch_link_seeds(GraphTable g, const int64_t* pos, int B, int k, int64_t num_nodes, uint64_t seed,
                       const int32_t* step_dev, int64_t* seeds, int32_t* n_pairs, cudaStream_t s);
// Mean BCE-with-logits over the pairs p < P with seed_local[p], seed_local[P + p] >= 0: logit = dot of the first C
// columns of those rows of Z (bf16 [rows, ld]), label = (p < B).  Adds into *loss / *correct (pre-zeroed) and, when
// dZ (fp32 [rows, ld], pre-zeroed) is given, the logit gradients of both endpoints with fp32 red.add.
void launch_link_bce(const void* Z, int ld, int C, const int32_t* seed_local, int P, int B, const int32_t* n_pairs,
                     float* loss, int32_t* correct, float* dZ, cudaStream_t s);

// ---- skipgram.cu (metapath2vec / DeepWalk skip-gram step) ---------------------------------------------------------
constexpr int kMaxMetaPath = 8;
// Node type of each walk position slot: slot 0 = source type of metapath[0], slot r + 1 = destination type of
// metapath[r]; position p > 0 has slot (p - 1) % R + 1.  off = first row of the type in the concatenated embedding
// table, n = node count of the type.
struct MetaPathTypes {
  int64_t off[kMaxMetaPath + 1];
  int64_t n[kMaxMetaPath + 1];
};
// state = [next walk step, Adam step, walk step of the current step]: [2] = [0]; [0] += 1; [1] += 1.
void launch_m2v_begin(int32_t* state, cudaStream_t s);
// rel: device array of R GraphTables (CSR rows = source ids).  out: int64 [n_walks, L + 1]; walk i starts at
// starts[i / W] and ends (-1 tail) at a dead end or an id outside its type.  *n_valid = #windows of C valid entries.
void launch_metapath_walk(const GraphTable* rel, int R, MetaPathTypes types, const int64_t* starts, int n_walks, int W,
                          int L, int C, uint64_t seed, const int32_t* step_dev, int64_t* out, int32_t* n_valid,
                          cudaStream_t s);
// node2vec's second-order walk over one relation from a type to itself (column-sorted CSR rows): the same output and
// dead-end contract as launch_metapath_walk.  w_ret / w_in / w_out are the unnormalised weights 1/p, 1 and 1/q divided
// by their maximum; L <= kNode2VecMaxWalk keeps the draw counters from wrapping.
constexpr int kNode2VecMaxWalk = 1 << 20;
void launch_node2vec_walk(const GraphTable* rel, MetaPathTypes types, const int64_t* starts, int n_walks, int W, int L,
                          int C, float w_ret, float w_in, float w_out, uint64_t seed, const int32_t* step_dev,
                          int64_t* out, int32_t* n_valid, cudaStream_t s);
// neg: int64 [n_walks * (L + 2 - C) * K, C]; K negative windows per window of the walks (all -1 for an invalid one).
void launch_sgns_negatives(const int64_t* walks, int n_walks, int L, int C, int K, int R, MetaPathTypes types,
                           uint64_t seed, const int32_t* step_dev, int64_t* neg, cudaStream_t s);
// SGNS loss (written to *loss) and its gradient red.added into grad (fp32 [rows, D], D % 8 == 0, D <= 512); sets
// touched[row] for every row looked up.
void launch_sgns_loss_grad(const int64_t* walks, const int64_t* neg, int n_walks, int L, int C, int K, int R,
                           MetaPathTypes types, const float* emb, int D, const int32_t* n_valid, float* grad,
                           uint8_t* touched, float* loss, cudaStream_t s);
// torch.optim.SparseAdam step *t_dev on the touched rows of w / m / v, then clears their grad rows and flags.
void launch_sparse_adam(float* w, float* grad, float* m, float* v, uint8_t* touched, int64_t rows, int D,
                        const int32_t* t_dev, float lr, float b1, float b2, float eps, cudaStream_t s);

// ---- seal.cu (SEAL link prediction: per-link enclosing subgraph, DRNL and DGCNN, CTA per link) ------------------------
constexpr int kSealMaxHops = 4;
constexpr int kSealMaxLayers = 8;    // GCNConv(hidden) layers; one GCNConv(1) follows them
constexpr int kSealMaxNodes = 1024;  // per-link node capacity (local ids fit int16)
constexpr int kSealMeta = 5;         // per link: [nodes, edges kept, valid, truncated, edges before truncation]

// Per-link arena, [B, ...] with per-link strides max_nodes / max_edges.  CSRs are local: sptr / scol by source,
// dptr / dcol by destination, both with the target pair removed.  X holds the concatenated tanh outputs of the GCN
// layers ([max_nodes, total]), XW a [max_nodes, hidden] scratch, G the gradient of X.  C1 is ReLU(conv1) [16, k],
// flat ReLU(conv2) [dense], H1 ReLU(lin1) [128] before dropout, mask the dropout scale [128], sel the sort-pool
// rows [k] (-1 = zero padding).
struct SealArenaPtrs {
  int B, max_nodes, max_edges;
  int64_t* nodes; int32_t* z; int32_t* meta;
  int32_t* sptr; int16_t* scol; int32_t* dptr; int16_t* dcol;
  float* X; float* XW; float* G; float* C1; float* flat; float* H1; float* mask; int32_t* sel;
  float* logits; float* lossv; float* dlogit;
};

// Offsets of the DGCNN's tensors in the flat fp32 parameter vector.  GCN layer l < L is [hidden, in] (in = Z for
// l = 0, hidden after), layer L is [1, hidden]; total = hidden * L + 1, dense = (k / 2 - 4) * 32.
struct SealModel {
  int H, L, Z, total, k, dense;
  int64_t w[kSealMaxLayers + 1], bias[kSealMaxLayers + 1];
  int64_t c1w, c1b, c2w, c2b, l1w, l1b, l2w, l2b, P;
};

struct SealExtractArgs {
  GraphTable g;
  const int64_t* links;        // [2, B]
  int64_t num_nodes;
  int hops, cap_max;           // cap_max = max(caps) (0: every hop takes full rows)
  int caps[kSealMaxHops];      // caps[h] <= 0: full rows at hop h
  uint64_t seed;
  const int32_t* step;         // Philox step key of the neighbour draws
  int max_z;                   // < 0: no clamp
  int32_t* samp;               // [B, max_nodes, cap_max] scratch of the drawn row positions (cap_max > 0)
  int32_t* truncated;          // += links that hit a capacity
};

size_t seal_extract_smem(int max_nodes);
size_t seal_forward_smem(const SealModel& m, int max_nodes);
size_t seal_backward_smem(const SealModel& m, int max_nodes);
// Enclosing subgraphs, local CSRs and DRNL labels of the B links (CTA per link).
void launch_seal_extract(const SealExtractArgs& e, const SealArenaPtrs& a, cudaStream_t s);
// GCN stack, sort-pool, convs, MLP and BCE (CTA per link).  Loss terms and dlogit are divided by the batch's valid
// links; training = 0 uses no dropout (mask = 1).
void launch_seal_forward(const SealModel& m, const SealArenaPtrs& a, const float* prm, const float* labels,
                         int training, float p_drop, uint64_t seed, const int32_t* step, cudaStream_t s);
// Gradient of the link's loss term into partials[b, :P] (CTA per link; invalid links write nothing).
void launch_seal_backward(const SealModel& m, const SealArenaPtrs& a, const float* prm, float* partials, cudaStream_t s);
// grad[i] = sum over valid links b, in order, of partials[b, i]; *loss = sum of the valid links' loss terms.
void launch_seal_reduce(const SealModel& m, const SealArenaPtrs& a, const float* partials, float* grad, float* loss,
                        cudaStream_t s);

// ---- gat.cu (relational GAT engine kernels; H = heads * C, H a multiple of 64 in [64, 1024], C % 8 == 0) -----------
// Per-node attention scores of two row sets: out[set][row * heads + h] = <att[set][h], P[set][row, h*C : (h+1)*C]>
// for row < min(cum[set][idx[set]], cap[set]).  P[1] == nullptr skips the second set.  zero (optional, fp32
// [cap[0], heads]) is cleared on the valid rows of set 0.
struct GatScoreArgs {
  const void* P[2];             // bf16 [cap, H]
  const void* att[2];           // bf16 [H]
  float* out[2];                // fp32 [cap, heads]
  const int32_t* cum[2];
  int idx[2], cap[2];
  float* zero;
  int H, heads;
};
void launch_gat_scores(const GatScoreArgs& a, cudaStream_t s);

// Attention aggregation of one relation over its per-hop ELL blocks (targets t < min(cum[n_hops_targets],
// cap_targets)).  alpha[h]: fp32 [rows of hop h, k[h], heads] softmax weights, sign bit = (score <= 0).  Output:
// first/last select write / accumulate into acc (fp32 [cap, H]) / finish: Z = bf16(act(acc + out + sum_b bias[b])),
// act = inverted dropout(leaky_relu(., 0.01)) with the Philox key of launch_dropout_bf16 (thresh16 = 0: no dropout).
struct GatAggArgs {
  const void* P;                // bf16 [n_src, H] source projections
  const float* as;              // fp32 [n_src, heads]
  const float* ad;              // fp32 [cap_targets, heads]
  int H, heads;
  const int32_t* cum;
  int n_hops_targets, cap_targets;
  const int32_t* ell[4];
  int k[4];
  const int32_t* deg;
  float* alpha[4];
  float* acc;
  int first, last;
  const void* bias;             // bf16 [n_bias, H]
  int n_bias;
  int act;
  uint32_t thresh16;
  float dscale;
  uint64_t seed;
  int layer;
  const int32_t* step_dev;
  void* z;                      // bf16 [cap_targets, H]
};
void launch_gat_aggregate(const GatAggArgs& a, cudaStream_t s);

// Backward of the attention aggregation given G (bf16 [cap_targets, H]): dP += alpha G (fp32 red.add into source
// rows), da_src[s, h] += dscore (atomics), da_dst[t, h] = sum_j dscore; dal (alpha's layout) is scratch.
struct GatBwdArgs {
  const void* G;
  const void* P;
  int H, heads;
  const int32_t* cum;
  int n_hops_targets, cap_targets;
  const int32_t* ell[4];
  int k[4];
  const int32_t* deg;
  const float* alpha[4];
  float* dal[4];
  float* dP;                    // fp32 [n_src, H]
  float* da_src;                // fp32 [n_src, heads]
  float* da_dst;                // fp32 [cap_targets, heads]
};
void launch_gat_backward(const GatBwdArgs& a, cudaStream_t s);

// Projection gradients of one relation (see gat.cu): seg[0] = source rows (dP != nullptr: adds and re-zeroes the
// fp32 rows of k_gat_backward), seg[1] = separate destination rows (P == nullptr: none).  Term 0 is always present;
// term 1 (da1 != nullptr) folds the destination scores into the source rows when both ends share the projection.
struct GatScoreBwdArgs {
  struct Seg {
    const void* P;              // bf16 [cap, H] projection
    float* dP;                  // fp32 [cap, H] or nullptr
    const float* da0;           // fp32 [cap, heads]
    const void* att0;           // bf16 [H]
    float* gatt0;               // fp32 [H] gradient of att0 (accumulated)
    const float* da1;
    const void* att1;
    float* gatt1;
    const int32_t* cum1;        // rows carrying term 1: min(cum1[idx1], rows)
    int idx1;
    void* dPb;                  // bf16 [cap, H] output
    const int32_t* cum;
    int idx, cap;
  } seg[2];
  int H, heads;
};
void launch_gat_score_bwd(const GatScoreBwdArgs& a, cudaStream_t s);

// Activation backward of a GAT layer output Z (bf16 [cap, d]) and the column sums of its gradient into n_bias bias
// gradient slots (bias_g fp32 [n_bias, d], accumulated).  dH == nullptr: dPre is an input (no activation).
struct GatActBwdArgs {
  const float* dH;
  const void* Z;
  void* dPre;
  const int32_t* cum;
  int n_hops, cap, d;
  float slope;
  uint32_t thresh16;
  float dscale;
  uint64_t seed;
  int layer;
  const int32_t* step_dev;
  float* bias_g;
  int n_bias;
};
void launch_gat_act_bwd(const GatActBwdArgs& a, cudaStream_t s);

// ---- hgt.cu (HGT engine kernels; H = heads * D, H a multiple of 64 in [64, 1024], D % 8 == 0) ----------------------
// Cross-relation attention of one (layer, destination type) over its n_rel <= kHgtMaxRel incoming relations, targets
// t < min(cum[n_hops_targets], cap_targets).  Source rows are bf16 [n_src, kv_ld] with K at column 0 and V at column
// v_off.  s = <qq_r[t, h], k_j,h> prior_r[h] scale; alpha (fp32 [rows of hop h, k[h], heads] per relation) is the
// softmax over the slots of every relation; u_r[t] = sum_j alpha v_j (bf16 [cap_targets, n_rel * H]).
constexpr int kHgtMaxRel = 8;
struct HgtAttnArgs {
  const void* qq;               // bf16 [cap_targets, n_rel * H]
  void* u;                      // bf16 [cap_targets, n_rel * H]
  int H, heads, n_rel, kv_ld, v_off;
  float scale;                  // 1 / sqrt(D)
  const int32_t* cum;
  int n_hops_targets, cap_targets;
  struct Rel {
    const void* kv;
    const float* prior;         // fp32 [heads]
    const int32_t* deg;
    const int32_t* ell[4];
    int k[4];
    float* alpha[4];
  } rel[kHgtMaxRel];
};
void launch_hgt_attention(const HgtAttnArgs& a, cudaStream_t s);

// Backward of launch_hgt_attention given dU (bf16 [cap_targets, n_rel * H]): dqq (bf16, rows [T, round_up(T, 128))
// zeroed), dK / dV added with red.add into fp32 rows dkv [n_src, 2H] = [dK | dV], dprior [heads] accumulated (one
// atomic per (relation, head) per CTA); dal (two floats per alpha entry) is scratch.
struct HgtAttnBwdArgs {
  const void* du;
  const void* qq;
  void* dqq;
  int H, heads, n_rel, kv_ld, v_off;
  float scale;
  const int32_t* cum;
  int n_hops_targets, cap_targets;
  struct Rel {
    const void* kv;
    const float* prior;
    const int32_t* deg;
    const int32_t* ell[4];
    int k[4];
    const float* alpha[4];
    float* dal[4];
    float* dkv;
    float* dprior;
  } rel[kHgtMaxRel];
};
void launch_hgt_attention_bwd(const HgtAttnBwdArgs& a, cudaStream_t s);

// dY == nullptr: Y = gelu(X) (exact erf) on rows < T.  dY given: Y = bf16(dY gelu'(X)), rows [T, round_up(T, 128)) = 0.
void launch_hgt_gelu(const void* X, void* Y, const int32_t* cum, int n_hops, int cap, int d, const void* dY,
                     cudaStream_t s);

// Gated skip connection (see hgt.cu): forward out = sigmoid(skip) A + (1 - sigmoid(skip)) X; backward (dZ32 or dZ16)
// out = dA, dX += (1 - sigmoid(skip)) dZ, skip_g += sum dZ (A - X) sigmoid'(skip).
struct HgtGateArgs {
  const void* A;                // bf16 [cap, d]
  const void* X;                // bf16 [cap, d]
  void* out;                    // bf16 [cap, d]
  const float* skip;            // fp32 scalar
  const float* dZ32;
  const void* dZ16;
  float* dX;                    // fp32 [cap, d] or nullptr
  float* skip_g;
  const int32_t* cum;
  int n_hops, cap, d;
};
void launch_hgt_gate(const HgtGateArgs& a, cudaStream_t s);

// Block-diagonal relation images (att_g == nullptr) or the inverse map of their dense fp32 gradients (see hgt.cu).
struct HgtBlockArgs {
  const void* att;              // bf16 [n_rel, heads, D, D]
  const void* msg;
  void* att_img;                // bf16 [n_rel * H, H]
  void* msg_img;                // bf16 [H, n_rel * H]
  float* att_dense;             // fp32 [n_rel * H, H]
  float* msg_dense;             // fp32 [H, n_rel * H]
  float* att_g;                 // fp32 [n_rel, heads, D, D]
  float* msg_g;
  int n_rel, heads, D;
};
void launch_hgt_blocks(const HgtBlockArgs& a, cudaStream_t s);

// bf16 [cap, 3H] = [dK | dQ | dV] from fp32 dkv [cap, 2H] (rows < min(cum[idx], cap), re-zeroed) and bf16 dq [., H]
// (rows < cum[idx_q]; nullptr: none); bias_g [3H] accumulates the column sums.
struct HgtKqvCastArgs {
  float* dkv;
  const void* dq;
  void* out;
  float* bias_g;
  const int32_t* cum;
  int idx, idx_q, cap, H;
  int cap_q;                 // rows of dq: nq is clamped to it like every extent read from a counter
};
void launch_hgt_kqv_cast(const HgtKqvCastArgs& a, cudaStream_t s);

// ---- peer.cu (collectives over NVLink peer memory, CUDA-graph capturable) ------
struct PeerPtrs {
  int world, rank;
  const float* g[kMaxParts];   // gradient buffer of every rank, mapped on this device
  int32_t* flags[kMaxParts];   // barrier flag array [2 * world] of every rank, mapped on this device
};
void launch_peer_barrier(const PeerPtrs& p, int which, int32_t* epoch_dev, int32_t* err, cudaStream_t s);
void launch_adam_peer(const PeerPtrs& p, float* param, float* m, float* v, void* p_bf16, int64_t n, float lr,
                      float b1, float b2, float eps, float wd, int32_t* step_dev, float gscale,
                      cudaStream_t s, const int32_t* err = nullptr);

// ---- sage_tc.cu (wgmma fused gather+aggregate+GEMM) ---------------------------
struct SageFusedArgs {
  SageAggArgs agg;              // agg.out may be nullptr (A tile is not materialised)
  const void* w_packed;         // bf16, wgmma SWIZZLE_128B K-major image, [K/64][N][64]
  const void* bias;             // bf16 [N]
  int n_out;                    // N (multiple of 16, <= 256)
  int relu;
  void* z;                      // bf16 [cap_targets, N]
  void* a_save;                 // optional bf16 [cap_targets, 2d] for backward
  int feat_fp8;                 // 1: agg.feat rows are MXFP8 (d e4m3 bytes + d/32 UE8M0 scales, 16-byte padded)
};
// 1 if the fused kernel takes layer width d -> n_out (its shared memory fits) and, when `feat` is given, can address
// every row of that feature table with its 32-bit row handles (4-bit part, 28-bit row inside the part).
int sage_fused_supported(int d, int n_out, const RowTable* feat = nullptr);
void launch_sage_fused(const SageFusedArgs& a, int num_sms, cudaStream_t s);
// W [N, K] row-major bf16 -> packed swizzled image used by launch_sage_fused.
void launch_pack_weight(const void* w, int n, int k, void* packed, cudaStream_t s);


// ---- tc_gemm.cu (TMA-fed wgmma GEMMs: forward layers 2..L, dA, split-K dW) ------------------------
struct TcProblem {
  int a_mn, b_mn;          // operand major-ness: 0 = K-major (row-major [rows, K]), 1 = MN-major ([K rows, M/N cols])
  int epi;                 // 0: bf16 out (+bias, +ReLU) through a TMA store; 1: fp32 red-add (split-K)
  int bn;                  // tile width: 64 / 128 / 256, divides n
  int m, n, k;             // static extents (capacity for the dynamic one)
  const int32_t* dyn;      // device counters; the dynamic extent is min(dyn[dyn_idx], dyn_cap)
  int dyn_idx, dyn_cap;
  int dyn_is_k;            // 0: the dynamic extent is M (forward / dA); 1: it is K (dW)
  const void* bias;        // bf16 [n] or nullptr (epi 0)
  int relu;
  float* out32;            // epi 1: fp32 [m_valid, ld32]
  int ld32, m_valid;
};
struct TcGemmArgs {
  int n_prob;
  TcProblem p[2];
  // {next item, CTAs done}, zero between launches: CTAs claim work items with atomicAdd on [0]; the last CTA to
  // finish zeroes both, so the next launch (or CUDA-graph replay) starts from item 0.  One buffer per plan, and a
  // plan is never launched concurrently with itself.
  int* tickets;
};
struct alignas(64) TcGemmLaunch {
  unsigned char maps[6][128];   // CUtensorMap A0, B0, C0, A1, B1, C1
  TcGemmArgs args;
  int max_items;                // upper bound of work items (grid = min(#SMs, max_items)); 0 = #SMs
};
// bf16 [rows, cols] row-major (pitch ld elements) tensor map with a {box_cols = 64, box_rows} SWIZZLE_128B box.
// Returns 0 on success (1: driver entry point unavailable, 2: encode failed).
int make_tmap_bf16_2d(void* out_map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_cols,
                      int box_rows);
size_t tc_gemm_smem_bytes();

// ---- hetero_infer.cu (full-neighbourhood attention of the heterogeneous engines' layer-wise inference) ----------
// Both kernels walk the COMPLETE CSR row of every target r in [r0, r1) (global ids of the destination type; rows of the
// relation graph are targets, columns are global source ids, ids outside [0, n_src) are skipped).  A row is reduced by
// one lane group, or, above kFullRowHubDeg neighbours (full_rows.cuh; HGT: summed over its relations), by the whole CTA
// with per-group partials merged in group order.  The path depends on the degree alone, so every row has one fixed
// reduction order: no floating-point atomics, bitwise identical for any chunking.  Every exp is of a score minus its row
// maximum.

// R-GAT, one relation r = (s -> t):  e_ij,h = leaky_relu(as[j, h] + ad[i, h], 0.2),  alpha = softmax over i's complete
// in-row per head,  out_i = concat_h sum_j alpha_ij,h P[j, h-block]  (fp32).  first / last as in GatAggArgs:
// acc[i - r0] = out (first) or += out; the last relation writes z[i - r0] = bf16(act(acc + out + sum_b bias[b])),
// act = leaky_relu(., 0.01).  A target without neighbours in r contributes 0 (its output is the bias sum).
struct GatFullAggArgs {
  GraphTable g;
  const void* P;                // bf16 [n_src, H] source projections
  const float* as;              // fp32 [n_src, heads]
  const float* ad;              // fp32 [>= r1, heads] target scores, by global target id
  int64_t n_src;
  int H, heads;
  int64_t r0, r1;
  float* acc;                   // fp32 [r1 - r0, H]
  int first, last;
  const void* bias;             // bf16 [n_bias, H]
  int n_bias;
  int act;
  void* z;                      // bf16 [r1 - r0, H]
};
void launch_gat_full_aggregate(const GatFullAggArgs& a, cudaStream_t s);

// HGT, one destination type with n_rel <= kHgtMaxRel relations (g[r]: device array of their CSR tables):
//   s_ij,h = <qq_r[i, h], k_j,h> prior_r[h] scale   for every neighbour j of i in every relation r
//   alpha  = one softmax per (i, h) over all of them,   u_r[i, h] = bf16(sum_{j in r} alpha_ij,h v_j,h)
// qq and u are chunk rows ([r1 - r0, n_rel * H]); kv[r] is the source type's [K | Q | V] table (bf16 [n_src, kv_ld],
// V at column v_off) by global id.
struct HgtFullAttnArgs {
  const GraphTable* g;          // device [n_rel]
  const void* kv[kHgtMaxRel];
  int64_t n_src[kHgtMaxRel];
  const float* prior[kHgtMaxRel];   // fp32 [heads]
  int n_rel, H, heads, kv_ld, v_off;
  float scale;                  // 1 / sqrt(D)
  const void* qq;
  void* u;
  int64_t r0, r1;
};
void launch_hgt_full_attention(const HgtFullAttnArgs& a, cudaStream_t s);

// ---- link_topk.cu (exact top-K link retrieval over a candidate id range) ---------------------------------------
// For every query row i of [0, n): the k ids c of [lo, hi) with the largest fp32 <emb[queries[i]], emb[c]> (bf16
// wgmma, fp32 accumulation), ordered by (score desc, id asc), excluding queries[i] itself and the columns of row
// queries[i] of g (column-sorted; g.num_parts = 0 or a row past the graph excludes nothing).  Slots past the number of
// eligible candidates get id -1 and score -inf.
struct LinkTopkArgs {
  GraphTable g;
  const int64_t* queries;       // [n], each in [0, N)
  int64_t n;
  int64_t lo, hi;               // candidate ids [lo, hi), hi - lo < 2^31
  int d, k;                     // d a multiple of 8 in [8, 512], k in [1, 128]
  int64_t* part_keys;           // scratch [splits, n, k]
  int64_t* ids;                 // [n, k]
  float* scores;                // [n, k]
};
struct alignas(64) LinkTopkLaunch {
  unsigned char maps[2][128];   // CUtensorMap: gathered query rows bf16 [n, d]; candidate rows bf16 [hi - lo, d]
  LinkTopkArgs args;
  int splits, tiles_per_split;  // candidate tiles of 64 ids per split; every split non-empty
  int stages;                   // from link_topk_stages
};
// Candidate ring stages that fit `smem_limit` bytes of shared memory at (d, k) (0: none fit).
int link_topk_stages(int d, int k, size_t smem_limit);
size_t link_topk_smem_bytes(int d, int k, int stages);
// resident CTAs per SM at (d, k, stages)
int link_topk_ctas_per_sm(int d, int k, int stages);
void launch_link_topk(const LinkTopkLaunch& L, cudaStream_t s);

// ---- kge.cu (knowledge-graph embeddings: TransE, DistMult, ComplEx, RotatE) -------------------------------------------
// Entity rows are fp32 [D] or [re | im] (2D: ComplEx, RotatE); relation rows [D] (RotatE: the phase) or [re | im]
// (ComplEx).  D is a multiple of 8 in [8, 512].  p (1 or 2) is TransE's norm; margin is RotatE's score offset and the
// margin of the TransE / DistMult ranking loss.
enum KgeModel { kKgeTransE = 0, kKgeDistMult = 1, kKgeComplEx = 2, kKgeRotatE = 3 };
int kge_entity_parts(int model);
int kge_relation_parts(int model);
// neg[i * K + j] for i < min(*n_dev, B): uniform in [0, N), Philox(seed, step, i, j).  Slots past n are not written.
void launch_kge_negatives(const int32_t* n_dev, int B, int K, int64_t N, uint64_t seed, const int32_t* step_dev,
                          int64_t* neg, cudaStream_t s);
// trip int64 [3, B] (head, relation, tail rows); the first min(*n_dev, B) columns are the positives.  Positive i
// corrupts its head (i < n / 2) or tail with neg[i * K + j].  Writes the loss to *loss, red.adds the gradients into
// gent / grel and sets tent / trel for every row looked up.
void launch_kge_loss_grad(int model, const int64_t* trip, int B, const int32_t* n_dev, const int64_t* neg, int K,
                          const float* ent, const float* rel, int64_t N, int64_t R, int D, float margin, int p,
                          float* gent, float* grel, uint8_t* tent, uint8_t* trel, float* loss, cudaStream_t s);
// out[i] = score(h[i], r[i], t[i]), ids in range.
void launch_kge_score(int model, const int64_t* h, const int64_t* r, const int64_t* t, int64_t n, const float* ent,
                      const float* rel, int D, float margin, int p, float* out, cudaStream_t s);
// counts[i] = (#candidates scoring above the true entity << 32) + #candidates tied with it, over every entity except
// the true one and the ids of the query's filter range.  tail: query (h, r, ?) with truth t, else (?, r, t) with
// truth h.  keys (sorted int64, may be null): (f R + r) N + c with f the query's fixed entity.
struct KgeRankArgs {
  int model, D, p;
  float margin;
  bool tail;
  const int64_t *h, *r, *t;     // [n], ids in range
  int64_t n, N, R;
  const float *ent, *rel;
  const int64_t* keys;
  int64_t n_keys;
  float* den;                   // scratch [N] (TransE)
  float* q;                     // scratch [n, entity width]
  unsigned long long* counts;   // [n]
  int splits, tiles_per_split;  // candidate tiles of 64 ids per split
};
void launch_kge_rank(const KgeRankArgs& a, cudaStream_t s);

// programmatic-dependent-launch switch (launch_utils.h); returns the previous value
int set_pdl(int on);
void launch_tc_gemm(const TcGemmLaunch& L, int num_sms, cudaStream_t s);

}  // namespace glt
