"""Ranking evaluation of link predictors: exact top-K retrieval over every candidate node, and the metrics published
link-prediction results report (recall@K, OGB's Hits@K and MRR).

`link_topk(emb, queries, k)` ranks each query against every candidate by the dot product of their embeddings, the
score `GraphSageLinkEngine`, `MetaPath2VecEngine` and `link_auc` use.  On a CUDA `emb` one sm_90a kernel
(csrc/cuda/link_topk.cu) computes the scores with bf16 tensor-core MMAs and fp32 accumulation and keeps each query's
running top-K on chip, so the [queries, candidates] score matrix is never written.  On CPU tensors a chunked torch path
(fp32 matmul of the same bf16-rounded values, -inf over the excluded ids, top-k) has the same contract; its fp32 sums
are ordered differently, so the two paths agree up to near-ties.

The metrics are small reductions in plain torch, on the CPU or the GPU.
"""
from typing import Optional, Tuple, Union

import torch

from ..ops import require_native

MAX_K = 128


def _check_topk_args(emb: torch.Tensor, queries: torch.Tensor, k: int, candidates) -> Tuple[int, int]:
  if emb.dim() != 2:
    raise ValueError(f'emb must be 2-D [N, d], got shape {tuple(emb.shape)}')
  if emb.dtype not in (torch.bfloat16, torch.float32):
    raise ValueError(f'emb must be bf16 or fp32, not {emb.dtype}')
  n_nodes, d = emb.shape
  if d % 8 != 0 or not 8 <= d <= 512:
    raise ValueError(f'the embedding width must be a multiple of 8 in [8, 512], not {d}')
  if int(k) != k or not 1 <= k <= MAX_K:
    raise ValueError(f'k must be an integer in [1, {MAX_K}], not {k}')
  if queries.dim() != 1 or queries.dtype != torch.int64:
    raise ValueError('queries must be a 1-D int64 tensor of node ids')
  if candidates is None:
    lo, hi = 0, n_nodes
  else:
    lo, hi = (int(c) for c in candidates)
    if not 0 <= lo <= hi <= n_nodes:
      raise ValueError(f'candidates ({lo}, {hi}) must be an id range inside [0, {n_nodes})')
  if queries.numel() > 0:
    qmin, qmax = int(queries.min()), int(queries.max())
    if qmin < 0 or qmax >= n_nodes:
      raise ValueError(f'query ids must lie in [0, {n_nodes}), got [{qmin}, {qmax}]')
  return lo, hi


def _csr(graph) -> Tuple[torch.Tensor, torch.Tensor]:
  """(indptr, indices) of a `data.Graph` built from a Topology, or of an (indptr, indices) pair."""
  if isinstance(graph, (tuple, list)):
    indptr, indices = graph
    return torch.as_tensor(indptr), torch.as_tensor(indices)
  if getattr(graph, 'topo', None) is None:
    raise ValueError('the graph needs its Topology (a Graph assembled from shards has none on the host)')
  return graph.topo.indptr, graph.topo.indices


def _topk_torch(emb: torch.Tensor, queries: torch.Tensor, k: int, lo: int, hi: int, exclude,
                chunk_bytes: int = 1 << 28) -> Tuple[torch.Tensor, torch.Tensor]:
  n = queries.numel()
  ids = torch.full((n, k), -1, dtype=torch.int64)
  scores = torch.full((n, k), float('-inf'), dtype=torch.float32)
  n_cand = hi - lo
  if n == 0 or n_cand == 0:
    return ids, scores
  cand = emb[lo:hi].float()
  indptr, indices = _csr(exclude) if exclude is not None else (None, None)
  rows = max(1, chunk_bytes // (4 * n_cand))
  for r0 in range(0, n, rows):
    q = queries[r0:r0 + rows]
    m = q.numel()
    s = emb[q].float() @ cand.T
    own = (q >= lo) & (q < hi)
    s[torch.arange(m)[own], q[own] - lo] = float('-inf')
    if indptr is not None:
      has_row = q < indptr.numel() - 1
      qr = torch.where(has_row, q, torch.zeros_like(q))
      deg = torch.where(has_row, indptr[qr + 1] - indptr[qr], torch.zeros_like(q))
      r = torch.repeat_interleave(torch.arange(m), deg)
      pos = torch.repeat_interleave(indptr[qr] - torch.cumsum(deg, 0) + deg, deg) + torch.arange(int(deg.sum()))
      c = indices[pos].to(torch.int64)
      inside = (c >= lo) & (c < hi)
      s[r[inside], c[inside] - lo] = float('-inf')
    # every entry >= each row's k-th largest value, then (score desc, id asc) by a stable sort of id-ordered columns
    kk = min(k, n_cand)
    kth = torch.topk(s, kk, dim=1).values[:, -1:]
    width = int((s >= kth).sum(1).max())
    top_s, top_i = torch.topk(s, width, dim=1)
    by_id = torch.argsort(top_i, dim=1)
    top_s, top_i = top_s.gather(1, by_id), top_i.gather(1, by_id)
    order = torch.sort(top_s, dim=1, descending=True, stable=True).indices[:, :kk]
    top_s, top_i = top_s.gather(1, order), top_i.gather(1, order)
    keep = top_s > float('-inf')
    ids[r0:r0 + m, :kk] = torch.where(keep, top_i + lo, torch.full_like(top_i, -1))
    scores[r0:r0 + m, :kk] = top_s
  return ids, scores


def link_topk(emb: torch.Tensor, queries: torch.Tensor, k: int, candidates: Optional[Tuple[int, int]] = None,
              exclude=None) -> Tuple[torch.Tensor, torch.Tensor]:
  """The k best candidates of every query by dot-product score, over all candidates: exact top-K retrieval.

  Args:
    emb: [N, d] node embeddings, bf16, or fp32 (rounded to bf16 once; scores are of the rounded values).  d is a
      multiple of 8 in [8, 512].  Entries must be finite.
    queries: int64 [n] node ids in [0, N) on emb's device; n may be 0.
    k: 1 <= k <= 128.
    candidates: None for every node id [0, N), or an id range (lo, hi), e.g. the item block of a user-item graph.
    exclude: None, or a `data.Graph` whose row q lists ids never returned for query q (typically the training graph).
      Rows must be column-sorted, as `Topology` builds them (not checked).  A query id at or past the graph's row
      count excludes nothing; duplicate ids and ids outside the candidate range are harmless.  The query itself is
      never returned.

  Returns (ids int64 [n, k], scores fp32 [n, k]) with score = <emb[q], emb[c]> accumulated in fp32, sorted by score
  descending with ties broken by the smaller id; ids are global node ids.  Slots past the number of eligible
  candidates hold id -1 and score -inf.

  A CUDA `emb` with a 'CUDA' or 'ZERO_COPY' exclusion graph (or none) runs the sm_90a kernel, whose results are
  bitwise identical from run to run; CPU tensors with a 'CPU' graph (or none) run a chunked torch path.  Mixed devices
  raise ValueError.
  """
  if not isinstance(queries, torch.Tensor):
    queries = torch.as_tensor(queries, dtype=torch.int64)
  if queries.device != emb.device:
    raise ValueError(f'queries are on {queries.device}, emb on {emb.device}')
  lo, hi = _check_topk_args(emb, queries, k, candidates)
  k = int(k)
  if exclude is not None:
    on_cpu = exclude.mode == 'CPU'
    if on_cpu != (emb.device.type == 'cpu') or (not on_cpu and int(exclude.device) != emb.device.index):
      where = 'the CPU' if on_cpu else f'cuda:{exclude.device}'
      raise ValueError(f'the exclusion graph lives on {where}, emb on {emb.device}')
  emb = emb.to(torch.bfloat16).contiguous()
  if emb.device.type == 'cpu':
    return _topk_torch(emb, queries.contiguous(), k, lo, hi, exclude)
  if emb.device.type != 'cuda':
    raise ValueError(f'emb must be a CPU or CUDA tensor, not on {emb.device}')
  handle = exclude.graph_handler if exclude is not None else None
  return require_native().link_topk(emb, queries.contiguous(), k, lo, hi, handle, 0)


def link_scores(emb: torch.Tensor, pairs: torch.Tensor, chunk: int = 1 << 16) -> torch.Tensor:
  """fp32 dot products <emb[u], emb[v]> of the pairs [2, n], on emb's device.  At most `chunk` pairs of fp32 rows are
  materialised at a time."""
  pairs = torch.as_tensor(pairs).to(emb.device)
  if pairs.dim() != 2 or pairs.size(0) != 2:
    raise ValueError(f'pairs must be [2, n], got shape {tuple(pairs.shape)}')
  out = torch.empty(pairs.size(1), dtype=torch.float32, device=emb.device)
  for i in range(0, pairs.size(1), chunk):
    u, v = pairs[0, i:i + chunk], pairs[1, i:i + chunk]
    out[i:i + chunk] = (emb[u].float() * emb[v].float()).sum(-1)
  return out


def link_recall_at_k(ids: torch.Tensor, truth, queries: torch.Tensor, chunk: int = 1 << 20) -> Tuple[float, float]:
  """Recall@K of retrieved ids [n, K] (from `link_topk`) against held-out neighbours.

  truth: a `data.Graph` or an (indptr, indices) CSR; row q lists the held-out neighbours of query q (duplicates count
  once; a query id at or past its row count has none).  queries: int64 [n], the query of each row of `ids`.
  Returns (recall, hit_rate) over the queries that have any held-out neighbour: recall is the mean of
  |found| / |held-out|, hit_rate the fraction with at least one found.  Both are 0.0 when no query has any.
  """
  indptr, indices = _csr(truth)
  dev = ids.device
  indptr, indices = indptr.to(dev, torch.int64), indices.to(dev, torch.int64)
  queries = torch.as_tensor(queries).to(dev, torch.int64)
  n = queries.numel()
  if ids.dim() != 2 or ids.size(0) != n:
    raise ValueError(f'ids must be [n, K] with one row per query ({n}), got shape {tuple(ids.shape)}')
  has_row = (queries >= 0) & (queries < indptr.numel() - 1)
  qr = torch.where(has_row, queries, torch.zeros_like(queries))
  deg = torch.where(has_row, indptr[qr + 1] - indptr[qr], torch.zeros_like(queries))
  r = torch.repeat_interleave(torch.arange(n, device=dev), deg)
  pos = torch.repeat_interleave(indptr[qr] - torch.cumsum(deg, 0) + deg, deg) + torch.arange(int(deg.sum()), device=dev)
  t = indices[pos]
  if r.numel() > 0:   # one (query row, neighbour) pair per distinct held-out neighbour
    span = int(t.max()) + 2
    key = torch.unique(r * span + (t + 1))
    r, t = key // span, key % span - 1
  relevant = torch.bincount(r, minlength=n)
  found = torch.zeros(n, dtype=torch.int64, device=dev)
  for i in range(0, r.numel(), chunk):
    rr, tt = r[i:i + chunk], t[i:i + chunk]
    found.index_add_(0, rr, (ids[rr] == tt.unsqueeze(1)).any(1).to(torch.int64))
  counted = relevant > 0
  if not bool(counted.any()):
    return 0.0, 0.0
  recall = (found[counted].double() / relevant[counted].double()).mean()
  hit = (found[counted] > 0).double().mean()
  return float(recall), float(hit)


def link_hits_at_k(pos_scores: torch.Tensor, neg_scores: torch.Tensor, k: int) -> float:
  """OGB's Hits@K (ogbl-collab, -ppa, -ddi): the fraction of positive scores strictly greater than the k-th largest
  negative score; 1.0 when there are fewer than k negatives."""
  neg_scores = neg_scores.reshape(-1)
  if neg_scores.numel() < k:
    return 1.0
  kth = torch.topk(neg_scores.to(pos_scores.device), k).values[-1]
  return float((pos_scores > kth).double().mean())


def link_mrr(pos_scores: torch.Tensor, neg_scores: torch.Tensor) -> float:
  """OGB's citation2 mean reciprocal rank: positive i is ranked against its own negatives neg_scores[i] ([n, m]) at
  1 + the mean of the optimistic count (negatives >) and the pessimistic count (negatives >=)."""
  if neg_scores.dim() != 2 or neg_scores.size(0) != pos_scores.numel():
    raise ValueError(f'neg_scores must be [n, m] with one row per positive, got shape {tuple(neg_scores.shape)}')
  pos = pos_scores.reshape(-1, 1)
  optimistic = (neg_scores > pos).sum(1)
  pessimistic = (neg_scores >= pos).sum(1)
  rank = 1.0 + 0.5 * (optimistic + pessimistic).double()
  return float((1.0 / rank).mean())
