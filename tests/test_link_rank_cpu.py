"""Top-K link retrieval on the CPU path and the ranking metrics (models/link_rank.py) against brute force and
hand-computed values."""
import os
import subprocess
import sys

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import (link_hits_at_k, link_mrr, link_recall_at_k, link_scores,
                                                link_topk)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def brute_topk(emb, queries, k, lo, hi, excl_rows=None):
  """float64 scores of the bf16 values, (score desc, id asc), padded with (-1, -inf).  excl_rows: {query: ids}."""
  e = emb.to(torch.bfloat16).double().cpu()
  ids = torch.full((len(queries), k), -1, dtype=torch.int64)
  scores = torch.full((len(queries), k), float('-inf'), dtype=torch.float64)
  for i, q in enumerate(queries.tolist()):
    banned = {q} | set((excl_rows or {}).get(q, ()))
    cand = [c for c in range(lo, hi) if c not in banned]
    s = (e[cand] @ e[q]).tolist()
    best = sorted(zip(s, cand), key=lambda t: (-t[0], t[1]))[:k]
    for j, (sc, c) in enumerate(best):
      ids[i, j], scores[i, j] = c, sc
  return ids, scores


def int_emb(n, d, seed, lo=-2, hi=2):
  """small integer entries: exact in bf16, and their fp32 dot products are exact"""
  g = torch.Generator().manual_seed(seed)
  return torch.randint(lo, hi + 1, (n, d), generator=g).to(torch.bfloat16)


def rows_of(indptr, indices):
  return {r: indices[indptr[r]:indptr[r + 1]].tolist() for r in range(indptr.numel() - 1)}


def excl_graph(n_rows, n_cols, seed, extra=()):
  """random column-sorted CSR with duplicates, plus (row, col) pairs in `extra`"""
  g = torch.Generator().manual_seed(seed)
  src = torch.randint(0, n_rows, (n_rows * 6,), generator=g)
  dst = torch.randint(-3, n_cols + 3, (n_rows * 6,), generator=g).clamp(min=0)   # ids past the range, duplicates
  for r, c in extra:
    src = torch.cat([src, torch.tensor([r])])
    dst = torch.cat([dst, torch.tensor([c])])
  order = torch.argsort(src * (n_cols + 10) + dst)
  src, dst = src[order], dst[order]
  indptr = torch.zeros(n_rows + 1, dtype=torch.int64)
  indptr[1:] = torch.cumsum(torch.bincount(src, minlength=n_rows), 0)
  return indptr, dst


@pytest.mark.parametrize('d,k,n,lo,hi', [(8, 1, 5, 0, 50), (40, 7, 17, 0, 300), (64, 100, 3, 10, 60),
                                         (72, 5, 0, 0, 40), (16, 10, 9, 30, 30), (24, 12, 6, 5, 97)])
def test_cpu_topk_exact(d, k, n, lo, hi):
  N = 300
  emb = int_emb(N, d, seed=d + k)
  queries = torch.randint(0, N, (n,), generator=torch.Generator().manual_seed(n))
  ids, scores = link_topk(emb, queries, k, candidates=(lo, hi))
  rid, rs = brute_topk(emb, queries, k, lo, hi)
  assert ids.shape == (n, k) and ids.dtype == torch.int64 and scores.dtype == torch.float32
  assert torch.equal(ids, rid)
  assert torch.equal(scores.double(), rs)


def test_cpu_topk_exclusion():
  N, d, k = 200, 32, 20
  emb = int_emb(N, d, seed=3)
  hub = (5, list(range(0, 200, 1)))        # excludes every candidate
  indptr, indices = excl_graph(150, N, seed=1, extra=[(7, c) for c in range(0, 180)])
  rows = rows_of(indptr, indices)
  rows[5] = sorted(set(rows.get(5, [])) | set(hub[1]))
  src = torch.repeat_interleave(torch.arange(150), torch.tensor([len(rows[r]) for r in range(150)]))
  dst = torch.tensor([c for r in range(150) for c in rows[r]], dtype=torch.int64)
  topo = glt.data.Topology(torch.stack([src, dst]), layout='CSR', num_nodes=150)
  graph = glt.data.Graph(topo, 'CPU')
  t_rows = rows_of(topo.indptr, topo.indices)
  queries = torch.tensor([5, 7, 0, 3, 149, 170, 199, 7])   # 170 and 199 have no row: nothing excluded
  for lo, hi in [(0, N), (50, 120)]:
    ids, scores = link_topk(emb, queries, k, candidates=(lo, hi), exclude=graph)
    rid, rs = brute_topk(emb, queries, k, lo, hi, t_rows)
    assert torch.equal(ids, rid)
    assert torch.equal(scores.double(), rs)
  assert (ids[0] == -1).all() and torch.isinf(scores[0]).all()


def test_cpu_topk_fp32_is_its_bf16_rounding():
  emb = torch.randn(120, 48, generator=torch.Generator().manual_seed(0))
  q = torch.arange(0, 120, 7)
  a = link_topk(emb, q, 9)
  b = link_topk(emb.to(torch.bfloat16), q, 9)
  assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize('bad', [
  dict(emb=torch.zeros(10, 12)), dict(emb=torch.zeros(10, 520)), dict(emb=torch.zeros(10, 8, dtype=torch.int32)),
  dict(k=0), dict(k=129), dict(queries=torch.tensor([10])), dict(queries=torch.tensor([-1])),
  dict(queries=torch.tensor([1], dtype=torch.int32)), dict(candidates=(3, 2)), dict(candidates=(0, 11)),
])
def test_cpu_topk_rejects(bad):
  args = dict(emb=torch.zeros(10, 8), queries=torch.tensor([1, 2]), k=3, candidates=None)
  args.update(bad)
  with pytest.raises(ValueError):
    link_topk(args['emb'], args['queries'], args['k'], candidates=args['candidates'])


def test_link_scores_chunked():
  emb = torch.randn(50, 16, generator=torch.Generator().manual_seed(1))
  pairs = torch.randint(0, 50, (2, 37), generator=torch.Generator().manual_seed(2))
  ref = (emb[pairs[0]] * emb[pairs[1]]).sum(-1)
  assert torch.allclose(link_scores(emb, pairs, chunk=5), ref, atol=1e-5)


def test_hits_at_k():
  neg = torch.tensor([0.1, 0.5, 0.3, 0.9])
  pos = torch.tensor([0.95, 0.5, 0.4, 0.2])
  assert link_hits_at_k(pos, neg, 1) == pytest.approx(0.25)     # > 0.9
  assert link_hits_at_k(pos, neg, 2) == pytest.approx(0.25)     # > 0.5, strictly
  assert link_hits_at_k(pos, neg, 3) == pytest.approx(0.75)     # > 0.3
  assert link_hits_at_k(pos, neg, 5) == 1.0                     # fewer than k negatives


def test_mrr_ties():
  pos = torch.tensor([1.0, 2.0])
  neg = torch.tensor([[1.0, 1.0, 0.0], [3.0, 2.0, 2.0]])
  # row 0: optimistic 0, pessimistic 2 -> rank 2; row 1: optimistic 1, pessimistic 3 -> rank 3
  assert link_mrr(pos, neg) == pytest.approx((1 / 2 + 1 / 3) / 2)


def test_recall_at_k():
  # truth rows: 0 -> {1, 2, 2}, 1 -> {}, 2 -> {0}; query 9 is past the rows
  indptr = torch.tensor([0, 3, 3, 4])
  indices = torch.tensor([1, 2, 2, 0])
  queries = torch.tensor([0, 1, 2, 9])
  ids = torch.tensor([[2, 5, -1], [0, 2, 3], [4, 5, 6], [1, 2, 3]])
  recall, hit = link_recall_at_k(ids, (indptr, indices), queries)
  assert recall == pytest.approx((1 / 2 + 0 / 1) / 2)        # queries 1 and 9 have no held-out edges
  assert hit == pytest.approx(0.5)
  assert link_recall_at_k(ids[1:2], (indptr, indices), queries[1:2]) == (0.0, 0.0)


def test_example_rank_k():
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  out = subprocess.run([sys.executable, 'examples/graph_sage_unsup.py', '--mode', 'engine', '--epochs', '1',
                        '--steps-per-epoch', '5', '--rank-k', '10'], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
  assert out.returncode == 0, out.stderr[-2000:]
  assert 'held-out link AUC' in out.stdout
  assert 'recall@10' in out.stdout and 'Hits@10' in out.stdout and 'MRR' in out.stdout
