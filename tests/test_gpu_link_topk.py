"""The top-K link retrieval kernel (csrc/cuda/link_topk.cu) through `link_topk`, against a float64 brute force with the
(score desc, id asc) order: every width, k and query count it accepts, candidate ranges that are not tile multiples,
every exclusion-graph layout, the split count, and the CPU path."""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageLinkEngine, link_topk
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def ref_topk(emb, queries, k, lo, hi, excl=None):
  """float64 brute force on the device.  excl: (row positions into queries, column ids) pairs to drop."""
  e = emb.to(torch.bfloat16).double()
  n = queries.numel()
  s = e[queries] @ e[lo:hi].T
  own = (queries >= lo) & (queries < hi)
  s[torch.arange(n, device=DEV)[own], queries[own] - lo] = float('-inf')
  if excl is not None:
    r, c = excl
    inside = (c >= lo) & (c < hi)
    s[r[inside], c[inside] - lo] = float('-inf')
  kk = min(k, hi - lo)
  order = torch.sort(s, dim=1, descending=True, stable=True).indices[:, :kk]   # ties: ascending column
  sc = s.gather(1, order)
  ids = torch.full((n, k), -1, dtype=torch.int64, device=DEV)
  scores = torch.full((n, k), float('-inf'), dtype=torch.float64, device=DEV)
  ids[:, :kk] = torch.where(sc > float('-inf'), order + lo, torch.full_like(order, -1))
  scores[:, :kk] = sc
  return ids, scores, s


def int_emb(n, d, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randint(-2, 3, (n, d), generator=g, device=DEV).to(torch.bfloat16)


def excl_pairs(queries, indptr, indices):
  """(row position, column) of every exclusion entry of every query row (rows past the CSR have none)"""
  indptr, indices = indptr.to(DEV), indices.to(DEV, torch.int64)
  has = queries < indptr.numel() - 1
  qr = torch.where(has, queries, torch.zeros_like(queries))
  deg = torch.where(has, indptr[qr + 1] - indptr[qr], torch.zeros_like(queries))
  r = torch.repeat_interleave(torch.arange(queries.numel(), device=DEV), deg)
  pos = torch.repeat_interleave(indptr[qr] - torch.cumsum(deg, 0) + deg, deg) + torch.arange(int(deg.sum()), device=DEV)
  return r, indices[pos]


def check_exact(emb, queries, k, lo, hi, exclude=None, excl=None):
  ids, scores = link_topk(emb, queries, k, candidates=(lo, hi), exclude=exclude)
  rid, rs, _ = ref_topk(emb, queries, k, lo, hi, excl)
  assert ids.shape == (queries.numel(), k) and scores.dtype == torch.float32
  assert torch.equal(ids, rid)
  assert torch.equal(scores.double(), rs)
  return ids, scores


@pytest.mark.parametrize('d', [8, 40, 64, 72, 200, 256, 512])
@pytest.mark.parametrize('k', [1, 7, 64, 100, 128])
def test_exact_widths_and_k(d, k):
  """small integer entries: exact, and heavily tied, so the id tie-break is tested at every (d, k)"""
  N = 1500                                                  # 23.4 candidate tiles
  emb = int_emb(N, d, seed=d * 1000 + k)
  queries = torch.randint(0, N, (65,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(k))
  check_exact(emb, queries, k, 0, N)
  check_exact(emb, queries, k, 37, 1200)                    # lo > 0, not tile multiples


@pytest.mark.parametrize('n', [0, 1, 63, 64, 65, 1000])
def test_exact_query_counts(n):
  N, d, k = 2000, 72, 20
  emb = int_emb(N, d, seed=n)
  queries = torch.randint(0, N, (n,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(n))
  check_exact(emb, queries, k, 0, N)


@pytest.mark.parametrize('lo,hi', [(0, 5), (100, 164), (100, 101), (10, 10), (1900, 2000)])
def test_fewer_candidates_than_k(lo, hi):
  N, d, k = 2000, 64, 100
  emb = int_emb(N, d, seed=lo)
  queries = torch.tensor([0, 3, 100, 150, 1999, 1950], device=DEV)   # some inside their own candidate range
  ids, _ = check_exact(emb, queries, k, lo, hi)
  assert (ids[:, max(0, hi - lo):] == -1).all()


def test_random_bf16_valid_topk():
  """every score is the float64 dot of the bf16 values within an fp32 accumulation bound, and the set is a top-K"""
  N, n, k = 5000, 300, 100
  for d in (40, 256, 512):
    g = torch.Generator(device=DEV).manual_seed(d)
    emb = torch.randn(N, d, generator=g, device=DEV).to(torch.bfloat16)
    queries = torch.randint(0, N, (n,), generator=g, device=DEV)
    ids, scores = link_topk(emb, queries, k)
    assert (ids >= 0).all() and (ids != queries[:, None]).all()
    e = emb.double()
    exact = (e[queries].unsqueeze(1) * e[ids]).sum(-1)
    mag = (e[queries].abs().unsqueeze(1) * e[ids].abs()).sum(-1)
    tol = d * 2.0 ** -23 * mag + 1e-30
    assert ((scores.double() - exact).abs() <= tol).all()
    assert (scores[:, :-1] >= scores[:, 1:]).all()
    _, _, s = ref_topk(emb, queries, k, 0, N)
    s.scatter_(1, ids, float('-inf'))                       # the eligible candidates not returned
    slack = d * 2.0 ** -23 * (e[queries].abs() @ e.abs().T).max(1).values
    assert (scores[:, -1].double() >= s.max(1).values - 2 * slack).all()


def _excl_csr(N, hub_rows=(5,), all_row=9):
  """column-sorted CSR over N rows: random rows with duplicates and ids past N, a hub row of 900 entries (14 tiles), and
  a row that excludes every id."""
  g = torch.Generator().manual_seed(3)
  src = torch.randint(0, N, (N * 8,), generator=g)
  dst = torch.randint(0, N + 50, (N * 8,), generator=g)
  extra_s = [torch.full((900,), h) for h in hub_rows] + [torch.full((N,), all_row)]
  extra_d = [torch.randint(0, N, (900,), generator=g) for _ in hub_rows] + [torch.arange(N)]
  src, dst = torch.cat([src] + extra_s), torch.cat([dst] + extra_d)
  order = torch.argsort(src * (N + 100) + dst)
  src, dst = src[order], dst[order]
  indptr = torch.zeros(N + 1, dtype=torch.int64)
  indptr[1:] = torch.cumsum(torch.bincount(src, minlength=N), 0)
  return indptr, dst


@pytest.mark.parametrize('layout', ['int32', 'int64', 'two_shards', 'zero_copy'])
def test_exclusion_layouts(layout):
  N, d, k = 3000, 64, 50
  R = 2500                                                  # rows R.. have no exclusion row
  indptr, indices = _excl_csr(R)
  if layout == 'int32':
    shards = [{'indptr': indptr.to(DEV), 'indices': indices.to(DEV, torch.int32), 'row_begin': 0, 'row_end': R}]
  elif layout == 'int64':
    shards = [{'indptr': indptr.to(DEV), 'indices': indices.to(DEV), 'row_begin': 0, 'row_end': R}]
  elif layout == 'two_shards':
    h = 7                                                 # row 9 (excludes all) in shard 1, the hub in shard 0
    shards = [{'indptr': indptr[:h + 1].to(DEV), 'indices': indices[:indptr[h]].to(DEV), 'row_begin': 0,
               'row_end': h},
              {'indptr': (indptr[h:] - indptr[h]).to(DEV), 'indices': indices[indptr[h]:].to(DEV), 'row_begin': h,
               'row_end': R}]
  else:
    shards = [{'indptr': indptr.pin_memory(), 'indices': indices.to(torch.int32).pin_memory(), 'row_begin': 0,
               'row_end': R}]
  graph = glt.data.Graph.from_shards(shards, 0)
  graph._keep_shards = shards
  emb = int_emb(N, d, seed=11)
  queries = torch.cat([torch.tensor([5, 9, 0, 2499, 2500, 2999, 5], device=DEV),
                       torch.randint(0, N, (200,), device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))])
  excl = excl_pairs(queries, indptr, indices)
  for lo, hi in ((0, N), (130, 2031)):
    check_exact(emb, queries, k, lo, hi, exclude=graph, excl=excl)
  ids, scores = check_exact(emb, queries, k, 0, R, exclude=graph, excl=excl)
  assert (ids[1] == -1).all() and torch.isinf(scores[1]).all()   # row 9 excludes every candidate of [0, R)


def test_splits_are_bitwise_identical(native):
  N, d, k = 20000, 128, 100
  g = torch.Generator(device=DEV).manual_seed(0)
  emb = torch.randn(N, d, generator=g, device=DEV).to(torch.bfloat16)
  queries = torch.randint(0, N, (200,), generator=g, device=DEV)
  indptr, indices = _excl_csr(N)
  graph = glt.data.Graph.from_shards(
      [{'indptr': indptr.to(DEV), 'indices': indices.to(DEV, torch.int32), 'row_begin': 0, 'row_end': N}], 0)
  outs = [native.link_topk(emb, queries, k, 10, N - 7, graph.graph_handler, s) for s in (1, 3, 0, 0)]
  for ids, scores in outs[1:]:
    assert torch.equal(ids, outs[0][0])
    assert torch.equal(scores.view(torch.int32), outs[0][1].view(torch.int32))


def test_fp32_is_its_bf16_rounding():
  emb = torch.randn(3000, 96, device=DEV)
  q = torch.arange(0, 3000, 11, device=DEV)
  a, b = link_topk(emb, q, 30), link_topk(emb.to(torch.bfloat16), q, 30)
  assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_gpu_matches_cpu():
  N, d, k = 4000, 64, 64
  g = torch.Generator(device=DEV).manual_seed(2)
  emb = torch.randn(N, d, generator=g, device=DEV).to(torch.bfloat16)
  queries = torch.randint(0, N, (150,), generator=g, device=DEV)
  ei = rmat_edges(N, 40000, seed=3)
  topo = glt.data.Topology(torch.cat([ei, ei.flip(0)], 1), layout='CSR', num_nodes=N)
  ids, scores = link_topk(emb, queries, k, exclude=glt.data.Graph(topo, 'CUDA', 0))
  cids, cscores = link_topk(emb.cpu(), queries.cpu(), k, exclude=glt.data.Graph(topo, 'CPU'))
  tol = 1e-4 + 1e-5 * cscores.abs()                      # fp32 sums of 64 products in two orders
  assert ((scores.cpu() - cscores).abs() <= tol).all()
  # the id lists agree except where two candidates' scores are within fp32 rounding of each other
  same = ids.cpu() == cids
  near_tie = (scores.cpu() - cscores).abs() <= tol
  assert (same | near_tie).all()
  assert same.float().mean() > 0.99


def test_bad_arguments_raise(native):
  emb = torch.zeros(100, 64, device=DEV, dtype=torch.bfloat16)
  q = torch.tensor([1, 2], device=DEV)
  bad_native = [
      (emb.float(), q, 5, 0, 100), (emb[:, :60].contiguous(), q, 5, 0, 100), (emb.t().contiguous()[:, :96], q, 5, 0, 64),
      (torch.zeros(100, 520, device=DEV, dtype=torch.bfloat16), q, 5, 0, 100), (emb, q, 0, 0, 100), (emb, q, 129, 0, 100),
      (emb, q, 5, -1, 100), (emb, q, 5, 50, 40), (emb, q, 5, 0, 101), (emb, q.int(), 5, 0, 100),
      (emb, q.cpu(), 5, 0, 100), (emb, torch.tensor([100], device=DEV), 5, 0, 100),
      (emb, torch.tensor([-1], device=DEV), 5, 0, 100), (emb.cpu(), q, 5, 0, 100),
      (emb[:, ::2], q, 5, 0, 100),
  ]
  for args in bad_native:
    with pytest.raises(RuntimeError):
      native.link_topk(*args, None, 0)
  with pytest.raises(RuntimeError):
    native.link_topk(emb, q, 5, 0, 100, None, -1)
  for call in (lambda: link_topk(emb, q.cpu(), 5), lambda: link_topk(emb, q, 5, candidates=(0, 101)),
               lambda: link_topk(emb, q, 200), lambda: link_topk(emb[:, :12], q, 5),
               lambda: link_topk(emb, q, 5, exclude=glt.data.Graph(glt.data.Topology(
                   torch.zeros(2, 1, dtype=torch.int64), layout='CSR', num_nodes=1), 'CPU'))):
    with pytest.raises(ValueError):
      call()
  ids, _ = native.link_topk(emb, q, 5, 0, 100, None, 0)    # the process is still healthy
  torch.cuda.synchronize()
  assert ids.shape == (2, 5)


def test_engine_state_is_untouched():
  N, Fdim = 3000, 64
  ei = rmat_edges(N, 30000, seed=4)
  topo = glt.data.Topology(torch.cat([ei, ei.flip(0)], 1), layout='CSR', num_nodes=N)
  graph = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(0)
  feats = torch.randn(N, Fdim, device=DEV).to(torch.bfloat16)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageLinkEngine(graph, ut._table(), Fdim, N, fanouts=[5, 5], batch_size=256, hidden=128,
                            out_channels=64, device=DEV, use_cuda_graph=False, seed=5)
  pairs = torch.cat([ei, ei.flip(0)], 1)
  for i in range(3):
    eng.train_step(pairs[:, i * 256:(i + 1) * 256].to(DEV))
  eng.flush()
  torch.cuda.synchronize()
  snap = eng.state_dict()
  p16 = eng.p16.clone()
  emb = eng.inference()
  ids, scores = link_topk(emb, torch.arange(0, N, 5, device=DEV), 20, exclude=graph)
  torch.cuda.synchronize()
  after = eng.state_dict()
  for key in ('p32', 'm', 'v'):
    assert torch.equal(after[key], snap[key]), key
  assert after['step'] == snap['step']
  assert torch.equal(eng.p16, p16)
  assert (ids >= 0).all()
