"""SealEngine: per-link enclosing subgraphs and DRNL labels (k_seal_extract) against a Python / scipy oracle, the
DGCNN forward and backward against a float64 oracle of the reference module, Adam against torch.optim.Adam, CUDA-graph
replay, checkpoints, padding, learning a planted block graph, the example's engine mode, and argument errors."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.nn.functional as F
from scipy.sparse.csgraph import shortest_path

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import SealEngine

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _graph(ei, n):
  g = glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=n), 'CUDA', 0)
  g.lazy_init()
  return g


def _random_graph(n=60, seed=0):
  """Symmetric random graph with two hubs, isolated nodes (n-3 .. n-1), a self-loop and a duplicated edge."""
  gen = torch.Generator().manual_seed(seed)
  m = n - 3
  src = torch.randint(0, m, (2 * n,), generator=gen)
  dst = torch.randint(0, m, (2 * n,), generator=gen)
  hubs = torch.tensor([0, 1])
  hs = hubs.repeat_interleave(m // 2)
  hd = torch.randint(0, m, (hs.numel(),), generator=gen)
  src, dst = torch.cat([src, hs]), torch.cat([dst, hd])
  keep = src != dst
  ei = torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)
  ei = torch.cat([ei, ei.flip(0)], 1)
  ei = torch.cat([ei, torch.tensor([[5, 6, 6], [5, 7, 7]]), torch.tensor([[7], [6]])], 1)   # self-loop, duplicate 6->7
  return ei, n


def _csr(g):
  return g.topo.indptr.cpu().tolist(), g.topo.indices.cpu().tolist()


def oracle_extract(indptr, indices, s, d, hops, max_nodes, max_edges, max_z=None):
  """Nodes in discovery order, local edges in (source, row position) order, DRNL labels, truncated flag."""
  row = lambda u: indices[indptr[u]:indptr[u + 1]]
  nodes, pos, fb, fe, trunc = [s, d], {s: 0, d: 1}, 0, 2, False
  for _ in range(hops):
    if trunc or fb >= fe:
      break
    for f in range(fb, fe):
      for v in row(nodes[f]):
        if v not in pos:
          if len(nodes) >= max_nodes:
            trunc = True
            break
          pos[v] = len(nodes)
          nodes.append(v)
      if trunc:
        break
    fb, fe = fe, len(nodes)
  edges = []
  for lu, u in enumerate(nodes):
    for v in row(u):
      if v in pos and (lu, pos[v]) not in ((0, 1), (1, 0)):
        edges.append((lu, pos[v]))
  if len(edges) > max_edges:
    trunc, edges = True, edges[:max_edges]
  n = len(nodes)
  z = drnl(edges, n)
  if max_z is not None:
    z = np.minimum(z, max_z)
  return nodes, edges, z, trunc


def drnl(edges, n):
  """The reference's DRNL: scipy shortest paths on the undirected subgraph with the other endpoint deleted."""
  e = np.array(edges, dtype=np.int64).reshape(-1, 2)
  adj = sp.csr_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n))
  dist = []
  for src, rem in ((0, 1), (1, 0)):
    idx = [i for i in range(n) if i != rem]
    sub = adj[idx, :][:, idx]
    dd = shortest_path(sub, directed=False, unweighted=True, indices=idx.index(src))
    dist.append(np.insert(dd, rem, 0.0))
    dist[-1][rem] = np.inf
  ds, dd = dist
  D = ds + dd
  with np.errstate(invalid='ignore'):
    z = 1 + np.minimum(ds, dd) + (D // 2) * (D // 2 + D % 2 - 1)
  z[~np.isfinite(z)] = 0
  z[0] = z[1] = 1
  return z.astype(np.int64)


def engine_subgraph(eng, b):
  meta = eng.arena.meta[b].cpu().tolist()
  n, e = meta[0], meta[1]
  nodes = eng.arena.nodes[b, :n].cpu().tolist()
  sptr = eng.arena.sptr[b, :n + 1].cpu().tolist()
  scol = eng.arena.scol[b, :e].cpu().tolist()
  edges = [(u, scol[q]) for u in range(n) for q in range(sptr[u], sptr[u + 1])]
  dptr = eng.arena.dptr[b, :n + 1].cpu().tolist()
  dcol = eng.arena.dcol[b, :e].cpu().tolist()
  edges_t = [(dcol[q], v) for v in range(n) for q in range(dptr[v], dptr[v + 1])]
  z = eng.arena.z[b, :n].cpu().numpy()
  return meta, nodes, edges, edges_t, z


def _links(n, seed, count=40):
  gen = torch.Generator().manual_seed(seed)
  return torch.randint(0, n, (2, count), generator=gen)


# ------------------------------------------------------------------ 1. extraction
@pytest.mark.parametrize('hops', [1, 2, 3])
def test_extraction_matches_oracle(hops):
  ei, n = _random_graph()
  g = _graph(ei, n)
  indptr, indices = _csr(g)
  links = torch.cat([_links(n, hops), torch.tensor([[6, 5, 0, 57, 58], [7, 5, 1, 58, 3]])], 1)   # edge, self-loop node,
  eng = SealEngine(g, n, num_hops=hops, max_nodes=1024, max_edges=4096, max_z=1000, sort_k=10, hidden=8,
                   num_layers=1, batch_size=links.shape[1])                                      # hubs, isolated
  eng._extract(links.to(DEV))
  for b in range(links.shape[1]):
    s, d = links[:, b].tolist()
    meta, nodes, edges, edges_t, z = engine_subgraph(eng, b)
    if s == d:
      assert meta[2] == 0
      continue
    o_nodes, o_edges, o_z, _ = oracle_extract(indptr, indices, s, d, hops, 1024, 4096)
    assert nodes == o_nodes
    assert edges == o_edges                                          # multiset and its (source, row) order
    assert sorted(edges_t) == sorted(o_edges)
    assert np.array_equal(z, o_z)
  assert eng.truncated() == 0


def test_truncation_keeps_the_discovery_prefix():
  ei, n = _random_graph(seed=3)
  g = _graph(ei, n)
  indptr, indices = _csr(g)
  links = _links(n, 7, 48)
  for max_nodes, max_edges in ((8, 4096), (1024, 12), (6, 5)):
    eng = SealEngine(g, n, num_hops=2, max_nodes=max_nodes, max_edges=max_edges, max_z=1000, sort_k=10, hidden=8,
                     num_layers=1, batch_size=links.shape[1])
    eng._extract(links.to(DEV))
    expect = 0
    for b in range(links.shape[1]):
      s, d = links[:, b].tolist()
      meta, nodes, edges, _, z = engine_subgraph(eng, b)
      if s == d:
        continue
      o_nodes, o_edges, o_z, tr = oracle_extract(indptr, indices, s, d, 2, max_nodes, max_edges)
      assert nodes == o_nodes and edges == o_edges and np.array_equal(z, o_z)
      assert meta[3] == int(tr)
      expect += int(tr)
    assert expect > 0
    assert eng.truncated() == expect


def test_neighbour_caps_hold_and_are_keyed_by_seed_and_step():
  ei, n = _random_graph(n=200, seed=4)
  g = _graph(ei, n)
  indptr, indices = _csr(g)
  adj = [set(indices[indptr[u]:indptr[u + 1]]) for u in range(n)]
  links = _links(n, 9, 64)
  kw = dict(num_hops=2, num_neighbors=[3, 2], max_nodes=1024, max_edges=8192, max_z=1000, sort_k=10, hidden=8,
            num_layers=1, batch_size=links.shape[1])
  eng = SealEngine(g, n, seed=1, **kw)
  eng._extract(links.to(DEV))
  first = [engine_subgraph(eng, b)[1] for b in range(links.shape[1])]
  for b, nodes in enumerate(first):
    s, d = links[:, b].tolist()
    if s == d:
      continue
    # every node past the endpoints is a neighbour of an earlier node, and a hop adds at most sum(min(deg, cap))
    for i, v in enumerate(nodes[2:], 2):
      assert any(v in adj[u] for u in nodes[:i])
    assert len(nodes) - 2 <= 6 + 6 * 2                            # hop 1 adds <= 2 x 3 nodes, hop 2 <= 2 per hop-1 node
  eng._extract(links.to(DEV))
  assert [engine_subgraph(eng, b)[1] for b in range(links.shape[1])] == first       # same (seed, step)
  eng.state[0] += 1
  eng._extract(links.to(DEV))
  assert [engine_subgraph(eng, b)[1] for b in range(links.shape[1])] != first       # next step
  eng.state[0] -= 1
  other = SealEngine(g, n, seed=2, **kw)
  other._extract(links.to(DEV))
  assert [engine_subgraph(other, b)[1] for b in range(links.shape[1])] != first     # other seed
  big = SealEngine(g, n, seed=1, **{**kw, 'num_neighbors': [1024, 1024]})           # caps above every degree
  big._extract(links.to(DEV))
  for b in range(links.shape[1]):
    s, d = links[:, b].tolist()
    if s != d:
      assert engine_subgraph(big, b)[1] == oracle_extract(indptr, indices, s, d, 2, 1024, 8192)[0]


# ------------------------------------------------------------------ float64 oracle of the reference DGCNN
class GCNConv64(torch.nn.Module):
  """PyG GCNConv: lin (no bias), A + I with input self-loops replaced, destination degrees, bias after."""

  def __init__(self, cin, cout):
    super().__init__()
    self.lin = torch.nn.Linear(cin, cout, bias=False)
    self.bias = torch.nn.Parameter(torch.zeros(cout))

  def forward(self, x, src, dst):
    n = x.shape[0]
    keep = src != dst
    loops = torch.arange(n)
    src, dst = torch.cat([src[keep], loops]), torch.cat([dst[keep], loops])
    deg = torch.zeros(n, dtype=x.dtype).index_add_(0, dst, torch.ones(dst.numel(), dtype=x.dtype))
    norm = deg[src].rsqrt() * deg[dst].rsqrt()
    h = self.lin(x)
    return torch.zeros_like(h).index_add_(0, dst, h[src] * norm[:, None]) + self.bias


class RefDGCNN(torch.nn.Module):
  """The reference example's DGCNN with GCNConv and MLP([dense, 128, 1]) spelled out; same parameter names."""

  def __init__(self, num_features, hidden, num_layers, k):
    super().__init__()
    self.k = k
    self.convs = torch.nn.ModuleList([GCNConv64(num_features, hidden)] +
                                     [GCNConv64(hidden, hidden) for _ in range(num_layers - 1)] +
                                     [GCNConv64(hidden, 1)])
    total = hidden * num_layers + 1
    self.conv1 = torch.nn.Conv1d(1, 16, total, total)
    self.conv2 = torch.nn.Conv1d(16, 32, 5, 1)
    dense = (int((k - 2) / 2 + 1) - 5 + 1) * 32
    self.mlp = torch.nn.Module()
    self.mlp.lins = torch.nn.ModuleList([torch.nn.Linear(dense, 128), torch.nn.Linear(128, 1)])

  def node_features(self, x, src, dst):
    xs = [x]
    for conv in self.convs:
      xs.append(torch.tanh(conv(xs[-1], src, dst)))
    return torch.cat(xs[1:], -1)

  def head(self, pooled, mask):
    h = pooled.reshape(1, 1, -1)
    h = F.max_pool1d(F.relu(self.conv1(h)), 2, 2)
    h = F.relu(self.conv2(h)).reshape(1, -1)
    h = F.relu(self.mlp.lins[0](h)) * mask
    return self.mlp.lins[1](h).reshape(())


def ref_model(eng):
  m = RefDGCNN(eng.max_z + 1, eng.hidden, eng.num_layers, eng.k).double()
  m.load_state_dict({k: v.double().cpu() for k, v in eng.state_dict()['model'].items()})
  return m


def check_sort_pool(key, sel, n, k, tol=1e-5):
  """sel is a top-k of key (descending) up to tol; rows past n are padding."""
  got = [i for i in sel[:min(n, k)]]
  assert sorted(got) == sorted(set(got)) and all(0 <= i < n for i in got)
  assert all(i == -1 for i in sel[min(n, k):])
  vals = key[got]
  assert bool((vals[:-1] >= vals[1:] - tol).all())
  rest = np.setdiff1d(np.arange(n), got)
  if len(rest) and len(got):
    assert key[rest].max() <= vals.min() + tol


def oracle_logits(eng, m, links, mask=None):
  """float64 logits of the reference module on the engine's subgraphs and sort-pool rows (checked to be a top-k)."""
  out = []
  for b in range(links.shape[1]):
    meta, nodes, edges, _, z = engine_subgraph(eng, b)
    if not meta[2]:
      out.append(None)
      continue
    n = meta[0]
    e = torch.tensor(edges, dtype=torch.int64).reshape(-1, 2)
    x = F.one_hot(torch.from_numpy(np.minimum(z, eng.max_z).astype(np.int64)), eng.max_z + 1).double()
    X = m.node_features(x, e[:, 0], e[:, 1])
    sel = eng.arena.sel[b].cpu().tolist()
    check_sort_pool(X[:, -1].detach().numpy(), sel, n, eng.k)
    pooled = torch.zeros(eng.k, X.shape[1], dtype=torch.float64)
    idx = [i for i in sel if i >= 0]
    pooled[:len(idx)] = X[idx]
    mk = torch.ones(128, dtype=torch.float64) if mask is None else mask[b].double().cpu()
    out.append(m.head(pooled, mk))
  return out


def _block_graph(blocks=4, size=40, p_in=0.25, p_out=0.01, seed=0):
  gen = torch.Generator().manual_seed(seed)
  n = blocks * size
  blk = torch.arange(n) // size
  prob = torch.where(blk[:, None] == blk[None, :], p_in, p_out)
  a = torch.rand(n, n, generator=gen) < prob
  a = torch.triu(a, 1)
  a = a | a.t()
  return a.nonzero().t().contiguous(), n


# ------------------------------------------------------------------ 2. forward
# fp32 kernels (fmaf, tanhf) against float64: logits agree to 1e-4 relative + 1e-4 absolute.
@pytest.mark.parametrize('hidden,num_layers,k', [(8, 1, 10), (32, 3, 10), (32, 2, 16), (64, 4, 12), (128, 2, 30)])
def test_forward_matches_float64(hidden, num_layers, k):
  ei, n = _block_graph(seed=hidden)
  g = _graph(ei, n)
  links = torch.cat([ei[:, :20], _links(n, k, 20)], 1)
  eng = SealEngine(g, n, num_hops=1 if hidden == 128 else 2, max_nodes=256, max_edges=8192, hidden=hidden,
                   num_layers=num_layers, sort_k=k, max_z=40, dropout=0.0, batch_size=links.shape[1], seed=hidden)
  logits = eng.predict(links.to(DEV)).cpu()
  m = ref_model(eng)
  ref = oracle_logits(eng, m, links)
  for b, r in enumerate(ref):
    if r is not None:
      assert abs(float(logits[b]) - float(r)) <= 1e-4 + 1e-4 * abs(float(r)), (b, float(logits[b]), float(r))


def test_forward_fewer_exactly_and_more_than_k_nodes():
  # on the path 0 - 1 - ... - 11, the 4-hop subgraphs of (0, 2), (0, 11) and (3, 8) have 7, 10 and 12 nodes; k = 10
  src = torch.arange(11)
  ei = torch.cat([torch.stack([src, src + 1]), torch.stack([src + 1, src])], 1)
  g = _graph(ei, 12)
  links = torch.tensor([[0, 0, 3], [2, 11, 8]])
  eng = SealEngine(g, 12, num_hops=4, max_nodes=64, max_edges=256, hidden=8, num_layers=2, sort_k=10, max_z=30,
                   dropout=0.0, batch_size=3)
  logits = eng.predict(links.to(DEV)).cpu()
  assert eng.arena.meta[:, 0].tolist() == [7, 10, 12]
  for b, r in enumerate(oracle_logits(eng, ref_model(eng), links)):
    assert abs(float(logits[b]) - float(r)) <= 1e-4 + 1e-4 * abs(float(r))


# ------------------------------------------------------------------ 3. backward and Adam
def _grads(eng, links, labels):
  eng._stage(links, eng.links, labels, eng.labels)
  eng._extract(eng.links)
  eng._forward(eng.labels, True)
  eng._backward()
  torch.cuda.synchronize()
  return eng.grad.cpu().clone(), float(eng.loss[0])


@pytest.mark.parametrize('dropout', [0.0, 0.5])
def test_gradient_matches_float64_autograd(dropout):
  ei, n = _block_graph(seed=11)
  g = _graph(ei, n)
  links = torch.cat([ei[:, :12], _links(n, 3, 12)], 1)
  labels = torch.cat([torch.ones(12), torch.zeros(12)])
  eng = SealEngine(g, n, num_hops=2, max_nodes=256, max_edges=8192, hidden=16, num_layers=2, sort_k=12, max_z=40,
                   dropout=dropout, batch_size=links.shape[1], seed=4)
  grad, loss = _grads(eng, links.to(DEV), labels.to(DEV))
  m = ref_model(eng)
  logits = oracle_logits(eng, m, links, mask=eng.mask if dropout else None)
  valid = [b for b, r in enumerate(logits) if r is not None]
  ref_loss = F.binary_cross_entropy_with_logits(torch.stack([logits[b] for b in valid]),
                                                labels[valid].double())
  ref_loss.backward()
  assert abs(loss - float(ref_loss)) <= 1e-5 + 1e-5 * abs(float(ref_loss))
  named = dict(m.named_parameters())
  scale = max(float(p.grad.abs().max()) for p in named.values())
  for name, off, shape in eng.layout:
    ref = named[name].grad.reshape(-1)
    got = grad[off:off + math.prod(shape)].double()
    assert torch.allclose(got, ref, rtol=1e-3, atol=1e-5 * scale), (name, float((got - ref).abs().max()))


def test_adam_step_matches_torch():
  ei, n = _block_graph(seed=12)
  g = _graph(ei, n)
  links = torch.cat([ei[:, :8], _links(n, 5, 8)], 1).to(DEV)
  labels = torch.cat([torch.ones(8), torch.zeros(8)]).to(DEV)
  eng = SealEngine(g, n, num_hops=1, max_nodes=128, max_edges=4096, hidden=8, num_layers=2, sort_k=10, max_z=20,
                   dropout=0.0, batch_size=16, lr=1e-2, use_cuda_graph=False)
  p = torch.nn.Parameter(eng.params.cpu().clone())
  opt = torch.optim.Adam([p], lr=1e-2)
  for _ in range(3):
    grad, _ = _grads(eng, links, labels)
    eng._update()
    p.grad = grad
    opt.step()
  torch.testing.assert_close(eng.params.cpu(), p.detach(), rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------ 4. runtime
def _train_setup(use_cuda_graph, seed=0, dropout=0.5):
  ei, n = _block_graph(seed=21)
  g = _graph(ei, n)
  eng = SealEngine(g, n, num_hops=2, num_neighbors=[8, 4], max_nodes=128, hidden=16, num_layers=2, sort_k=0.6,
                   dropout=dropout, batch_size=32, lr=1e-3, calibration_links=ei[:, :200], seed=seed,
                   use_cuda_graph=use_cuda_graph)
  eng.warmup_and_capture()
  gen = torch.Generator().manual_seed(1)
  batches = []
  for _ in range(4):
    pos = ei[:, torch.randint(0, ei.shape[1], (16,), generator=gen)]
    neg = torch.randint(0, n, (2, 16), generator=gen)
    batches.append((torch.cat([pos, neg], 1).to(DEV), torch.cat([torch.ones(16), torch.zeros(16)]).to(DEV)))
  return eng, batches


def test_captured_steps_equal_eager_bitwise():
  a, batches = _train_setup(True)
  b, _ = _train_setup(False)
  for links, labels in batches:
    la, lb = a.train_step(links, labels), b.train_step(links, labels)
    assert torch.equal(la, lb)
  assert torch.equal(a.params, b.params)
  assert torch.equal(a.exp_avg_sq, b.exp_avg_sq)


def test_state_dict_round_trip_resumes_the_same_draws():
  a, batches = _train_setup(True)
  for links, labels in batches[:2]:
    a.train_step(links, labels)
  sd = a.state_dict()
  for links, labels in batches[2:]:
    a.train_step(links, labels)
  b, _ = _train_setup(True)
  b.load_state_dict(sd)
  for links, labels in batches[2:]:
    b.train_step(links, labels)
  assert torch.equal(a.params, b.params)
  assert torch.equal(a.mask, b.mask)


def test_padding_and_invalid_links_add_nothing():
  ei, n = _block_graph(seed=13)
  g = _graph(ei, n)
  links = torch.cat([ei[:, :6], _links(n, 8, 6)], 1)
  labels = torch.cat([torch.ones(6), torch.zeros(6)])
  bad = torch.tensor([[-1, 3, n, 2], [4, 3, 1, n + 5]])
  mixed = torch.cat([links[:, :5], bad, links[:, 5:]], 1)
  mixed_labels = torch.cat([labels[:5], torch.tensor([1., 0., 1., 1.]), labels[5:]])
  kw = dict(num_hops=2, max_nodes=128, max_edges=4096, hidden=8, num_layers=2, sort_k=10, max_z=30, dropout=0.0,
            batch_size=20)
  e1 = SealEngine(g, n, **kw)
  e2 = SealEngine(g, n, **kw)
  g1, l1 = _grads(e1, links.to(DEV), labels.to(DEV))
  g2, l2 = _grads(e2, mixed.to(DEV), mixed_labels.to(DEV))
  assert torch.equal(g1, g2) and l1 == l2
  assert int(e2.arena.meta[:, 2].sum()) == 12


def test_predict_equals_the_no_dropout_forward():
  a, batches = _train_setup(False)
  links, labels = batches[0]
  a.train_step(links, labels)
  p = a.predict(links)
  a._stage(links, a.links, labels, a.labels)
  a._extract(a.links)
  a._forward(a.labels, False)
  assert torch.equal(p, a.arena.logits[:links.shape[1]])
  assert bool((a.mask == 1).all())


# ------------------------------------------------------------------ 5. learns
def _auc(pos, neg):
  s = torch.cat([pos, neg]).double()
  r = s.argsort().argsort().double() + 1
  return float((r[:pos.numel()].sum() - pos.numel() * (pos.numel() + 1) / 2) / (pos.numel() * neg.numel()))


def test_learns_a_planted_block_graph():
  ei, n = _block_graph(blocks=4, size=50, p_in=0.2, p_out=0.01, seed=31)
  und = ei[:, ei[0] < ei[1]]
  gen = torch.Generator().manual_seed(2)
  und = und[:, torch.randperm(und.shape[1], generator=gen)]
  held, train = und[:, :100], und[:, 100:]
  train_ei = torch.cat([train, train.flip(0)], 1)
  neg = torch.randint(0, n, (2, 100), generator=gen)
  # held-out links are structurally predictable: common-neighbour AUC on the training graph
  a = torch.zeros(n, n)
  a[train_ei[0], train_ei[1]] = 1
  cn = lambda l: (a[l[0]] * a[l[1]]).sum(1)
  cn_auc = _auc(cn(held), cn(neg))
  assert cn_auc > 0.75
  g = _graph(train_ei, n)
  eng = SealEngine(g, n, num_hops=1, max_nodes=256, hidden=32, num_layers=3, sort_k=0.6, dropout=0.5, batch_size=64,
                   lr=1e-3, calibration_links=train, seed=0)
  eng.warmup_and_capture()
  for step in range(200):
    pos = train[:, torch.randint(0, train.shape[1], (32,), generator=gen)]
    ng = torch.randint(0, n, (2, 32), generator=gen)
    eng.train_step(torch.cat([pos, ng], 1).to(DEV), torch.cat([torch.ones(32), torch.zeros(32)]).to(DEV))
  auc = _auc(eng.predict(held.to(DEV)).cpu(), eng.predict(neg.to(DEV)).cpu())
  print(f'common-neighbour AUC {cn_auc:.3f}, engine AUC {auc:.3f}')
  # the first H100 run gave 0.829 (common neighbours: 0.767); 0.75 leaves a margin and is far above chance
  assert auc > 0.75


# ------------------------------------------------------------------ 6. errors
def test_constructor_errors():
  ei, n = _block_graph(seed=1)
  g = _graph(ei, n)
  cpu = glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=n), 'CPU')
  base = dict(max_edges=1024, max_z=20, sort_k=10)
  bad = [dict(graph=cpu), dict(num_hops=0), dict(num_hops=5), dict(num_neighbors=[3]), dict(max_nodes=1),
         dict(max_nodes=2048), dict(max_edges=0), dict(hidden=0), dict(num_layers=9), dict(sort_k=5),
         dict(sort_k=1.5), dict(sort_k=True), dict(max_z=0), dict(dropout=1.0), dict(batch_size=0), dict(lr=0.0),
         dict(num_neighbors=[2000, 2], max_nodes=1024), dict(max_edges=None), dict(num_nodes=0)]
  for kw in bad:
    args = {**base, **kw}
    graph = args.pop('graph', g)
    nn_ = args.pop('num_nodes', n)
    with pytest.raises(ValueError):
      SealEngine(graph, nn_, **args)
  with pytest.raises(ValueError):
    SealEngine(g, n, hidden=256, num_layers=8, max_nodes=1024, sort_k=2048, max_edges=64, max_z=20)   # shared memory


def test_binding_errors():
  ei, n = _block_graph(seed=1)
  g = _graph(ei, n)
  eng = SealEngine(g, n, num_hops=1, max_nodes=64, max_edges=1024, hidden=8, num_layers=1, sort_k=10, max_z=20,
                   batch_size=4)
  A, h = eng.arena, g.graph_handler
  good = torch.zeros(2, 4, dtype=torch.int64, device=DEV)
  call = lambda links, **kw: A.extract(h, links, n, kw.get('hops', 1), kw.get('caps', [0]), 0, eng.state, 20,
                                       eng.trunc)
  call(good)
  for links in (good.int(), good[:, :3].contiguous(), good.cpu(), good.t().contiguous()):
    with pytest.raises(RuntimeError):
      call(links)
  with pytest.raises(RuntimeError):
    call(good, hops=5, caps=[0] * 5)
  with pytest.raises(RuntimeError):
    call(good, caps=[5])                                           # above the arena's cap_max
  with pytest.raises(RuntimeError):
    A.forward(eng.params[:-1], eng.labels, True, 0.0, 0, eng.state)
  with pytest.raises(RuntimeError):
    A.forward(eng.params.double(), eng.labels, True, 0.0, 0, eng.state)
  with pytest.raises(RuntimeError):
    A.forward(eng.params, eng.labels, True, 1.0, 0, eng.state)
  with pytest.raises(RuntimeError):
    A.backward(eng.params.cpu())
  with pytest.raises(RuntimeError):
    A.reduce(eng.grad, torch.zeros(2, device=DEV))
  for kw in (dict(max_nodes=2000), dict(max_nodes=1), dict(k=9), dict(num_layers=0), dict(hidden=300)):
    args = dict(device=0, batch_size=4, max_nodes=64, max_edges=64, hidden=8, num_layers=1, num_labels=4, k=10)
    args.update(kw)
    with pytest.raises(RuntimeError):
      type(A)(**args)
  torch.cuda.synchronize()


# ------------------------------------------------------------------ 7. example
def test_example_engine_mode_runs():
  r = subprocess.run([sys.executable, 'seal_link_pred.py', '--mode', 'engine', '--links', '400', '--epochs', '2'],
                     cwd=os.path.join(ROOT, 'examples'), capture_output=True, text=True, timeout=600)
  assert r.returncode == 0, r.stderr[-2000:]
  assert 'test AUC' in r.stdout
