"""Full-neighbourhood layer-wise inference of the heterogeneous engines (HeteroSageEngine / HeteroGatEngine /
HeteroHgtEngine.inference) and its kernels (csrc/cuda/hetero_infer.cu, the mean-only mode of sage_full_aggregate).

Engines: against fp32 PyTorch recomputations over the complete CSR of every relation with the engines' bf16 rounding
points, on a three-type schema with a same-type relation, source types of different widths, a paper cited 5200 times
and papers without any in-neighbour; determinism and chunk invariance; the fanout >= degree limit of evaluate_batch;
an engine trained through CUDA-graph replays left untouched; HBM vs HBM-plus-pinned-host feature tables.
Kernels: against float64 at heads 1 to 8 and H 64 to 1024, rows of degree 0, 1 and k and hubs, scores near 100.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import HeteroGatEngine, HeteroHgtEngine, HeteroSageEngine

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
SIZES = {'paper': 3000, 'author': 1500, 'inst': 200}
DIMS = {'paper': 128, 'author': 64, 'inst': 64}
HUB, N_ISO = 7, 100                     # paper HUB is cited 5200 times; the last N_ISO papers have no in-neighbour
CLASSES = 19
ENGINES = {'rsage': HeteroSageEngine, 'rgat': HeteroGatEngine, 'hgt': HeteroHgtEngine}


# --------------------------------------------------------------------------- schema
def _rand_edges(g, n_src, n_dst, m, dst_hi=None):
  return torch.stack([torch.randint(0, n_src, (m,), generator=g), torch.randint(0, dst_hi or n_dst, (m,), generator=g)])


def _schema_edges(seed=0):
  g = torch.Generator().manual_seed(seed)
  P, A, I = SIZES['paper'], SIZES['author'], SIZES['inst']
  live = P - N_ISO
  cites = _rand_edges(g, P, P, 12000, live)
  hub = torch.stack([torch.randint(0, P, (5200,), generator=g), torch.full((5200,), HUB, dtype=torch.int64)])
  writes = _rand_edges(g, A, P, 6000, live)
  return {('paper', 'cites', 'paper'): torch.cat([cites, hub], 1),
          ('author', 'writes', 'paper'): writes,
          ('paper', 'rev_writes', 'author'): writes.flip(0),
          ('inst', 'employs', 'author'): _rand_edges(g, I, A, 2000),
          ('inst', 'hosts', 'paper'): _rand_edges(g, I, P, 3000, live),
          ('author', 'affiliated_with', 'inst'): _rand_edges(g, A, I, 2000)}


def _small_degree_edges(seed=1, max_deg=6):
  """Every relation: unique edges, in-degree <= max_deg."""
  out = {}
  for et, ei in _schema_edges(seed).items():
    ei = ei[:, ~((ei[0] == ei[1]) & (et[0] == et[2]))]
    ei = torch.unique(ei, dim=1)
    n_dst = SIZES[et[2]]
    order = torch.argsort(ei[1], stable=True)
    ei = ei[:, order]
    first = torch.searchsorted(ei[1], ei[1])
    out[et] = ei[:, (torch.arange(ei.shape[1]) - first) < max_deg]
    assert int(torch.bincount(out[et][1], minlength=n_dst).max()) <= max_deg
  return out


class _Data:
  def __init__(self, edges, split_host=False, seed=3):
    self.edges = edges
    self.graphs, self.topos, self.tables, self.keep = {}, {}, {}, []
    for et, ei in edges.items():
      topo = glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=SIZES[et[2]])
      self.topos[et] = topo
      self.graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
    g = torch.Generator().manual_seed(seed)
    self.feats = {t: torch.randn(SIZES[t], DIMS[t], generator=g).to(torch.bfloat16).to(DEV) for t in SIZES}
    for t, x in self.feats.items():
      ut = glt.data.UnifiedTensor(0, torch.bfloat16)
      if split_host:
        ut.append_shared_tensor(x[:SIZES[t] // 3])
        ut.append_cpu_tensor(x[SIZES[t] // 3:].cpu())
      else:
        ut.append_shared_tensor(x)
      self.tables[t] = ut._table()
      self.keep.append(ut)
    self.labels = torch.randint(0, CLASSES, (SIZES['paper'],), generator=g).to(DEV)

  def csr(self, et):
    """(dst, src) of every edge of a relation, in CSR order."""
    topo = self.topos[et]
    indptr, indices = topo.indptr.to(DEV), topo.indices.to(DEV)
    dst = torch.repeat_interleave(torch.arange(indptr.numel() - 1, device=DEV), indptr[1:] - indptr[:-1])
    return dst, indices.long()


def _engine(kind, data, fan=(4, 3), train_steps=3, use_graph=False, **kw):
  args = dict(fanouts=list(fan), batch_size=256, hidden=128, num_classes=CLASSES, edge_dir='in', lr=5e-3, seed=1,
              device=DEV, use_cuda_graph=use_graph)
  if kind != 'rsage':
    args['heads'] = 4
  if kind == 'rgat':
    args['dropout'] = 0.2
  args.update(kw)
  eng = ENGINES[kind](data.graphs, data.tables, data.labels, dict(DIMS), dict(SIZES), 'paper', **args)
  eng._keep = data
  if use_graph:
    eng.warmup_and_capture(n_eager=1)
  gen = torch.Generator().manual_seed(9)
  for _ in range(train_steps):
    eng.train_step(torch.randperm(SIZES['paper'], generator=gen)[:256].to(DEV))
  torch.cuda.synchronize()
  return eng


# --------------------------------------------------------------------------- fp32 references over the full CSR
def bf(x):
  return x.to(torch.bfloat16).float()


def _seg_softmax(e, dst, n):
  heads = e.shape[1]
  m = torch.full((n, heads), -float('inf'), device=DEV, dtype=e.dtype).scatter_reduce(
      0, dst.unsqueeze(1).expand(-1, heads), e, 'amax', include_self=True)
  ex = torch.exp(e - m[dst])
  den = torch.zeros(n, heads, device=DEV, dtype=e.dtype).index_add_(0, dst, ex)
  return ex / den[dst]


def _ref_rsage(eng, data):
  X = {t: data.feats[eng.ntypes[t]].float() for t in range(len(eng.ntypes))}
  for l in range(1, eng.L + 1):
    Z = {}
    for t in eng.targets[l]:
      n = SIZES[eng.ntypes[t]]
      blocks = []
      for r in eng.in_rel[l][t]:
        dst, src = data.csr(eng.edge_types[r])
        deg = torch.bincount(dst, minlength=n).clamp(min=1).unsqueeze(1).float()
        blocks.append(torch.zeros(n, X[eng.nt[r]].shape[1], device=DEV).index_add_(0, dst, X[eng.nt[r]][src]) / deg)
      A = bf(torch.cat(blocks + [X[t]], 1))
      z = A @ eng.param(('W', l, t)).float().t() + eng.param(('b', l, t)).float()
      Z[t] = bf(F.relu(z) if l < eng.L else z)
    X = Z
  return X[eng.tid['paper']][:, :eng.C]


def _ref_rgat(eng, data):
  H, hd = eng.hidden, eng.heads
  C = H // hd
  p = lambda *k: eng.param(k).float()    # noqa: E731
  X = {t: data.feats[eng.ntypes[t]].float() for t in range(len(eng.ntypes))}
  for l in range(1, eng.L + 1):
    Z = {}
    for t in eng.targets[l]:
      n = SIZES[eng.ntypes[t]]
      pre = torch.zeros(n, H, device=DEV)
      for r in eng.in_rel[l][t]:
        s = eng.nt[r]
        dst, src = data.csr(eng.edge_types[r])
        hs = bf(X[s] @ p('W_src', l, r).t())
        gd = bf(X[t] @ eng._w_dst(l, r).float().t())
        a_s = (hs.view(-1, hd, C) * p('att_src', l, r).view(hd, C)).sum(-1)
        a_d = (gd.view(-1, hd, C) * p('att_dst', l, r).view(hd, C)).sum(-1)
        al = _seg_softmax(F.leaky_relu(a_s[src] + a_d[dst], 0.2), dst, n)
        pre += torch.zeros(n, H, device=DEV).index_add_(0, dst, (al.unsqueeze(-1) * hs[src].view(-1, hd, C)).view(-1, H))
        pre += p('bias', l, r)
      Z[t] = bf(F.leaky_relu(pre, 0.01) if l < eng.L else pre)
    X = Z
  st = eng.tid['paper']
  return bf(X[st] @ p('head_W').t() + p('head_b'))[:, :eng.C]


def _ref_hgt(eng, data):
  H, hd = eng.hidden, eng.heads
  D = H // hd
  p = lambda *k: eng.param(k).float()    # noqa: E731
  X = {u: bf(F.relu(data.feats[eng.ntypes[u]].float() @ p('in_W', u).t() + p('in_b', u))) for u in eng.in_types}
  for l in range(1, eng.L + 1):
    KQV = {u: bf(X[u] @ p('kqv_W', l, u).t() + p('kqv_b', l, u)) for u in eng.kqv_types[l]}
    Z = {}
    for t in eng.targets[l]:
      n = SIZES[eng.ntypes[t]]
      rels = eng.in_rel[l][t]
      Q = KQV[t][:, H:2 * H]
      scores, dsts, vals = [], [], []
      for r in rels:
        dst, src = data.csr(eng.edge_types[r])
        W_att = p('att', l, r)
        qq = bf(Q @ torch.block_diag(*W_att).t())
        k = KQV[eng.nt[r]][:, :H]
        sc = (qq[dst].view(-1, hd, D) * k[src].view(-1, hd, D)).sum(-1) * eng._p32(('prior', l, r)).float() / math.sqrt(D)
        scores.append(sc); dsts.append(dst); vals.append(KQV[eng.nt[r]][src, 2 * H:])
      al = _seg_softmax(torch.cat(scores), torch.cat(dsts), n).split([s.shape[0] for s in scores])
      agg = torch.zeros(n, H, device=DEV)
      for r, a, dst, v in zip(rels, al, dsts, vals):
        u = bf(torch.zeros(n, H, device=DEV).index_add_(0, dst, (a.unsqueeze(-1) * v.view(-1, hd, D)).view(-1, H)))
        agg += u @ torch.block_diag(*p('msg', l, r))
      ge = bf(F.gelu(bf(agg)))
      a_ = bf(ge @ p('a_W', l, t).t() + p('a_b', l, t))
      g = torch.sigmoid(eng._p32(('skip', l, t)).float())
      Z[t] = bf(g * a_ + (1 - g) * X[t])
    X = Z
  st = eng.tid['paper']
  return bf(X[st] @ p('head_W').t() + p('head_b'))[:, :eng.C]


REFS = {'rsage': _ref_rsage, 'rgat': _ref_rgat, 'hgt': _ref_hgt}


def _check_close(got, ref):
  assert got.shape == ref.shape and got.dtype == torch.bfloat16
  torch.testing.assert_close(got.float(), ref, rtol=2e-2, atol=2e-2)
  agree = (got.float().argmax(1) == ref.argmax(1)).float().mean().item()
  assert agree >= 0.99, agree


@pytest.fixture(scope='module')
def data():
  return _Data(_schema_edges())


@pytest.fixture(scope='module', params=list(ENGINES))
def trained(request, data):
  return request.param, _engine(request.param, data)


# --------------------------------------------------------------------------- engines
def test_inference_matches_fp32_reference(native, data, trained):
  kind, eng = trained
  deg = torch.bincount(data.csr(('paper', 'cites', 'paper'))[0], minlength=SIZES['paper'])
  assert int(deg[HUB]) >= 5000 and int(deg[-N_ISO:].sum()) == 0
  got = eng.inference()
  assert got.shape == (SIZES['paper'], CLASSES)
  _check_close(got, REFS[kind](eng, data))


def test_inference_is_deterministic_and_independent_of_chunking(native, trained):
  _, eng = trained
  a = eng.inference()
  assert torch.equal(a, eng.inference())
  assert torch.equal(a, eng.inference(chunk_rows=997))


@pytest.mark.parametrize('kind', list(ENGINES))
def test_inference_is_the_full_fanout_limit_of_evaluate_batch(native, kind):
  eng = _engine(kind, _Data(_small_degree_edges()), fan=(6, 6), train_steps=2)
  full = eng.inference()
  seeds = torch.randperm(SIZES['paper'], device=DEV)[:256]
  eng.evaluate_batch(seeds)
  sampled = (eng.Z[eng.L][eng.tid['paper']] if kind == 'rsage' else eng.logits)[:256, :eng.C]
  torch.testing.assert_close(sampled.float(), full[seeds].float(), rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize('kind', list(ENGINES))
def test_inference_leaves_a_captured_engine_untouched(native, data, kind):
  eng = _engine(kind, data, train_steps=4, use_graph=True)
  snap = {k: getattr(eng, k).clone() for k in ('p32', 'p16', 'm', 'v', 'g32', 'step_dev')}
  step, graph = eng.arena.step.clone(), eng._graph
  eng.inference(chunk_rows=1000)
  torch.cuda.synchronize()
  for k, v in snap.items():
    assert torch.equal(getattr(eng, k), v), k
  assert torch.equal(eng.arena.step, step) and eng._graph is graph
  loss = eng.train_step(torch.randperm(SIZES['paper'], device=DEV)[:256])
  assert torch.isfinite(loss).all()


@pytest.mark.parametrize('kind', list(ENGINES))
def test_inference_is_identical_across_feature_memory_tiers(native, kind):
  edges = _schema_edges()
  ref = _engine(kind, _Data(edges), train_steps=0).inference()
  assert torch.equal(_engine(kind, _Data(edges, split_host=True), train_steps=0).inference(), ref)


# --------------------------------------------------------------------------- kernels against float64
def _kernel_graph(n_dst, n_src, seed, hub_deg=600):
  """CSR rows: 0 (degree 0), 1 (degree 1), 2 (degree 40), 3 (a hub of hub_deg, repeated ids), the rest random <= 12;
  rows n_dst - 20 .. n_dst - 1 have no neighbours."""
  g = torch.Generator().manual_seed(seed)
  deg = torch.randint(0, 13, (n_dst,), generator=g)
  deg[:4] = torch.tensor([0, 1, 40, hub_deg])
  deg[-20:] = 0
  dst = torch.repeat_interleave(torch.arange(n_dst), deg)
  src = torch.randint(0, n_src, (int(deg.sum()),), generator=g)
  topo = glt.data.Topology(torch.stack([src, dst]).to(DEV), layout='CSC', num_nodes=n_dst)
  graph = glt.data.Graph(topo, 'CUDA', 0)
  graph._keep = topo
  indptr = topo.indptr.to(DEV)
  d = torch.repeat_interleave(torch.arange(n_dst, device=DEV), indptr[1:] - indptr[:-1])
  return graph, d, topo.indices.to(DEV).long()


# (heads, C): H = heads * C from 64 to 1024; 64 and 128 heads give each lane of a row several heads
SHAPES = [(1, 64), (2, 64), (4, 48), (8, 8), (1, 256), (8, 128), (4, 256), (16, 8), (32, 16), (64, 8), (128, 8)]


@pytest.mark.parametrize('scores', ['normal', 'large'])
@pytest.mark.parametrize('heads,C', SHAPES)
def test_gat_full_aggregate_matches_fp64(native, heads, C, scores):
  H = heads * C
  n_src, n_dst = 700, 300
  g = torch.Generator().manual_seed(H + heads)
  graphs = [_kernel_graph(n_dst, n_src, H + i, hub_deg=600 if i == 0 else 5000) for i in range(2)]
  P = [torch.randn(n_src, H, generator=g).to(torch.bfloat16).to(DEV) for _ in range(2)]
  sc = 100.0 / 3 if scores == 'large' else 1.0       # |score| up to ~100: an unshifted exp overflows fp32
  as_ = [(torch.randn(n_src, heads, generator=g) * sc).to(DEV) for _ in range(2)]
  ad = [(torch.randn(n_dst, heads, generator=g) * sc).to(DEV) for _ in range(2)]
  bias = torch.randn(2 * H, generator=g).to(torch.bfloat16).to(DEV)
  r0, r1 = 0, n_dst
  acc = torch.full((r1 - r0, H), 7.0, device=DEV)
  Z = torch.full((r1 - r0, H), 9.0, dtype=torch.bfloat16, device=DEV)
  for j in range(2):
    native.gat_full_aggregate(graphs[j][0].graph_handler, P[j], as_[j], ad[j], heads, r0, r1, acc=acc, first=j == 0,
                              last=j == 1, bias=bias if j == 1 else None, act=True, Z=Z if j == 1 else None)
  torch.cuda.synchronize()
  pre = bias.double().view(2, H).sum(0).expand(n_dst, H).clone()
  for j in range(2):
    _, dst, src = graphs[j]
    e = F.leaky_relu(as_[j].double()[src] + ad[j].double()[dst], 0.2)
    al = _seg_softmax(e, dst, n_dst)
    pre += torch.zeros(n_dst, H, dtype=torch.float64, device=DEV).index_add_(
        0, dst, (al.unsqueeze(-1) * P[j].double()[src].view(-1, heads, C)).view(-1, H))
  ref = F.leaky_relu(pre, 0.01)
  torch.testing.assert_close(Z.double(), ref, rtol=1e-2, atol=1e-2)
  assert torch.isfinite(Z.float()).all()
  # a degree-0 row (in both relations) is the bias only; chunking and repetition do not change a bit
  assert torch.equal(Z[-1].float(), bf(F.leaky_relu(bias.float().view(2, H).sum(0), 0.01)))
  Z2 = torch.empty_like(Z)
  for c0 in range(0, n_dst, 97):
    c1 = min(n_dst, c0 + 97)
    a2 = torch.empty(c1 - c0, H, device=DEV)
    for j in range(2):
      native.gat_full_aggregate(graphs[j][0].graph_handler, P[j], as_[j], ad[j], heads, c0, c1, acc=a2, first=j == 0,
                                last=j == 1, bias=bias if j == 1 else None, act=True, Z=Z2[c0:c1] if j == 1 else None)
  assert torch.equal(Z, Z2)


@pytest.mark.parametrize('scores', ['normal', 'large'])
@pytest.mark.parametrize('heads,D', SHAPES)
def test_hgt_full_attention_matches_fp64(native, heads, D, scores):
  H = heads * D
  n_dst, R = 300, 3
  n_src = [700, 300, 50]
  g = torch.Generator().manual_seed(H * 3 + heads)
  graphs = [_kernel_graph(n_dst, n_src[r], H + 7 * r, hub_deg=[100, 5000, 200][r]) for r in range(R)]
  kv = [torch.randn(n_src[r], 3 * H, generator=g).to(torch.bfloat16).to(DEV) for r in range(R)]
  sc = 100.0 if scores == 'large' else 1.0
  qq = (torch.randn(n_dst, R * H, generator=g) * (sc / math.sqrt(D))).to(torch.bfloat16).to(DEV)
  prior = [(torch.rand(heads, generator=g) + 0.5).to(DEV) for _ in range(R)]
  u = torch.full((n_dst, R * H), 9.0, dtype=torch.bfloat16, device=DEV)
  native.hgt_full_attention([gr[0].graph_handler for gr in graphs], qq, u, heads, 0, n_dst, kv, prior)
  torch.cuda.synchronize()
  scores_, dsts = [], []
  for r in range(R):
    _, dst, src = graphs[r]
    s = (qq.double()[:, r * H:(r + 1) * H][dst].view(-1, heads, D) * kv[r].double()[src, :H].view(-1, heads, D)).sum(-1)
    scores_.append(s * prior[r].double() / math.sqrt(D)); dsts.append(dst)
  al = _seg_softmax(torch.cat(scores_), torch.cat(dsts), n_dst).split([s.shape[0] for s in scores_])
  for r in range(R):
    _, dst, src = graphs[r]
    ref = torch.zeros(n_dst, H, dtype=torch.float64, device=DEV).index_add_(
        0, dst, (al[r].unsqueeze(-1) * kv[r].double()[src, 2 * H:].view(-1, heads, D)).view(-1, H))
    torch.testing.assert_close(u[:, r * H:(r + 1) * H].double(), ref, rtol=1e-2, atol=1e-2)
  assert bool((u[-20:] == 0).all()), 'a row without neighbours gets u = 0'
  u2 = torch.empty_like(u)
  for c0 in range(0, n_dst, 61):
    c1 = min(n_dst, c0 + 61)
    native.hgt_full_attention([gr[0].graph_handler for gr in graphs], qq[c0:c1], u2[c0:c1], heads, c0, c1, kv, prior)
  assert torch.equal(u, u2)


@pytest.mark.parametrize('d', [64, 128, 512])
def test_full_aggregate_mean_only_block(native, d):
  n_src, n_dst = 700, 300
  graph, dst, src = _kernel_graph(n_dst, n_src, d, hub_deg=5000)
  x = torch.randn(n_src, d, device=DEV).to(torch.bfloat16)
  out = torch.full((n_dst - 5, d + 128), 3.0, dtype=torch.bfloat16, device=DEV)
  native.sage_full_aggregate(graph.graph_handler, None, x, 0, 0, d, 5, n_dst, False, None, False, out[:, 64:64 + d],
                             mean_only=True)
  deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).unsqueeze(1).double()
  mean = (torch.zeros(n_dst, d, dtype=torch.float64, device=DEV).index_add_(0, dst, x.double()[src]) / deg)[5:]
  torch.testing.assert_close(out[:, 64:64 + d].double(), mean, rtol=1e-2, atol=1e-2)
  assert bool((out[:, :64] == 3).all() and (out[:, 64 + d:] == 3).all()), 'only the mean block is written'
  assert bool((out[-20:, 64:64 + d] == 0).all())


def test_full_attention_kernels_reject_unsupported_widths(native):
  graph, _, _ = _kernel_graph(50, 50, 0)
  gh = graph.graph_handler
  for H, heads in ((96, 1), (2048, 8), (128, 3), (128, 32)):
    P = torch.zeros(50, H, dtype=torch.bfloat16, device=DEV)
    s = torch.zeros(50, heads, device=DEV)
    with pytest.raises(RuntimeError, match='multiple of 64|heads'):
      native.gat_full_aggregate(gh, P, s, s, heads, 0, 50, Z=torch.zeros(50, H, dtype=torch.bfloat16, device=DEV))
    with pytest.raises(RuntimeError, match='multiple of 64|heads'):
      native.hgt_full_attention([gh], P, torch.zeros_like(P), heads, 0, 50,
                                [torch.zeros(50, 3 * H, dtype=torch.bfloat16, device=DEV)],
                                [torch.ones(heads, device=DEV)])
  with pytest.raises(RuntimeError, match='1 to 8 relations'):
    native.hgt_full_attention([gh] * 9, torch.zeros(50, 9 * 64, dtype=torch.bfloat16, device=DEV),
                              torch.zeros(50, 9 * 64, dtype=torch.bfloat16, device=DEV), 1, 0, 50,
                              [torch.zeros(50, 192, dtype=torch.bfloat16, device=DEV)] * 9, [torch.ones(1, device=DEV)] * 9)
