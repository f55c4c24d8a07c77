"""SealEngine's step kernels (csrc/cuda/seal.cu) stage by stage against float64.

Each forward stage is recomputed in float64 from the kernel's own fp32 output of the stage before it, so errors do not
compound and a failure names the stage: every GCN layer, the sort-pool rows (exactly), conv1, maxpool + conv2, the MLP,
the logit and the loss term.  Each valid link's row of gradient partials is compared with float64 autograd of that
link's loss term, and the reduced gradient and loss with a sequential fp32 sum of the valid links in link order.

The cases cover every range the engine accepts: hidden 1 to the largest the device's shared memory admits, 1 to 8
layers, odd k and k above max_nodes, 1 to 4 hops, clamped and unclamped labels; on subgraphs wider than the CTA (up to
1,024 nodes, with in-degrees in the hundreds), directed graphs, self-loops and duplicate edges, isolated endpoints and
endpoints in different components, exactly tied sort keys, and batches wider than the CTA with padding interleaved.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from graphlearn_for_pytorch_b200.models import SealEngine
from helpers import bound_ratio
from test_gpu_seal_engine import _graph, engine_subgraph, oracle_extract, ref_model

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
F64 = torch.float64
EPS = 2.0 ** -23            # twice fp32's unit roundoff: a margin for rounding the products and the terms themselves
GRAD_ATOL, GRAD_RTOL = 1e-4, 1e-3


# --------------------------------------------------------------------------- error bounds
def fp32_sum_bound(m, abs_sum):
  """Largest error of an fp32 sum of m terms (fmaf chain or tree, any order) whose magnitudes add to abs_sum:
  m * 2^-23 * abs_sum, twice the first-order bound m * u."""
  return m * EPS * abs_sum


def tanh_bound(pre_bound, y):
  """Error of tanhf(pre) when pre carries pre_bound: |tanh'| <= 1, plus tanhf's own 2 ulp (no fast-math in the build)."""
  return pre_bound + 2 * EPS * y.abs() + 2.0 ** -140


def grad_tol(ref):
  """Tolerance of an fp32 gradient partial against float64 autograd at the same forward point: GRAD_ATOL of the
  tensor's largest entry plus GRAD_RTOL of the entry."""
  return GRAD_ATOL * ref.abs().max() + GRAD_RTOL * ref.abs()


# --------------------------------------------------------------------------- the shared-memory envelope
def seal_smem_floats(hidden, num_layers, k, max_nodes):
  """seal_smem() of seal.cu: (forward, backward) dynamic shared memory of the per-link kernels, in floats."""
  total, kp = hidden * num_layers + 1, k // 2
  dense = (kp - 4) * 32
  stage = max(hidden * hidden, 16 * total, 32 * 16 * 5)
  fwd = stage + max_nodes + (k + max_nodes) + 128 + 16 * kp
  return fwd, fwd + dense + 16 * kp + 16 * k


def seal_extract_smem(max_nodes):
  """seal_extract_smem() of seal.cu, in bytes."""
  hs = 1
  while hs < 2 * (max_nodes + 256):
    hs <<= 1
  return hs * 12 + max_nodes * 8 + 3 * (max_nodes + 1) * 4 + 2 * max_nodes * 2


def seal_smem_bytes(hidden, num_layers, k, max_nodes):
  return max(seal_extract_smem(max_nodes), 4 * max(seal_smem_floats(hidden, num_layers, k, max_nodes)))


def optin_smem():
  return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def largest_hidden(num_layers, k, max_nodes, limit):
  return max(h for h in range(1, 257) if seal_smem_bytes(h, num_layers, k, max_nodes) <= limit)


def largest_k(hidden, num_layers, max_nodes, limit):
  return max(k for k in range(10, 2049) if seal_smem_bytes(hidden, num_layers, k, max_nodes) <= limit)


# --------------------------------------------------------------------------- graphs
def _sym(ei):
  return torch.cat([ei, ei.flip(0)], 1)


def wide_graph():
  """3,000 nodes of average degree ~12 and a hub joined to 600 of them: 2-hop subgraphs of about 200 to over 1,024 nodes;
  where the hub is an endpoint or a first-hop node its in-degree inside the subgraph is in the hundreds."""
  gen = torch.Generator().manual_seed(5)
  n = 3000
  ei = torch.randint(1, n, (2, 18000), generator=gen)
  hub = torch.stack([torch.zeros(600, dtype=torch.int64), torch.randperm(n - 1, generator=gen)[:600] + 1])
  ei = torch.cat([ei, hub], 1)
  ei = ei[:, ei[0] != ei[1]]
  return _sym(torch.unique(ei, dim=1)), n


def directed_graph():
  """Random directed edges: rows are asymmetric, so the source and destination CSRs of a subgraph differ."""
  gen = torch.Generator().manual_seed(6)
  n = 120
  ei = torch.randint(0, n, (2, 700), generator=gen)
  return torch.unique(ei[:, ei[0] != ei[1]], dim=1), n


def loops_graph():
  """Symmetric random graph with a self-loop on every third node (two on every ninth) and 60 duplicated edges."""
  gen = torch.Generator().manual_seed(7)
  n = 100
  ei = torch.randint(0, n, (2, 300), generator=gen)
  ei = _sym(torch.unique(ei[:, ei[0] != ei[1]], dim=1))
  loops = torch.arange(0, n, 3)
  loops = torch.cat([loops, torch.arange(0, n, 9)])
  dup = ei[:, torch.randperm(ei.shape[1], generator=gen)[:60]]
  return torch.cat([ei, torch.stack([loops, loops]), dup], 1), n


def degenerate_graph():
  """Two components (0..39 and 40..79) and isolated nodes 80..89."""
  gen = torch.Generator().manual_seed(8)
  a = torch.randint(0, 40, (2, 120), generator=gen)
  ei = torch.cat([a, a + 40], 1)
  return _sym(torch.unique(ei[:, ei[0] != ei[1]], dim=1)), 90


def star_graph():
  """A star: centre 0 and leaves 1..60.  Every leaf's row is [0], so the leaves of a subgraph get identical GCN rows
  and exactly tied sort keys; a 2-hop subgraph of two leaves holds 61 nodes, more than k."""
  leaves = torch.arange(1, 61)
  return _sym(torch.stack([torch.zeros_like(leaves), leaves])), 61


GRAPHS = {'wide': wide_graph, 'directed': directed_graph, 'loops': loops_graph, 'degenerate': degenerate_graph,
          'star': star_graph}


def case_links(graph, ei, n, count, seed):
  """Graph edges, random pairs, the links the graph's fixture is for, then two invalid links (-1, and s == d)."""
  gen = torch.Generator().manual_seed(seed)
  pos = ei[:, torch.randint(0, ei.shape[1], (count // 2,), generator=gen)]
  rnd = torch.randint(0, n, (2, count - count // 2), generator=gen)
  special = {
      'wide': [[0, 0, 1], [1, 2, 0]],                                  # the hub as an endpoint: truncated
      'degenerate': [[80, 81, 0, 3, 85], [81, 0, 45, 60, 86]],         # isolated, isolated + component, two components
      'star': [[1, 5, 0], [2, 60, 7]],
  }.get(graph, [[], []])
  links = torch.cat([pos, torch.tensor(special, dtype=torch.int64), rnd, torch.tensor([[-1, 4], [3, 4]])], 1)
  return links, (torch.arange(links.shape[1]) % 2 == 0).float()


# --------------------------------------------------------------------------- engine runs
def make_engine(g, n, hidden, layers, k, hops, max_z, max_nodes, max_edges, dropout, batch, seed=0):
  eng = SealEngine(g, n, num_hops=hops, max_nodes=max_nodes, max_edges=max_edges, hidden=hidden, num_layers=layers,
                   sort_k=k, max_z=max_z, dropout=dropout, batch_size=batch, seed=seed, use_cuda_graph=False)
  # GCNConv biases start at zero; draw them so that every parameter enters every stage
  gen = torch.Generator().manual_seed(seed + 100)
  for name, off, shape in eng.layout:
    if name.startswith('convs.') and name.endswith('bias'):
      eng.params[off:off + math.prod(shape)] = (torch.rand(shape, generator=gen) * 0.6 - 0.3).to(DEV)
  return eng


def run_step(eng, links, labels):
  """extract, forward (training, so with the engine's dropout), backward and reduce on one batch; host copies."""
  eng._stage(links.to(DEV), eng.links, labels.to(DEV), eng.labels)
  eng._extract(eng.links)
  eng._forward(eng.labels, True)
  eng._backward()
  torch.cuda.synchronize()
  A = eng.arena
  h = {k: getattr(A, k).cpu() for k in ('meta', 'sptr', 'scol', 'z', 'X', 'sel', 'C1', 'flat', 'H1', 'mask', 'logits',
                                        'lossv', 'partials')}
  h['labels'] = eng.labels.cpu()
  h['grad'], h['loss'] = eng.grad.cpu(), eng.loss.cpu()
  return h


def _params(eng):
  return {name: t.detach().double().cpu() for name, t in eng.parameters_dict().items()}


def _subgraph(h, b):
  """n, local edges (source, destination) from the source CSR in (source, row) order, and the clamped labels."""
  n, e = int(h['meta'][b, 0]), int(h['meta'][b, 1])
  sptr = h['sptr'][b, :n + 1].long()
  src = torch.repeat_interleave(torch.arange(n), sptr.diff())
  return n, src, h['scol'][b, :e].long(), h['z'][b, :n].long()


def _worst(ratios, stage, r):
  ratios[stage] = max(ratios.get(stage, 0.0), r)


def check_forward(eng, P, h, b, nv, ratios):
  """Every forward stage of link b from the kernel's previous stage; the bound ratio per stage goes into ratios."""
  H, L, k, Z = eng.hidden, eng.num_layers, eng.k, eng.max_z + 1
  T, kp = H * L + 1, k // 2
  t2 = kp - 4
  n, src, dst, z = _subgraph(h, b)
  keep = src != dst
  s, d = src[keep], dst[keep]
  indeg = torch.zeros(n, dtype=F64).index_add_(0, d, torch.ones(d.numel(), dtype=F64))
  dinv = (indeg + 1).rsqrt()
  coef = (dinv[s] * dinv[d])[:, None]
  X = h['X'][b, :n].double()
  for l in range(L + 1):
    W, bias = P[f'convs.{l}.lin.weight'], P[f'convs.{l}.bias']
    if l == 0:
      xw = W[:, z.clamp(max=Z - 1)].t()
      xa = xw.abs()
    else:
      xin = X[:, (l - 1) * H:l * H]
      xw, xa = xin @ W.t(), xin.abs() @ W.abs().t()
    agg = (dinv * dinv)[:, None] * xw
    agg = agg.index_add_(0, d, coef * xw[s])
    aga = (dinv * dinv)[:, None] * xa
    aga = aga.index_add_(0, d, coef * xa[s])
    ref = torch.tanh(agg + bias)
    # H products, in-degree + 1 aggregation terms, the bias, and 4 for rsqrtf's 2 ulp in each normalisation factor
    m = (H + indeg + 6)[:, None]
    bound = tanh_bound(fp32_sum_bound(m, aga + bias.abs()), ref)
    _worst(ratios, f'layer {l}', bound_ratio(X[:, l * H:l * H + W.shape[0]], ref, bound))

  # sort-pool: the top k of the kernel's own last channel, descending, ties to the lower local id, then -1
  sel = h['sel'][b].long()
  order = torch.sort(h['X'][b, :n, T - 1], descending=True, stable=True).indices
  want = torch.full((k,), -1, dtype=torch.int64)
  want[:min(n, k)] = order[:k]
  assert torch.equal(sel, want), ('sort-pool rows', b, sel.tolist(), want.tolist())

  rows = sel >= 0
  pooled = torch.zeros(k, T, dtype=F64)
  pooled[rows] = X[sel[rows]]
  w1, b1 = P['conv1.weight'].reshape(16, T), P['conv1.bias']
  pre = (pooled @ w1.t()).t() + b1[:, None]
  bound = fp32_sum_bound(T + 1, (pooled.abs() @ w1.abs().t()).t() + b1.abs()[:, None])
  bound[:, ~rows] = 0                                  # a padding row is ReLU(bias) exactly
  C1 = h['C1'][b].double()
  _worst(ratios, 'conv1', bound_ratio(C1, pre.clamp(min=0), bound))
  assert bool((C1[pre < -bound] == 0).all()) and bool((C1 >= 0).all()), ('conv1 ReLU', b)

  # maxpool selects from the kernel's C1 exactly; conv2 sums 80 products and the bias
  M = torch.maximum(C1[:, 0:2 * kp:2], C1[:, 1:2 * kp:2])
  win = M.unfold(1, 5, 1)                              # [16, t2, 5]
  w2, b2 = P['conv2.weight'], P['conv2.bias']
  pre = torch.einsum('ock,ctk->ot', w2, win) + b2[:, None]
  bound = fp32_sum_bound(81, torch.einsum('ock,ctk->ot', w2.abs(), win) + b2.abs()[:, None])
  flat = h['flat'][b].double().reshape(32, t2)
  _worst(ratios, 'conv2', bound_ratio(flat, pre.clamp(min=0), bound))
  assert bool((flat[pre < -bound] == 0).all()), ('conv2 ReLU', b)

  flat = flat.reshape(-1)
  l1w, l1b = P['mlp.lins.0.weight'], P['mlp.lins.0.bias']
  pre = l1w @ flat + l1b
  bound = fp32_sum_bound(flat.numel() + 1, l1w.abs() @ flat + l1b.abs())
  H1 = h['H1'][b].double()
  _worst(ratios, 'lin1', bound_ratio(H1, pre.clamp(min=0), bound))
  assert bool((H1[pre < -bound] == 0).all()), ('lin1 ReLU', b)
  mk = h['mask'][b]
  if eng.dropout > 0:
    assert bool(((mk == 0) | (mk == 1 / (1 - eng.dropout))).all()), ('dropout mask', b)
  else:
    assert bool((mk == 1).all()), ('dropout mask', b)

  h1 = (h['H1'][b] * mk).double()                     # the kernel's fp32 product
  l2w, l2b = P['mlp.lins.1.weight'].reshape(-1), P['mlp.lins.1.bias']
  pre = l2w @ h1 + l2b
  bound = fp32_sum_bound(129, l2w.abs() @ h1 + l2b.abs())
  x = h['logits'][b].double()
  _worst(ratios, 'logit', bound_ratio(x, pre, bound))

  # loss term: BCE-with-logits of the kernel's logit / valid links; expf, log1pf, the division and the products
  y = h['labels'][b].double()
  lin, soft = x.clamp(min=0) - x * y, torch.log1p(torch.exp(-x.abs()))
  ref = (lin + soft) / nv
  _worst(ratios, 'loss term', bound_ratio(h['lossv'][b].double(), ref, 8 * EPS * (lin.abs() + soft) / nv))


def link_gradients(eng, model, h, b, nv):
  """float64 autograd of link b's loss term BCE / nv, at the kernel's forward point: its sort-pool rows, its ReLU
  and maxpool decisions (from C1, flat and H1) and its dropout mask."""
  H, L, k = eng.hidden, eng.num_layers, eng.k
  T, kp = H * L + 1, k // 2
  n, src, dst, z = _subgraph(h, b)
  model.zero_grad()
  X = model.node_features(F.one_hot(z, eng.max_z + 1).double(), src, dst)
  sel = h['sel'][b].long()
  rows = sel[sel >= 0]
  pooled = torch.cat([X[rows], torch.zeros(k - rows.numel(), T, dtype=F64)])
  C1, flat, H1 = h['C1'][b], h['flat'][b].reshape(32, kp - 4), h['H1'][b]
  c1 = model.conv1(pooled.reshape(1, 1, -1))[0] * (C1 > 0)
  idx = 2 * torch.arange(kp) + (C1[:, 1:2 * kp:2] > C1[:, 0:2 * kp:2]).long()
  c2 = model.conv2(c1.gather(1, idx)[None])[0] * (flat > 0)
  hh = model.mlp.lins[0](c2.reshape(-1)) * (H1 > 0) * h['mask'][b].double()
  logit = model.mlp.lins[1](hh)[0]
  loss = F.binary_cross_entropy_with_logits(logit, h['labels'][b].double()) / nv
  loss.backward()
  return {name: p.grad for name, p in model.named_parameters()}


def check_gradients(eng, model, h, b, nv, ratios):
  ref = link_gradients(eng, model, h, b, nv)
  for name, off, shape in eng.layout:
    r = ref[name].reshape(-1)
    got = h['partials'][b, off:off + r.numel()].double()
    ratio = bound_ratio(got, r, grad_tol(r))
    _worst(ratios, 'gradient', ratio)
    if ratio > 1:
      ratios.setdefault('gradient tensors over', []).append((b, name))


def check_reduce(h):
  """grad and loss = the valid links' partials and loss terms summed in link order in fp32 (k_seal_reduce), bitwise."""
  valid = torch.nonzero(h['meta'][:, 2] == 1).reshape(-1).tolist()
  g = torch.zeros(h['partials'].shape[1])
  loss = torch.zeros(1)
  for b in valid:
    g += h['partials'][b]
    loss += h['lossv'][b]
  assert torch.equal(h['grad'], g), ('reduce', int((h['grad'] != g).sum()))
  assert torch.equal(h['loss'], loss), ('reduced loss', float(h['loss']), float(loss))


def _report(tag, ratios):
  over = ratios.pop('gradient tensors over', [])
  print(f'{tag}: max error / bound = ' + ', '.join(f'{s} {r:.3f}' for s, r in ratios.items()))
  for stage, r in ratios.items():                      # forward stages in order, so a failure names the first
    assert stage == 'gradient' or r <= 1, (stage, r)
  assert not over, ('gradient', over[:8])


# --------------------------------------------------------------------------- 1-4. shapes and graphs
# graph, hidden, num_layers, k, num_hops, max_z, max_nodes, max_edges.  'max' is the largest hidden (or k) the
# device's shared memory admits at that shape.
CASES = [
    ('loops', 1, 1, 10, 1, 3, 256, 8192),
    ('directed', 3, 2, 11, 2, 40, 256, 8192),
    ('loops', 8, 8, 31, 3, 2 ** 16, 256, 8192),
    ('directed', 33, 5, 64, 4, 40, 256, 8192),
    ('degenerate', 64, 2, 10, 2, 3, 256, 8192),
    ('star', 200, 1, 11, 2, 40, 256, 8192),
    ('wide', 128, 2, 64, 2, 40, 1024, 1 << 16),        # subgraphs of 200 to 1,024 nodes
    ('wide', 64, 2, 300, 2, 3, 256, 8192),             # k > max_nodes; max_nodes truncates
    ('wide', 8, 3, 10, 2, 40, 1024, 3000),             # max_edges truncates
    ('wide', 'max', 1, 10, 2, 40, 1024, 1 << 16),
    ('loops', 32, 2, 'max', 3, 40, 256, 8192),
]


@pytest.mark.parametrize('dropout', [0.0, 0.5])
@pytest.mark.parametrize('graph,hidden,layers,k,hops,max_z,max_nodes,max_edges', CASES)
def test_stages_and_link_gradients_match_float64(graph, hidden, layers, k, hops, max_z, max_nodes, max_edges,
                                                 dropout):
  limit = optin_smem()
  if hidden == 'max':
    hidden = largest_hidden(layers, k, max_nodes, limit)
  if k == 'max':
    k = largest_k(hidden, layers, max_nodes, limit)
  ei, n = GRAPHS[graph]()
  g = _graph(ei, n)
  links, labels = case_links(graph, ei, n, 12 if graph == 'wide' else 24, seed=hops)
  eng = make_engine(g, n, hidden, layers, k, hops, max_z, max_nodes, max_edges, dropout, links.shape[1] + 2)
  h = run_step(eng, links, labels)
  meta = h['meta']
  nv = int(meta[:, 2].sum())
  assert nv == int(((links[0] >= 0) & (links[0] != links[1])).sum())
  if graph == 'wide':
    assert int(meta[:, 0].max()) == max_nodes and int(meta[:, 3].sum()) > 0   # the hub's links fill max_nodes
    if max_nodes == 1024:
      assert int(((meta[:, 0] > 256) & (meta[:, 3] == 0)).sum()) > 0
  P, model = _params(eng), ref_model(eng)
  ratios = {}
  for b in range(links.shape[1]):
    if meta[b, 2]:
      check_forward(eng, P, h, b, nv, ratios)
      check_gradients(eng, model, h, b, nv, ratios)
  check_reduce(h)
  _report(f'{graph} hidden={hidden} layers={layers} k={k} hops={hops} max_z={max_z} max_nodes={max_nodes} '
          f'max_edges={max_edges} dropout={dropout}', ratios)


def test_fixtures_extract_as_the_oracle():
  """The new fixtures' subgraphs are what the tests above assume: nodes, source-CSR edges and labels as the oracle,
  with the destination CSR holding the same edges; directed rows, self-loops, duplicates, z = 0 nodes, wide
  subgraphs and hub in-degrees in the hundreds are present."""
  seen = {'asymmetric': False, 'self-loop': False, 'duplicate': False, 'z0': False, 'isolated pair': False,
          'wide untruncated': False, 'hub in-degree': 0}
  for graph, max_nodes, max_edges in (('directed', 256, 8192), ('loops', 256, 8192), ('degenerate', 256, 8192),
                                      ('wide', 1024, 1 << 16)):
    ei, n = GRAPHS[graph]()
    g = _graph(ei, n)
    indptr, indices = g.topo.indptr.cpu().tolist(), g.topo.indices.cpu().tolist()
    links, _ = case_links(graph, ei, n, 12 if graph == 'wide' else 24, seed=2)
    eng = make_engine(g, n, 8, 1, 10, 2, 1000, max_nodes, max_edges, 0.0, links.shape[1])
    eng._extract(links.to(DEV))
    for b in range(links.shape[1]):
      s, d = links[:, b].tolist()
      meta, nodes, edges, edges_t, z = engine_subgraph(eng, b)
      if not meta[2]:
        continue
      o_nodes, o_edges, o_z, tr = oracle_extract(indptr, indices, s, d, 2, max_nodes, max_edges)
      assert nodes == o_nodes and edges == o_edges and sorted(edges_t) == sorted(o_edges)
      assert (z == o_z).all() and meta[3] == int(tr)
      es = set(edges)
      seen['asymmetric'] |= any((v, u) not in es for u, v in edges)
      seen['self-loop'] |= any(u == v for u, v in edges)
      seen['duplicate'] |= len(es) < len(edges)
      seen['z0'] |= bool((z == 0).any())
      seen['isolated pair'] |= meta[0] == 2 and meta[1] == 0
      seen['wide untruncated'] |= meta[0] > 256 and not tr
      deg = torch.bincount(torch.tensor([v for _, v in edges] or [0]), minlength=meta[0])
      seen['hub in-degree'] = max(seen['hub in-degree'], int(deg.max()))
  assert all(seen[key] for key in seen if key != 'hub in-degree'), seen
  assert seen['hub in-degree'] >= 200, seen


# --------------------------------------------------------------------------- 5. batches wider than the CTA
@pytest.mark.parametrize('batch', [300, 1000])
def test_large_batches_count_score_and_reduce_in_link_order(batch):
  ei, n = loops_graph()
  g = _graph(ei, n)
  gen = torch.Generator().manual_seed(batch)
  count = batch - 13                                   # the last 13 slots are padding
  links = torch.randint(0, n, (2, count), generator=gen)
  links[:, ::4] = ei[:, torch.randint(0, ei.shape[1], (links[:, ::4].shape[1],), generator=gen)]
  links[0, 3::7] = -1                                  # invalid links interleaved: -1, s == d, id past N
  links[1, 5::11] = links[0, 5::11]
  links[1, 6::13] = n
  labels = (torch.arange(count) % 4 == 0).float()
  eng = make_engine(g, n, 8, 2, 10, 2, 40, 256, 8192, 0.5, batch)
  h = run_step(eng, links, labels)
  meta = h['meta']
  ok = (links[0] >= 0) & (links[1] < n) & (links[0] != links[1])
  assert torch.equal(meta[:count, 2] == 1, ok) and not bool(meta[count:, 2].any())
  nv = int(ok.sum())
  # every link's loss term from its logit with the batch's valid-link count; invalid links score 0
  x, y = h['logits'][:count].double(), labels.double()
  lin, soft = x.clamp(min=0) - x * y, torch.log1p(torch.exp(-x.abs()))
  ratio = bound_ratio(h['lossv'][:count][ok].double(), ((lin + soft) / nv)[ok], (8 * EPS * (lin.abs() + soft) / nv)[ok])
  assert ratio <= 1, ('loss terms', ratio)
  assert not bool(h['logits'][:count][~ok].any()) and not bool(h['lossv'][:count][~ok].any())
  # stages and partials of a sample of valid links across the batch, most of them past the first 256
  valid = torch.nonzero(ok).reshape(-1)
  sample = valid[torch.linspace(0, valid.numel() - 1, 12).round().long()].tolist()
  P, model = _params(eng), ref_model(eng)
  ratios = {'loss terms (all links)': ratio}
  for b in sample:
    check_forward(eng, P, h, b, nv, ratios)
    check_gradients(eng, model, h, b, nv, ratios)
  check_reduce(h)
  _report(f'batch {batch} ({nv} valid)', ratios)


# --------------------------------------------------------------------------- 6. the shared-memory envelope
def test_largest_hidden_and_k_build_and_one_past_raises():
  limit = optin_smem()
  ei, n = star_graph()
  g = _graph(ei, n)
  kw = dict(max_edges=256, max_z=20, batch_size=2)
  limits = []
  for max_nodes, layers, k in ((256, 1, 10), (1024, 1, 10), (1024, 8, 64)):
    hmax = largest_hidden(layers, k, max_nodes, limit)
    limits.append(f'hidden <= {hmax} at max_nodes={max_nodes} num_layers={layers} k={k}')
    SealEngine(g, n, hidden=hmax, num_layers=layers, sort_k=k, max_nodes=max_nodes, **kw)
    if hmax < 256:
      with pytest.raises(ValueError, match='shared memory'):
        SealEngine(g, n, hidden=hmax + 1, num_layers=layers, sort_k=k, max_nodes=max_nodes, **kw)
  for hidden, layers, max_nodes in ((32, 3, 256), (32, 3, 1024), (128, 2, 256), (128, 2, 1024)):
    kmax = largest_k(hidden, layers, max_nodes, limit)
    limits.append(f'k <= {kmax} at hidden={hidden} num_layers={layers} max_nodes={max_nodes}')
    SealEngine(g, n, hidden=hidden, num_layers=layers, sort_k=kmax, max_nodes=max_nodes, **kw)
    if kmax < 2048:
      with pytest.raises(ValueError, match='shared memory'):
        SealEngine(g, n, hidden=hidden, num_layers=layers, sort_k=kmax + 1, max_nodes=max_nodes, **kw)
  print(f'shared memory per block (opt-in) {limit} bytes: ' + '; '.join(limits))
