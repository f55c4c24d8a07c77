"""MetaPath2VecEngine: metapath walks (k_metapath_walk), SGNS negatives, the fused loss / gradient against float64
autograd, SparseAdam against torch.optim.SparseAdam, CUDA-graph replay, learning planted communities, and the
argument errors of the engine and its bindings."""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
EPS = 1e-15


def _graph(ei, n):
  g = glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=n), 'CUDA', 0)
  g.lazy_init()
  return g


def _typed_graph():
  """Node types a (7), b (6), c (5); relations ab, bc, ca and their reverses ba, cb, ac.  a6 has no ab edge, b5 no bc
  edge, c4 no ca edge (dead ends of the forward relations)."""
  sizes = {'a': 7, 'b': 6, 'c': 5}
  gen = torch.Generator().manual_seed(5)
  edges = {}
  for s, d, dead in (('a', 'b', 6), ('b', 'c', 5), ('c', 'a', 4)):
    src = torch.arange(sizes[s]).repeat_interleave(3)
    dst = torch.randint(0, sizes[d], (src.numel(),), generator=gen)
    keep = src != dead
    ei = torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)
    edges[(s, s + d, d)] = ei
    edges[(d, d + s, s)] = ei.flip(0)
  graphs = {e: _graph(ei, max(sizes[e[0]], sizes[e[2]])) for e, ei in edges.items()}
  return edges, graphs, sizes


REL = {'ab': ('a', 'ab', 'b'), 'bc': ('b', 'bc', 'c'), 'ca': ('c', 'ca', 'a'), 'ba': ('b', 'ba', 'a'),
       'cb': ('c', 'cb', 'b'), 'ac': ('a', 'ac', 'c')}
PATHS = {1: ['ab'], 3: ['ab', 'bc', 'ca'], 6: ['ab', 'bc', 'cb', 'ba', 'ac', 'ca']}


def _slot_types(eng):
  return [eng.metapath[0][0]] + [e[2] for e in eng.metapath]


def _windows(eng):
  """(rows [n_walks, J, C] in the concatenated table, valid [n_walks, J], slot offsets [J, C]) of the last walks."""
  walks = eng.walks.cpu()
  L, C, R = eng.walk_length, eng.context_size, eng.R
  slot = torch.tensor([0] + [(p - 1) % R + 1 for p in range(1, L + 1)])
  st = _slot_types(eng)
  off = torch.tensor([eng.offsets[t] for t in st])[slot]
  n = torch.tensor([eng.num_nodes[t] for t in st])[slot]
  wins = walks.unfold(1, C, 1)                                       # [n_walks, J, C]
  off_w, n_w = off.unfold(0, C, 1), n.unfold(0, C, 1)               # [J, C]
  valid = ((wins >= 0) & (wins < n_w)).all(-1)
  return wins + off_w, valid, off_w, n_w


def _host_walk_checks(eng, edges, starts):
  walks = eng.walks.cpu()
  W, L, R, C = eng.walks_per_node, eng.walk_length, eng.R, eng.context_size
  sets = {e: set(map(tuple, edges[e].t().tolist())) for e in eng.metapath}
  has_out = {e: set(edges[e][0].tolist()) for e in eng.metapath}
  n_windows = 0
  for i in range(walks.shape[0]):
    w = walks[i].tolist()
    st = int(starts[i // W])
    if st < 0:
      assert all(x == -1 for x in w), w                              # padded start: all -1
      continue
    assert w[0] == st
    ended = False
    for s in range(1, L + 1):
      rel = eng.metapath[(s - 1) % R]
      if ended:
        assert w[s] == -1, w
      elif w[s] == -1:
        assert w[s - 1] not in has_out[rel], (w, rel)              # -1 only at a dead end
        ended = True
      else:
        assert (w[s - 1], w[s]) in sets[rel], (w, s, rel)
    n_valid = sum(x >= 0 for x in w)
    n_windows += max(0, n_valid - C + 1)
  assert int(eng.n_valid) == n_windows


# --------------------------------------------------------------------------- 1. walks
@pytest.mark.parametrize('R,L', [(1, 1), (3, 2), (3, 3), (3, 7), (6, 4), (6, 6), (6, 13)])
def test_walks_follow_the_metapath(native, R, L):
  edges, graphs, sizes = _typed_graph()
  mp = [REL[r] for r in PATHS[R]]
  eng = MetaPath2VecEngine(graphs, sizes, mp, embedding_dim=8, walk_length=L, context_size=2, walks_per_node=3,
                           num_negative_samples=1, batch_size=10, device=DEV, use_cuda_graph=False)
  starts = torch.tensor([0, 1, 2, 3, 4, 5, 6, -1, 2, -1])
  eng._stage(starts.to(DEV))
  eng._sample()
  torch.cuda.synchronize()
  _host_walk_checks(eng, edges, starts)
  # dead ends are reached: a6 has no ab edge, so its walks are [6, -1, ...]
  assert bool((eng.walks.view(10, 3, L + 1)[6, :, 1] == -1).all())


def test_deepwalk_first_steps_are_uniform(native):
  from scipy.stats import chisquare
  N, hub_deg = 64, 40
  src = torch.cat([torch.zeros(hub_deg, dtype=torch.int64), torch.arange(1, N)])
  dst = torch.cat([torch.arange(1, hub_deg + 1), (torch.arange(1, N) % (N - 1)) + 1])
  ei = torch.unique(torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1), dim=1)
  g = _graph(ei, N)
  eng = MetaPath2VecEngine({('n', 'to', 'n'): g}, {'n': N}, [('n', 'to', 'n')], embedding_dim=8, walk_length=2,
                           context_size=2, walks_per_node=250, num_negative_samples=1, batch_size=80, device=DEV,
                           use_cuda_graph=False)
  eng._stage(torch.zeros(80, dtype=torch.int64, device=DEV))
  eng._sample()
  first = eng.walks[:, 1].cpu()
  nbrs = ei[1][ei[0] == 0]
  counts = torch.stack([(first == v).sum() for v in nbrs]).double()
  assert int(counts.sum()) == first.numel()                          # every first step is a neighbour of the hub
  p = chisquare(counts.numpy()).pvalue                               # 20000 draws over 40 neighbours
  assert p > 1e-3, (p, counts)


def test_walks_are_keyed_by_seed_and_step(native):
  edges, graphs, sizes = _typed_graph()
  eng = MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[3]], embedding_dim=8, walk_length=12,
                           context_size=3, walks_per_node=4, num_negative_samples=2, batch_size=7, device=DEV)
  starts = torch.arange(7, device=DEV)
  walks = torch.empty_like(eng.walks)
  n_valid = torch.zeros(1, dtype=torch.int32, device=DEV)

  def walk(step, seed=0):
    native.metapath_walk(eng.mp, starts, 4, 3, seed, torch.tensor([step], dtype=torch.int32, device=DEV), walks,
                         n_valid)
    return walks.clone()
  a = walk(5)
  assert torch.equal(a, walk(5))                                     # bitwise reproducible
  assert not torch.equal(a, walk(6)) and not torch.equal(a, walk(5, seed=1))
  # successive replays of the captured step draw fresh walks
  eng.warmup_and_capture()
  seen = []
  for _ in range(3):
    eng.train_step(starts)
    seen.append(eng.walks.clone())
  assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2])
  assert int(eng.state[0]) == 3 and int(eng.state[1]) == 3


# --------------------------------------------------------------------------- 2. negatives
def test_negatives_types_centres_and_invalid_windows(native):
  edges, graphs, sizes = _typed_graph()
  K = 3
  eng = MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[6]], embedding_dim=8, walk_length=9,
                           context_size=4, walks_per_node=5, num_negative_samples=K, batch_size=8, device=DEV,
                           use_cuda_graph=False)
  eng._stage(torch.tensor([0, 1, 2, 6, 4, -1, 5, 3], device=DEV))
  eng._sample()
  rows, valid, off_w, n_w = _windows(eng)
  walks = eng.walks.cpu().unfold(1, eng.context_size, 1)
  J, C = walks.shape[1], eng.context_size
  neg = eng.negatives.cpu().view(-1, J, K, C)
  assert bool(valid.any()) and not bool(valid.all())
  v, nv = neg[valid], neg[~valid]
  assert bool((nv == -1).all())                                      # no negative for an invalid window
  assert torch.equal(v[:, :, 0], walks[valid][:, None, 0].expand(-1, K))   # same centre as the positive window
  n_valid_w = n_w.expand(walks.shape[0], J, C)[valid]              # [nv, C] type sizes per position
  assert bool(((v[:, :, 1:] >= 0) & (v[:, :, 1:] < n_valid_w[:, None, 1:])).all())
  # every context position draws over its type: the largest type's positions reach ids beyond the smaller types
  big = n_valid_w[:, None, 1:].expand_as(v[:, :, 1:]) == 7
  assert int(v[:, :, 1:][big].max()) >= 6


# --------------------------------------------------------------------------- 3. loss and gradient
def _ref_loss(eng, W):
  """float64 loss of the engine's last walks and negatives and the rows it looks up.  PyG's 1 - sigmoid(s) is written
  sigmoid(-s), the same function: in float64 the subtraction loses every digit of 1 - sigmoid(s) for s above ~35,
  which 512-wide N(0, 1) rows reach."""
  rows, valid, off_w, _ = _windows(eng)
  K, C = eng.num_negative_samples, eng.context_size
  J = rows.shape[1]
  vr = rows[valid]                                                   # [nv, C]
  neg = eng.negatives.cpu().view(-1, J, K, C)[valid]                 # [nv, K, C]
  nr = neg + off_w.expand(rows.shape[0], J, C)[valid][:, None, :]
  h = W[vr[:, 0]]
  s = (h[:, None, :] * W[vr[:, 1:]]).sum(-1)
  sn = (h[:, None, None, :] * W[nr[:, :, 1:]]).sum(-1)
  loss = -torch.log(torch.sigmoid(s) + EPS).mean() - torch.log(torch.sigmoid(-sn) + EPS).mean()
  looked = torch.unique(torch.cat([vr.flatten(), nr.flatten()]))
  return loss, looked, int(valid.sum())


@pytest.mark.parametrize('D', [8, 64, 128, 136, 512])
def test_loss_and_gradient_match_float64(native, D):
  N = 300                                                            # star: node 0 is in nearly every window
  leaves = torch.arange(1, N)
  ei = torch.cat([torch.stack([torch.zeros_like(leaves), leaves]), torch.stack([leaves, torch.zeros_like(leaves)])], 1)
  ring = torch.stack([leaves, leaves % (N - 1) + 1])
  ei = torch.unique(torch.cat([ei, ring], 1), dim=1)
  eng = MetaPath2VecEngine({('n', 'to', 'n'): _graph(ei, N)}, {'n': N}, [('n', 'to', 'n')], embedding_dim=D,
                           walk_length=16, context_size=5, walks_per_node=3, num_negative_samples=4, batch_size=24,
                           seed=D, device=DEV, use_cuda_graph=False)
  eng._stage(torch.randint(0, N, (24,), generator=torch.Generator().manual_seed(D)).to(DEV))
  W0 = eng.weight.clone()
  eng._sample()
  eng._loss_grad()
  torch.cuda.synchronize()
  W = W0.cpu().double().requires_grad_()
  loss, looked, nv = _ref_loss(eng, W)
  loss.backward()
  assert nv == int(eng.n_valid) and nv > 0
  hub_windows = int((eng.walks.cpu().unfold(1, 5, 1) == 0).any(-1).sum())
  assert hub_windows > 300                                           # the hub row sums hundreds of windows
  torch.testing.assert_close(eng.loss.cpu().double(), loss.detach().reshape(1), rtol=2e-5, atol=1e-5)
  ref = W.grad
  torch.testing.assert_close(eng.grad.cpu().double(), ref, rtol=1e-4, atol=2e-5 * float(ref.abs().max()))
  touched = torch.nonzero(eng.touched.cpu()).flatten()
  assert torch.equal(touched, looked)                                # exactly the rows nn.Embedding would list


def test_typed_loss_and_gradient_match_float64(native):
  edges, graphs, sizes = _typed_graph()
  eng = MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[3]], embedding_dim=64, walk_length=10,
                           context_size=4, walks_per_node=4, num_negative_samples=3, batch_size=7, device=DEV,
                           use_cuda_graph=False)
  eng._stage(torch.arange(7, device=DEV))
  W0 = eng.weight.clone()
  eng._sample()
  eng._loss_grad()
  W = W0.cpu().double().requires_grad_()
  loss, looked, _ = _ref_loss(eng, W)
  loss.backward()
  torch.testing.assert_close(eng.loss.cpu().double(), loss.detach().reshape(1), rtol=2e-5, atol=1e-5)
  torch.testing.assert_close(eng.grad.cpu().double(), W.grad, rtol=1e-4, atol=2e-5 * float(W.grad.abs().max()))
  assert torch.equal(torch.nonzero(eng.touched.cpu()).flatten(), looked)


# --------------------------------------------------------------------------- 4. optimizer
def test_sparse_adam_matches_torch(native):
  N = 2000
  gen = torch.Generator().manual_seed(3)
  ei = torch.randint(0, N, (2, 6000), generator=gen)
  ei = torch.unique(torch.cat([ei, ei.flip(0)], 1), dim=1)
  eng = MetaPath2VecEngine({('n', 'to', 'n'): _graph(ei, N)}, {'n': N}, [('n', 'to', 'n')], embedding_dim=32,
                           walk_length=8, context_size=3, walks_per_node=2, num_negative_samples=2, batch_size=16,
                           lr=0.01, device=DEV, use_cuda_graph=False)
  sd = eng.state_dict()                                              # a known state: small rows, warm moments
  sd['weight']['n'] = 0.2 * torch.randn(N, 32, generator=gen)
  eng.load_state_dict(sd)
  emb = torch.nn.Embedding(N, 32, sparse=True).to(DEV)
  with torch.no_grad():
    emb.weight.copy_(eng.weight)
  opt = torch.optim.SparseAdam(emb.parameters(), lr=0.01)
  W_init = eng.weight.clone()
  ever = torch.zeros(N, dtype=torch.bool)
  for step in range(3):
    eng.train_step(torch.randint(0, N, (16,), generator=gen))
    rows, valid, off_w, _ = _windows(eng)
    J, K, C = rows.shape[1], eng.num_negative_samples, eng.context_size
    vr = rows[valid].to(DEV)
    nr = eng.negatives.view(-1, J, K, C)[valid.to(DEV)]
    h = emb(vr[:, 0])
    s = (h[:, None, :] * emb(vr[:, 1:])).sum(-1)
    sn = (h[:, None, None, :] * emb(nr[:, :, 1:])).sum(-1)
    loss = -torch.log(torch.sigmoid(s) + EPS).mean() - torch.log(torch.sigmoid(-sn) + EPS).mean()
    opt.zero_grad()
    loss.backward()
    opt.step()
    torch.testing.assert_close(eng.loss[0], loss.detach(), rtol=1e-5, atol=1e-6)
    ever[torch.unique(torch.cat([vr.flatten(), nr.flatten()])).cpu()] = True
    torch.testing.assert_close(eng.weight, emb.weight.detach(), rtol=1e-5, atol=1e-5)
  st = opt.state[emb.weight]
  torch.testing.assert_close(eng.exp_avg, st['exp_avg'], rtol=1e-4, atol=1e-8)
  torch.testing.assert_close(eng.exp_avg_sq, st['exp_avg_sq'], rtol=1e-4, atol=1e-12)
  assert int(eng.state[1]) == 3 == int(st['step'])
  assert bool(ever.any()) and not bool(ever.all())
  untouched = (~ever).to(DEV)
  assert torch.equal(eng.weight[untouched], W_init[untouched])        # bitwise unchanged
  assert bool((eng.exp_avg[untouched] == 0).all()) and bool((eng.exp_avg_sq[untouched] == 0).all())
  assert int(eng.touched.sum()) == 0 and int((eng.grad != 0).sum()) == 0   # the update clears what the step marked


# --------------------------------------------------------------------------- 5. capture
def test_captured_steps_match_eager(native):
  edges, graphs, sizes = _typed_graph()
  kw = dict(embedding_dim=24, walk_length=11, context_size=4, walks_per_node=3, num_negative_samples=2,
            batch_size=7, seed=11, device=DEV)
  mp = [REL[r] for r in PATHS[6]]
  eager = MetaPath2VecEngine(graphs, sizes, mp, use_cuda_graph=False, **kw)
  graph = MetaPath2VecEngine(graphs, sizes, mp, use_cuda_graph=True, **kw)
  eager.warmup_and_capture()
  graph.warmup_and_capture()
  assert graph._graph is not None and eager._graph is None
  gen = torch.Generator().manual_seed(0)
  la, lb = [], []
  for _ in range(6):
    st = torch.randint(0, sizes['a'], (int(torch.randint(1, 8, (1,), generator=gen)),), generator=gen).pin_memory()
    la.append(float(eager.train_step(st)))
    lb.append(float(graph.train_step(st)))
    assert torch.equal(eager.walks, graph.walks) and torch.equal(eager.negatives, graph.negatives)
  torch.testing.assert_close(torch.tensor(lb), torch.tensor(la), rtol=1e-4, atol=1e-5)
  torch.testing.assert_close(graph.weight, eager.weight, rtol=1e-4, atol=1e-5)
  sd = graph.state_dict()
  assert sd['walk_step'] == 6 and sd['adam_step'] == 6


def test_state_dict_round_trip_resumes_the_same_walks(native):
  edges, graphs, sizes = _typed_graph()
  kw = dict(embedding_dim=16, walk_length=6, context_size=3, walks_per_node=2, num_negative_samples=2, batch_size=7,
            device=DEV)
  mp = [REL[r] for r in PATHS[3]]
  a = MetaPath2VecEngine(graphs, sizes, mp, **kw)
  a.warmup_and_capture()
  st = torch.arange(7)
  for _ in range(2):
    a.train_step(st)
  sd = a.state_dict()
  a.train_step(st)
  b = MetaPath2VecEngine(graphs, sizes, mp, seed=0, **kw)
  b.load_state_dict(sd)
  b.warmup_and_capture()
  b.train_step(st)
  assert torch.equal(a.walks, b.walks)
  torch.testing.assert_close(b.weight, a.weight, rtol=1e-5, atol=1e-6)


# --------------------------------------------------------------------------- 6. learning
def test_learns_planted_author_communities(native):
  k, per, papers_per = 4, 150, 150
  gen = torch.Generator().manual_seed(0)
  na, npap = k * per, k * papers_per
  comm_a = torch.arange(na) // per
  src, dst = [], []
  for a in range(na):
    own = comm_a[a] * papers_per + torch.randint(0, papers_per, (5,), generator=gen)
    other = torch.randint(0, npap, (1,), generator=gen)
    for p in torch.cat([own, other]).tolist():
      src.append(a)
      dst.append(p)
  writes = torch.unique(torch.tensor([src, dst]), dim=1)
  sizes = {'author': na, 'paper': npap}
  n = max(na, npap)
  graphs = {('author', 'writes', 'paper'): _graph(writes, n), ('paper', 'rev_writes', 'author'): _graph(writes.flip(0), n)}
  eng = MetaPath2VecEngine(graphs, sizes, [('author', 'writes', 'paper'), ('paper', 'rev_writes', 'author')],
                           embedding_dim=32, walk_length=20, context_size=5, walks_per_node=5, num_negative_samples=3,
                           batch_size=100, lr=0.05, device=DEV)
  eng.warmup_and_capture()
  perm = torch.randperm(na, generator=gen)
  train, test = perm[: na // 2], perm[na // 2:]

  def accuracy():
    e = torch.nn.functional.normalize(eng.embedding('author').cpu(), dim=1)
    cent = torch.stack([e[train][comm_a[train] == c].mean(0) for c in range(k)])
    return float(((e[test] @ cent.t()).argmax(1) == comm_a[test]).float().mean())
  acc0 = accuracy()
  losses = []
  for epoch in range(30):
    order = torch.randperm(na, generator=gen)
    for i in range(0, na, 100):
      losses.append(float(eng.train_step(order[i:i + 100])))
  acc = accuracy()
  first, last = sum(losses[:6]) / 6, sum(losses[-6:]) / 6
  print(f'planted communities: loss {first:.3f} -> {last:.3f}, accuracy {acc0:.3f} -> {acc:.3f} (chance {1 / k})')
  # measured on an H100: loss 3.878 -> 0.967, accuracy 0.243 (untrained) -> 1.000
  assert last < 0.5 * first
  assert acc0 < 0.5
  assert acc > 0.8


# --------------------------------------------------------------------------- 7. errors
def test_construction_errors_are_value_errors(native):
  edges, graphs, sizes = _typed_graph()
  mp3 = [REL[r] for r in PATHS[3]]
  bad = [
    dict(metapath=[REL['ab'], REL['ca']]),                           # b -> c does not chain
    dict(metapath=[REL['ab'], REL['bc']], walk_length=3),            # open path walked past its end
    dict(metapath=[REL['ab']] * 9),
    dict(metapath=[]),
    dict(metapath=[('a', 'nope', 'b')]),
    dict(context_size=1),
    dict(context_size=66, walk_length=64),
    dict(embedding_dim=12),
    dict(embedding_dim=520),
    dict(embedding_dim=0),
    dict(num_nodes={'a': 7, 'b': 6}),
    dict(walks_per_node=0),
    dict(num_negative_samples=0),
  ]
  for kw in bad:
    args = dict(metapath=mp3, num_nodes=sizes)
    args.update(kw)
    with pytest.raises(ValueError):
      MetaPath2VecEngine(graphs, args.pop('num_nodes'), args.pop('metapath'), device=DEV, **args)
  # an open path is fine while the walk stays on it
  MetaPath2VecEngine(graphs, sizes, [REL['ab'], REL['bc']], walk_length=2, context_size=2, device=DEV)
  with pytest.raises(ValueError):
    MetaPath2VecEngine(graphs, sizes, mp3, batch_size=4, device=DEV).train_step(torch.arange(5))


def _with_defaults(fn, defaults):
  """fn with positional arguments that are None taken from defaults."""
  def call(*over):
    args = list(defaults)
    for i, o in enumerate(over):
      if o is not None:
        args[i] = o
    return fn(*args)
  return call


def test_bindings_raise_on_bad_arguments(native):
  edges, graphs, sizes = _typed_graph()
  eng = MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[3]], embedding_dim=16, walk_length=6,
                           context_size=3, walks_per_node=2, num_negative_samples=2, batch_size=4, device=DEV,
                           use_cuda_graph=False)
  mp, C, K = eng.mp, eng.context_size, eng.num_negative_samples
  cur, t = eng.state[2:3], eng.state[1:2]
  gh = [graphs[e].graph_handler for e in eng.metapath]

  def raises(fn, *a):
    with pytest.raises(RuntimeError):
      fn(*a)
  raises(native.MetaPath, 0, gh * 3, [0] * 10, [5] * 10)              # 9 relations
  raises(native.MetaPath, 0, gh, [0, 0, 0], [5, 5, 5])               # slots != R + 1
  raises(native.MetaPath, 0, gh, [0] * 4, [5, 0, 5, 5])              # empty type
  st = eng.starts
  walk = _with_defaults(native.metapath_walk, (mp, st, 2, C, 0, cur, eng.walks, eng.n_valid))
  walk()
  raises(walk, None, st.int())
  raises(walk, None, st.cpu())
  raises(walk, None, None, 3)                                        # walks rows != starts * walks_per_node
  raises(walk, None, None, 0)
  raises(walk, None, None, None, 8)                                  # context beyond walk_length + 1
  raises(walk, None, None, None, 1)
  raises(walk, None, None, None, None, None, cur.long())
  raises(walk, None, None, None, None, None, None, eng.walks.cpu())
  raises(walk, None, None, None, None, None, None, eng.walks.int())
  raises(walk, None, None, None, None, None, None, None, eng.n_valid.float())
  neg = _with_defaults(native.sgns_negatives, (mp, eng.walks, C, K, 0, cur, eng.negatives))
  neg()
  raises(neg, None, None, None, 3)                                   # K does not match the buffer
  raises(neg, None, None, None, 0)
  raises(neg, None, None, None, None, None, None, eng.negatives[:-1])
  raises(neg, None, eng.walks[:, :-1])
  loss = _with_defaults(native.sgns_loss_grad,
                        (mp, eng.walks, eng.negatives, C, K, eng.weight, eng.n_valid, eng.grad, eng.touched, eng.loss))
  loss()
  raises(loss, None, None, None, None, None, eng.weight.double())
  raises(loss, None, None, None, None, None, eng.weight[:, :12].contiguous())
  raises(loss, None, None, None, None, None, eng.weight[:5])           # fewer rows than the metapath's types
  raises(loss, None, None, None, None, None, None, None, eng.grad[:, :8].contiguous())
  raises(loss, None, None, None, None, None, None, None, None, eng.touched[:-1])
  raises(loss, None, None, None, None, None, None, None, None, eng.touched.bool())
  raises(loss, None, None, None, None, None, None, None, None, None, eng.loss.cpu())
  adam = _with_defaults(native.sparse_adam,
                        (mp, eng.weight, eng.grad, eng.exp_avg, eng.exp_avg_sq, eng.touched, t, 0.01, 0.9, 0.999, 1e-8))
  adam()
  raises(adam, None, None, None, eng.exp_avg[:-1])
  raises(adam, None, None, None, None, eng.exp_avg_sq.cpu())
  raises(adam, None, None, None, None, None, None, t.cpu())
  raises(adam, None, None, None, None, None, None, None, -1.0)
  raises(adam, None, None, None, None, None, None, None, None, 1.0)
  raises(native.m2v_begin, eng.state[:2])
  raises(native.m2v_begin, eng.state.cpu())
  torch.cuda.synchronize()
