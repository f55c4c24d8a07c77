"""node2vec's p / q walks in MetaPath2VecEngine (k_node2vec_walk): the second-step distribution against the exact
transition probabilities, hub rows, the walk contract shared with k_metapath_walk, keyed draws, learning planted
communities, the argument errors of the engine and the binding, and the example script."""
import math
import os
import sys

import pytest
import torch
from scipy.stats import chisquare

from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine
from test_gpu_metapath2vec import PATHS, REL, _graph, _host_walk_checks, _typed_graph, _with_defaults

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
HOMO = [('n', 'to', 'n')]


def _engine(ei, n, **kw):
  args = dict(embedding_dim=8, walk_length=2, context_size=2, walks_per_node=10, num_negative_samples=1,
              batch_size=8, device=DEV, use_cuda_graph=False)
  args.update(kw)
  return MetaPath2VecEngine({HOMO[0]: _graph(ei, n)}, {'n': n}, HOMO, **args)


def _rows(rows):
  """{src: [dst, ...]} -> edge_index [2, E]."""
  src = [s for s, ds in rows.items() for _ in ds]
  dst = [d for ds in rows.values() for d in ds]
  return torch.tensor([src, dst])


def _second_steps(eng, start, steps):
  """Step-2 entries of the walks whose step 1 is node 1 (v), over `steps` steps that all start at `start`."""
  out = []
  for _ in range(steps):
    eng._stage(torch.full((eng.batch_size,), start, dtype=torch.int64, device=DEV))
    eng._sample()
    w = eng.walks.cpu()
    out.append(w[w[:, 1] == 1, 2])
  return torch.cat(out)


# --------------------------------------------------------------------------- 1. second-step distribution
@pytest.mark.parametrize('p,q', [(0.25, 4.0), (4.0, 0.25), (0.5, 2.0), (2.0, 0.5), (1 / 8, 8.0)])
def test_second_step_follows_p_q(native, p, q):
  t, v, a, b, c, d, e = range(7)
  ei = _rows({t: [v, a, b], v: [t, a, b, c, d, e]})
  eng = _engine(ei, 7, batch_size=2000, p=p, q=q)
  x = _second_steps(eng, t, 3)                                       # ~ 3 * 20000 / 3 walks through v
  assert x.numel() >= 10_000
  nodes = [t, a, b, c, d, e]
  obs = torch.stack([(x == u).sum() for u in nodes]).double()
  assert int(obs.sum()) == x.numel()                                 # every step 2 is a neighbour of v
  w = torch.tensor([1 / p, 1, 1, 1 / q, 1 / q, 1 / q], dtype=torch.float64)
  pv = chisquare(obs.numpy(), (w / w.sum() * x.numel()).numpy()).pvalue
  print(f'p={p} q={q}: counts {obs.tolist()} chi-square p-value {pv:.3g}')
  assert pv > 1e-3, (pv, obs)


# --------------------------------------------------------------------------- 2. hub rows
@pytest.mark.parametrize('p,q', [(0.25, 4.0), (1 / 8, 8.0)])
def test_hub_rows_follow_p_q(native, p, q):
  """t's row is 1500 copies of v and 1500 common nodes A (3000 entries: half the walks reach v at step 1); v's row is t,
  the 1500 nodes of A and 1500 far nodes F.  Most proposals are rejected and the searches of t's row are 12 deep."""
  h = 1500
  t, v = 0, 1
  A, F = list(range(2, 2 + h)), list(range(2 + h, 2 + 2 * h))
  n = 2 + 2 * h
  eng = _engine(_rows({t: [v] * h + A, v: [t] + A + F}), n, batch_size=1000, p=p, q=q)
  indptr = eng._graphs[0].topo.indptr
  assert int(indptr[1] - indptr[0]) == 2 * h and int(indptr[2] - indptr[1]) == 2 * h + 1
  x = _second_steps(eng, t, 3)                                       # ~ 3 * 10000 / 2 walks through v
  assert x.numel() >= 10_000
  obs = torch.tensor([(x == t).sum(), ((x >= 2) & (x < 2 + h)).sum(), (x >= 2 + h).sum()], dtype=torch.float64)
  assert int(obs.sum()) == x.numel()
  w = torch.tensor([1 / p, h, h / q], dtype=torch.float64)
  pv = chisquare(obs.numpy(), (w / w.sum() * x.numel()).numpy()).pvalue
  print(f'hub p={p} q={q}: return / common / far {obs.tolist()} chi-square p-value {pv:.3g}')
  assert pv > 1e-3, (pv, obs)


# --------------------------------------------------------------------------- 3. valid walks
def _dead_end_graph(n=40, seed=3):
  """Random directed graph on n nodes with rows of 0 to 4 entries: nodes 0 mod 7 have no out-edges."""
  gen = torch.Generator().manual_seed(seed)
  src = torch.arange(n).repeat_interleave(4)
  dst = torch.randint(0, n, (src.numel(),), generator=gen)
  keep = (src % 7 != 0) & (torch.rand(src.numel(), generator=gen) < 0.8)
  return torch.unique(torch.stack([src[keep], dst[keep]]), dim=1)


@pytest.mark.parametrize('L,C', [(1, 2), (5, 3), (30, 6)])
def test_walks_are_edges_with_dead_ends(native, L, C):
  n = 40
  ei = _dead_end_graph(n)
  eng = _engine(ei, n, walk_length=L, context_size=C, walks_per_node=3, batch_size=12, p=0.5, q=3.0)
  starts = torch.tensor([0, 1, 2, 3, 5, 7, -1, 13, 21, 39, -1, 40])    # 40 is outside the type: an empty walk
  eng._stage(starts.to(DEV))
  eng._sample()
  torch.cuda.synchronize()
  _host_walk_checks(eng, {HOMO[0]: ei}, torch.where(starts < n, starts, -1))
  assert bool((eng.walks.view(12, 3, L + 1)[0, :, 1:] == -1).all())   # node 0 is a dead end
  if L > 1:
    assert int(eng.n_valid) > 0


# --------------------------------------------------------------------------- 4. keyed draws
def test_walks_are_keyed_by_seed_and_step(native):
  n = 40
  eng = _engine(_dead_end_graph(n), n, walk_length=12, context_size=3, walks_per_node=4, batch_size=8, p=0.25, q=4.0)
  starts = torch.arange(1, 9, device=DEV)
  walks = torch.empty_like(eng.walks)
  n_valid = torch.zeros(1, dtype=torch.int32, device=DEV)

  def walk(step, seed=0):
    native.node2vec_walk(eng.mp, starts, 4, 3, seed, torch.tensor([step], dtype=torch.int32, device=DEV), walks,
                         n_valid, 0.25, 4.0)
    return walks.clone()
  a = walk(5)
  assert torch.equal(a, walk(5))                                     # bitwise reproducible
  assert not torch.equal(a, walk(6)) and not torch.equal(a, walk(5, seed=1))


def test_captured_steps_match_eager(native):
  N = 300
  gen = torch.Generator().manual_seed(1)
  ei = torch.randint(0, N, (2, 2400), generator=gen)
  ei = torch.unique(torch.cat([ei, ei.flip(0)], 1), dim=1)
  kw = dict(embedding_dim=24, walk_length=11, context_size=4, walks_per_node=3, num_negative_samples=2,
            batch_size=16, seed=11, p=4.0, q=0.25)
  eager = _engine(ei, N, use_cuda_graph=False, **kw)
  graph = _engine(ei, N, use_cuda_graph=True, **kw)
  eager.warmup_and_capture()
  graph.warmup_and_capture()
  assert graph._graph is not None
  la, lb, seen = [], [], []
  for _ in range(5):
    st = torch.randint(0, N, (16,), generator=gen).pin_memory()
    la.append(float(eager.train_step(st)))
    lb.append(float(graph.train_step(st)))
    assert torch.equal(eager.walks, graph.walks) and torch.equal(eager.negatives, graph.negatives)
    seen.append(graph.walks.clone())
  assert not torch.equal(seen[0], seen[1])                           # every replay draws fresh walks
  torch.testing.assert_close(torch.tensor(lb), torch.tensor(la), rtol=1e-4, atol=1e-5)
  torch.testing.assert_close(graph.weight, eager.weight, rtol=1e-4, atol=1e-5)


def test_p_q_one_is_the_deepwalk_path(native):
  n = 40
  ei = _dead_end_graph(n)
  kw = dict(walk_length=9, context_size=3, walks_per_node=3, batch_size=8, seed=4)
  a = _engine(ei, n, p=1.0, q=1.0, **kw)
  b = _engine(ei, n, **kw)
  st = torch.arange(8, device=DEV)
  for eng in (a, b):
    eng.warmup_and_capture()
    eng.train_step(st)
  assert torch.equal(a.walks, b.walks) and torch.equal(a.negatives, b.negatives)
  torch.testing.assert_close(a.weight, b.weight, rtol=1e-5, atol=1e-6)   # red.add order may differ


# --------------------------------------------------------------------------- 5. learning
def test_learns_planted_communities(native):
  k, per = 4, 150
  n = k * per
  gen = torch.Generator().manual_seed(0)
  comm = torch.arange(n) // per
  src = torch.arange(n).repeat_interleave(7)
  own = comm.repeat_interleave(7) * per + torch.randint(0, per, (src.numel(),), generator=gen)
  dst = torch.where(torch.arange(src.numel()) % 7 == 6, torch.randint(0, n, (src.numel(),), generator=gen), own)
  ei = torch.unique(torch.cat([torch.stack([src, dst]), torch.stack([dst, src])], 1), dim=1)
  eng = _engine(ei, n, embedding_dim=32, walk_length=20, context_size=5, walks_per_node=5, num_negative_samples=3,
                batch_size=100, lr=0.05, p=0.5, q=2.0, use_cuda_graph=True)
  eng.warmup_and_capture()
  perm = torch.randperm(n, generator=gen)
  train, test = perm[: n // 2], perm[n // 2:]

  def accuracy():
    e = torch.nn.functional.normalize(eng.embedding('n').cpu(), dim=1)
    cent = torch.stack([e[train][comm[train] == c].mean(0) for c in range(k)])
    return float(((e[test] @ cent.t()).argmax(1) == comm[test]).float().mean())
  acc0 = accuracy()
  losses = []
  for _ in range(30):
    order = torch.randperm(n, generator=gen)
    for i in range(0, n, 100):
      losses.append(float(eng.train_step(order[i:i + 100])))
  acc = accuracy()
  first, last = sum(losses[:6]) / 6, sum(losses[-6:]) / 6
  print(f'node2vec planted communities: loss {first:.3f} -> {last:.3f}, accuracy {acc0:.3f} -> {acc:.3f} '
        f'(chance {1 / k})')
  assert last < 0.5 * first
  assert acc > 0.8


# --------------------------------------------------------------------------- 6. errors
def test_construction_errors_are_value_errors(native):
  n = 40
  g = {HOMO[0]: _graph(_dead_end_graph(n), n)}
  for p, q in [(0.0, 1.0), (1.0, -2.0), (math.nan, 1.0), (1.0, math.inf), (0.1, 10.0), (100.0, 1.0)]:
    with pytest.raises(ValueError):
      MetaPath2VecEngine(g, {'n': n}, HOMO, p=p, q=q, device=DEV)
  MetaPath2VecEngine(g, {'n': n}, HOMO, p=1 / 8, q=8.0, device=DEV)     # r = 64, the bound
  _, graphs, sizes = _typed_graph()
  with pytest.raises(ValueError):                                    # a metapath of three relations
    MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[3]], p=2.0, device=DEV)
  with pytest.raises(ValueError):                                    # one relation between two types
    MetaPath2VecEngine(graphs, sizes, [REL['ab']], walk_length=1, context_size=2, q=2.0, device=DEV)
  MetaPath2VecEngine(graphs, sizes, [REL['ab']], walk_length=1, context_size=2, p=1.0, q=1.0, device=DEV)


def test_binding_raises_on_bad_arguments(native):
  n = 40
  eng = _engine(_dead_end_graph(n), n, walk_length=6, context_size=3, walks_per_node=2, batch_size=4, p=2.0, q=0.5)
  cur = eng.state[2:3]

  def raises(fn, *a):
    with pytest.raises(RuntimeError):
      fn(*a)
  st = eng.starts
  walk = _with_defaults(native.node2vec_walk, (eng.mp, st, 2, 3, 0, cur, eng.walks, eng.n_valid, 2.0, 0.5))
  walk()
  for p, q in [(0.0, 1.0), (-1.0, 1.0), (math.nan, 1.0), (1.0, math.inf), (1.0, 0.0), (0.1, 10.0), (65.0, 1.0)]:
    raises(walk, *([None] * 8), p, q)
  walk(*([None] * 8), 1 / 8, 8.0)                                    # r = 64 is accepted
  raises(walk, None, st.int())
  raises(walk, None, st.cpu())
  raises(walk, None, None, 3)                                        # walks rows != starts * walks_per_node
  raises(walk, None, None, 0)
  raises(walk, None, None, None, 8)                                  # context beyond walk_length + 1
  raises(walk, None, None, None, 1)
  raises(walk, None, None, None, None, None, cur.long())
  raises(walk, None, None, None, None, None, cur.cpu())
  raises(walk, None, None, None, None, None, None, eng.walks.cpu())
  raises(walk, None, None, None, None, None, None, eng.walks.int())
  raises(walk, None, None, None, None, None, None, eng.walks[:, :1].contiguous())
  raises(walk, None, None, None, None, None, None, None, eng.n_valid.float())
  long_walks = torch.empty(1, (1 << 20) + 2, dtype=torch.int64, device=DEV)   # draw counters would wrap
  raises(walk, None, st[:1], 1, 2, None, None, long_walks)
  _, graphs, sizes = _typed_graph()
  typed = MetaPath2VecEngine(graphs, sizes, [REL[r] for r in PATHS[3]], walk_length=6, context_size=3,
                             walks_per_node=2, batch_size=4, device=DEV)
  raises(walk, typed.mp, typed.starts, None, None, None, None, typed.walks)            # R = 3
  ab = MetaPath2VecEngine(graphs, sizes, [REL['ab']], walk_length=1, context_size=2, walks_per_node=2, batch_size=4,
                          device=DEV)
  raises(walk, ab.mp, ab.starts, None, 2, None, None, ab.walks)                         # a -> b
  torch.cuda.synchronize()


# --------------------------------------------------------------------------- 7. example
def test_example_runs(native):
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
  import node2vec
  res = node2vec.main(['--nodes', '3000', '--edges', '30000', '--p', '0.5', '--q', '2', '--embedding-dim', '16',
                       '--walk-length', '8', '--context-size', '4', '--walks-per-node', '2', '--batch-size', '256'])
  assert math.isfinite(res['loss']) and 0 <= res['valid_acc'] <= 1 and 0 <= res['test_acc'] <= 1
