"""KgeEngine: Philox negatives, the fused loss / gradient against float64 autograd of the transcribed formulas, SparseAdam
against torch.optim.SparseAdam, capture, score(), filtered and raw ranks against float64 brute force, learning on
synthetic_kg, checkpoints, the bindings' argument errors and the example."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from graphlearn_for_pytorch_b200.models import KgeEngine, kge_filter
from graphlearn_for_pytorch_b200.utils.synthetic import synthetic_kg

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
MODELS = ['transe', 'distmult', 'complex', 'rotate']
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------- float64 transcriptions
def ref_score(model, ent, rel, h, r, t, D, margin=1.0, p=1):
  E, Rl = ent, rel
  if model == 'transe':
    x = F.normalize(E[h], p=p, dim=-1) + Rl[r] - F.normalize(E[t], p=p, dim=-1)
    return -torch.linalg.vector_norm(x, ord=p, dim=-1)
  if model == 'distmult':
    return (E[h] * Rl[r] * E[t]).sum(-1)
  hr, hi, tr, ti = E[h][:, :D], E[h][:, D:], E[t][:, :D], E[t][:, D:]
  if model == 'complex':
    rr, ri = Rl[r][:, :D], Rl[r][:, D:]
    return (hr * rr * tr + hi * rr * ti + hr * ri * ti - hi * ri * tr).sum(-1)
  th = Rl[r]
  a = torch.cos(th) * hr - torch.sin(th) * hi - tr
  b = torch.cos(th) * hi + torch.sin(th) * hr - ti
  return margin - torch.linalg.vector_norm(torch.cat([a, b], -1), dim=-1)


def corrupt(trip, neg):
  """(heads, rels, tails) [n, K] of the corrupted triples: head replaced for i < n // 2, tail otherwise."""
  n, K = neg.shape
  h, r, t = (x.unsqueeze(1).expand(n, K) for x in trip)
  head = (torch.arange(n, device=neg.device) < n // 2).unsqueeze(1)
  return torch.where(head, neg, h), r, torch.where(head, t, neg)


def ref_loss(model, ent, rel, trip, neg, D, margin=1.0, p=1):
  n, K = neg.shape
  s_pos = ref_score(model, ent, rel, *trip, D, margin, p)
  nh, nr, nt = corrupt(trip, neg)
  s_neg = ref_score(model, ent, rel, nh.reshape(-1), nr.reshape(-1), nt.reshape(-1), D, margin, p).view(n, K)
  if model in ('transe', 'distmult'):
    return torch.clamp(margin - s_pos.unsqueeze(1) + s_neg, min=0).sum() / (n * K)
  return (F.softplus(-s_pos).sum() + F.softplus(s_neg).sum()) / (n + n * K)


def _engine(model, N=300, R=7, D=32, K=3, B=64, seed=0, **kw):
  return KgeEngine(N, R, model=model, hidden_channels=D, num_negatives=K, batch_size=B, seed=seed, device=DEV, **kw)


def _triples(N, R, n, seed=1, rel=None):
  g = torch.Generator().manual_seed(seed)
  h, t = torch.randint(0, N, (n,), generator=g), torch.randint(0, N, (n,), generator=g)
  r = torch.randint(0, R, (n,), generator=g) if rel is None else torch.full((n,), rel)
  return torch.stack([h, r, t])


def _run_stages(eng, trip):
  eng._stage(trip.to(DEV))
  eng._sample()
  eng._loss_grad()
  torch.cuda.synchronize()


def _ref_grads(eng, trip):
  n = trip.size(1)
  ent = eng.ent.double().cpu().requires_grad_()
  rel = eng.rel.double().cpu().requires_grad_()
  neg = eng.negatives[:n].cpu()
  loss = ref_loss(eng.model, ent, rel, tuple(trip), neg, eng.hidden_channels, eng.margin, eng.p_norm)
  loss.backward()
  return loss.detach(), ent.grad, rel.grad, neg


# ---------------------------------------------------------------------------------------------- negatives
@pytest.mark.parametrize('model', MODELS)
@pytest.mark.parametrize('n', [1, 7, 8, 64])
def test_negatives_rule_and_padding(model, n):
  eng = _engine(model, K=5, B=64, use_cuda_graph=False)
  trip = _triples(300, 7, n)
  _run_stages(eng, trip)
  neg = eng.negatives.cpu()
  assert (neg[n:] == -1).all(), 'padding slots must stay untouched'
  assert ((neg[:n] >= 0) & (neg[:n] < 300)).all()
  nh, nr, nt = corrupt(tuple(trip), neg[:n])
  assert torch.equal(nr, trip[1].unsqueeze(1).expand(n, 5))
  head = torch.arange(n) < n // 2
  assert torch.equal(nt[head], trip[2, head].unsqueeze(1).expand(-1, 5))
  assert torch.equal(nh[~head], trip[0, ~head].unsqueeze(1).expand(-1, 5))


@pytest.mark.parametrize('model', MODELS)
def test_negatives_deterministic_per_step(model):
  a, b = _engine(model, use_cuda_graph=False), _engine(model, use_cuda_graph=False)
  trip = _triples(300, 7, 64)
  outs = []
  for eng in (a, b):
    got = []
    for _ in range(2):
      _run_stages(eng, trip)
      got.append(eng.negatives.clone())
      eng._update()
    outs.append(got)
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
  assert not torch.equal(outs[0][0], outs[0][1])


def test_negatives_uniform_chi_square():
  N = 50
  eng = KgeEngine(N, 3, model='distmult', hidden_channels=8, num_negatives=64, batch_size=4096, device=DEV,
                  use_cuda_graph=False)
  _run_stages(eng, _triples(N, 3, 4096))
  counts = torch.bincount(eng.negatives.flatten().cpu(), minlength=N).double()
  exp = counts.sum() / N
  chi2 = float(((counts - exp) ** 2 / exp).sum())
  # 49 degrees of freedom: P(chi2 > 100) < 1e-5
  assert chi2 < 100, chi2


# ---------------------------------------------------------------------------------------------- loss and gradient
def _check_loss_grad(eng, trip):
  n = trip.size(1)
  _run_stages(eng, trip)
  loss, g_ent, g_rel, neg = _ref_grads(eng, trip)
  torch.testing.assert_close(eng.loss.double().cpu()[0], loss, rtol=1e-4, atol=1e-6)
  for got, ref in ((eng.grad_ent, g_ent), (eng.grad_rel, g_rel)):
    scale = float(ref.abs().max()) + 1e-30
    torch.testing.assert_close(got.double().cpu(), ref, rtol=1e-3, atol=2e-4 * scale)
  rows = torch.cat([trip[0], trip[2], neg.flatten()]).unique() if n else torch.empty(0, dtype=torch.long)
  t_ent = torch.zeros(eng.num_nodes, dtype=torch.uint8)
  t_ent[rows] = 1
  t_rel = torch.zeros(eng.num_relations, dtype=torch.uint8)
  t_rel[trip[1]] = 1
  assert torch.equal(eng.touched_ent.cpu(), t_ent)
  assert torch.equal(eng.touched_rel.cpu(), t_rel)


@pytest.mark.parametrize('model', MODELS)
@pytest.mark.parametrize('D', [8, 24, 64, 200, 512])
@pytest.mark.parametrize('K', [1, 3, 64])
def test_loss_grad_against_float64(model, D, K):
  eng = _engine(model, N=257, R=5, D=D, K=K, B=48, use_cuda_graph=False)
  trip = _triples(257, 5, 45)
  trip[0, 3] = trip[2, 3] = trip[0, 10]     # repeated entities, a self-loop
  _check_loss_grad(eng, trip)


@pytest.mark.parametrize('model', MODELS)
@pytest.mark.parametrize('D', [16, 256])
def test_loss_grad_one_relation(model, D):
  """Every positive shares relation 2: the CTA's pre-reduced relation row carries all of them."""
  eng = _engine(model, N=1000, R=4, D=D, K=4, B=1024, use_cuda_graph=False)
  _check_loss_grad(eng, _triples(1000, 4, 1000, rel=2))


@pytest.mark.parametrize('p', [1, 2])
def test_transe_norms_and_zero_rows(p):
  # margin 2: with r = 0 and a zero tail, a corrupted head scores exactly -1 (a unit row), which would put the margin
  # term of the default margin at exactly 0, where fp32 and float64 may fall on different sides
  eng = _engine('transe', N=64, R=3, D=24, K=3, B=32, p_norm=p, margin=2.0, use_cuda_graph=False)
  eng.ent[:6] = 0                          # zero rows: the clamped normalisation and a norm's zero gradient
  eng.ent[6:9] *= 1e-14                    # below the eps: clamped
  eng.rel[1] = 0
  trip = torch.tensor([[0, 1, 6, 7, 20, 21, 2, 30, 8, 3, 40, 41],
                       [1, 1, 0, 1, 2, 1, 0, 1, 1, 2, 0, 2],
                       [1, 0, 7, 6, 22, 23, 2, 8, 30, 3, 41, 40]])
  _check_loss_grad(eng, trip)


@pytest.mark.parametrize('model', MODELS)
def test_empty_batch(model):
  eng = _engine(model, use_cuda_graph=False)
  before = eng.ent.clone()
  loss = eng.train_step(torch.empty(3, 0, dtype=torch.int64))
  torch.cuda.synchronize()
  assert float(loss) == 0.0
  assert torch.equal(eng.ent, before)
  assert int(eng.touched_ent.sum()) == 0 and int(eng.grad_ent.abs().sum()) == 0


# ---------------------------------------------------------------------------------------------- SparseAdam, capture
@pytest.mark.parametrize('model', MODELS)
def test_sparse_adam_three_steps(model):
  # TransE at p = 2: at p = 1 a gradient entry that cancels exactly in float64 (a sum of +-1 / (n K)) can keep an fp32
  # residue, which Adam scales up to about lr * residue / (|residue| + eps); p = 1 gradients are checked above
  eng = _engine(model, N=200, R=6, D=16, K=2, B=40, use_cuda_graph=False, p_norm=2)
  params = [torch.nn.Parameter(eng.ent.double().cpu()), torch.nn.Parameter(eng.rel.double().cpu())]
  opt = torch.optim.SparseAdam(params, lr=eng.lr, betas=eng.betas, eps=eng.eps)
  for step in range(3):
    trip = _triples(200, 6, 40, seed=10 + step)
    before = eng.ent.clone()
    _run_stages(eng, trip)
    _, g_ent, g_rel, _ = _ref_grads(eng, trip)
    touched = (eng.touched_ent.bool().cpu(), eng.touched_rel.bool().cpu())
    eng._update()
    torch.cuda.synchronize()
    for prm, g, tch in zip(params, (g_ent, g_rel), touched):
      idx = tch.nonzero().flatten()
      prm.grad = torch.sparse_coo_tensor(idx.unsqueeze(0), g[idx], prm.shape)
    opt.step()
    for got, prm in zip((eng.ent, eng.rel), params):
      torch.testing.assert_close(got.double().cpu(), prm.detach(), rtol=1e-4, atol=2e-5)
    untouched = ~touched[0]
    assert torch.equal(eng.ent[untouched.to(DEV)], before[untouched.to(DEV)])
    assert int(eng.touched_ent.sum()) == 0 and int(eng.grad_ent.abs().sum()) == 0
    # continue both from the engine's fp32 tables so only one step's rounding is compared
    with torch.no_grad():
      params[0].copy_(eng.ent.double().cpu())
      params[1].copy_(eng.rel.double().cpu())


@pytest.mark.parametrize('model', MODELS)
def test_captured_matches_eager(model):
  # p = 2 for TransE, for the reason given in test_sparse_adam_three_steps: replays and eager steps add the same
  # gradients in different orders
  a, b = _engine(model, p_norm=2), _engine(model, use_cuda_graph=False, p_norm=2)
  a.warmup_and_capture()
  b.warmup_and_capture()
  assert a._graph is not None and b._graph is None
  assert a.kernels_per_step == b.kernels_per_step
  for step in range(4):
    trip = _triples(300, 7, 64 - step, seed=step).pin_memory()
    la, lb = a.train_step(trip), b.train_step(trip)
    torch.testing.assert_close(la, lb, rtol=1e-5, atol=1e-6)
  torch.testing.assert_close(a.ent, b.ent, rtol=1e-5, atol=1e-6)
  torch.testing.assert_close(a.rel, b.rel, rtol=1e-5, atol=1e-6)
  assert torch.equal(a.state, b.state)


# ---------------------------------------------------------------------------------------------- score, rank
@pytest.mark.parametrize('model', MODELS)
@pytest.mark.parametrize('D', [8, 72, 512])
def test_score_against_float64(model, D):
  eng = _engine(model, D=D, use_cuda_graph=False)
  trip = _triples(300, 7, 333)
  got = eng.score(*trip).double().cpu()
  ref = ref_score(model, eng.ent.double().cpu(), eng.rel.double().cpu(), *trip, D, eng.margin, eng.p_norm)
  torch.testing.assert_close(got, ref, rtol=1e-5, atol=1e-5)


def _brute_scores(eng, h, r, t, mode):
  """float64 [n, N] scores of every candidate entity in the query's open slot."""
  N = eng.num_nodes
  ent, rel = eng.ent.double().cpu(), eng.rel.double().cpu()
  n = h.numel()
  c = torch.arange(N).repeat(n)
  hh = c if mode == 'head' else h.repeat_interleave(N)
  tt = c if mode == 'tail' else t.repeat_interleave(N)
  s = ref_score(eng.model, ent, rel, hh, r.repeat_interleave(N), tt, eng.hidden_channels, eng.margin, eng.p_norm)
  return s.view(n, N)


def _allowed(eng, h, r, t, mode, known):
  """bool [n, N]: candidates that count (not the true entity, not filtered)."""
  n, N = h.numel(), eng.num_nodes
  ok = torch.ones(n, N, dtype=torch.bool)
  truth = t if mode == 'tail' else h
  ok[torch.arange(n), truth] = False
  if known is not None:
    for i in range(n):
      if mode == 'tail':
        m = (known[0] == h[i]) & (known[1] == r[i])
        ok[i, known[2, m]] = False
      else:
        m = (known[2] == t[i]) & (known[1] == r[i])
        ok[i, known[0, m]] = False
  return ok, truth


def _int_tables(eng, seed=3):
  g = torch.Generator().manual_seed(seed)
  eng.ent.copy_(torch.randint(-2, 3, eng.ent.shape, generator=g).float())
  eng.rel.copy_(torch.randint(-2, 3, eng.rel.shape, generator=g).float())


def _known(N, R, q, seed=5):
  """Known triples: the queries themselves, random triples sharing their (h, r) / (r, t), and duplicates."""
  g = torch.Generator().manual_seed(seed)
  extra = []
  for i in range(q.size(1)):
    k = int(torch.randint(0, 6, (1,), generator=g))
    extra.append(torch.stack([q[0, i].repeat(k), q[1, i].repeat(k), torch.randint(0, N, (k,), generator=g)]))
    extra.append(torch.stack([torch.randint(0, N, (k,), generator=g), q[1, i].repeat(k), q[2, i].repeat(k)]))
  kn = torch.cat([q] + extra + [q[:, :3]], 1)
  return kn


@pytest.mark.parametrize('model', ['distmult', 'complex'])
@pytest.mark.parametrize('N', [37, 64, 200])
@pytest.mark.parametrize('n', [1, 150])
@pytest.mark.parametrize('filtered', [False, True])
def test_rank_exact_on_integer_tables(model, N, n, filtered):
  eng = _engine(model, N=N, R=4, D=16, use_cuda_graph=False)
  _int_tables(eng)
  q = _triples(N, 4, n, seed=N + n)
  known = _known(N, 4, q) if filtered else None
  flt = kge_filter(known.to(DEV), N, 4) if filtered else None
  for mode in ('tail', 'head'):
    got = eng.rank(*q, mode=mode, filter=flt).cpu()
    s = _brute_scores(eng, *q, mode)
    ok, truth = _allowed(eng, *q, mode, known)
    st = s[torch.arange(n), truth].unsqueeze(1)
    ref = 1 + ((s > st) & ok).sum(1).double() + 0.5 * ((s == st) & ok).sum(1).double()
    assert torch.equal(got, ref), (mode, got[:8], ref[:8])
    assert float(((s == st) & ok).sum()) > 0 or n == 1   # the integer tables do tie


@pytest.mark.parametrize('model', ['transe', 'rotate'])
@pytest.mark.parametrize('N', [37, 200])
@pytest.mark.parametrize('filtered', [False, True])
def test_rank_band_on_random_tables(model, N, filtered):
  eng = _engine(model, N=N, R=4, D=40, use_cuda_graph=False)
  q = _triples(N, 4, 70, seed=N)
  known = _known(N, 4, q) if filtered else None
  flt = kge_filter(known.to(DEV), N, 4) if filtered else None
  tol = 1e-4
  for mode in ('tail', 'head'):
    got = eng.rank(*q, mode=mode, filter=flt).cpu()
    s = _brute_scores(eng, *q, mode)
    ok, truth = _allowed(eng, *q, mode, known)
    st = s[torch.arange(70), truth].unsqueeze(1)
    lo = 1 + ((s > st + tol) & ok).sum(1).double()
    hi = 1 + ((s > st - tol) & ok).sum(1).double()
    assert ((got >= lo) & (got <= hi)).all(), (mode, got, lo, hi)


@pytest.mark.parametrize('model', MODELS)
def test_rank_split_invariance_and_edges(model):
  N = 1000
  eng = _engine(model, N=N, R=5, D=24, use_cuda_graph=False)
  if model in ('distmult', 'complex'):
    _int_tables(eng)
  q = _triples(N, 5, 300, seed=7)
  flt = kge_filter(_known(N, 5, q).to(DEV), N, 5)
  for mode in ('tail', 'head'):
    ref = eng.rank(*q, mode=mode, filter=flt)
    for s in (1, 3, 16):
      assert torch.equal(eng.rank(*q, mode=mode, filter=flt, _splits=s), ref)
  assert eng.rank(*(x[:0] for x in q)).numel() == 0
  # a query whose filter removes every other entity ranks first
  h, r, t = 5, 2, 9
  all_known = torch.stack([torch.full((N,), h), torch.full((N,), r), torch.arange(N)])
  flt = kge_filter(all_known.to(DEV), N, 5)
  assert eng.rank([h], [r], [t], mode='tail', filter=flt).tolist() == [1.0]
  all_known = torch.stack([torch.arange(N), torch.full((N,), r), torch.full((N,), t)])
  flt = kge_filter(all_known.to(DEV), N, 5)
  assert eng.rank([h], [r], [t], mode='head', filter=flt).tolist() == [1.0]


@pytest.mark.parametrize('model', MODELS)
def test_test_metrics_from_ranks(model):
  eng = _engine(model, use_cuda_graph=False)
  q = _triples(300, 7, 90)
  flt = kge_filter(q.to(DEV), 300, 7)
  ranks = torch.cat([eng.rank(*q, mode='tail', filter=flt), eng.rank(*q, mode='head', filter=flt)]).cpu()
  mr, mrr, hits = eng.test(*q, k=10, filter=flt)
  assert mr == pytest.approx(float(ranks.mean()))
  assert mrr == pytest.approx(float((1 / ranks).mean()))
  assert hits == pytest.approx(float((ranks <= 10).double().mean()))
  rt = eng.rank(*q, mode='tail', filter=flt).cpu()
  assert eng.test(*q, k=3, filter=flt, mode='tail')[2] == pytest.approx(float((rt <= 3).double().mean()))


# ---------------------------------------------------------------------------------------------- learning, checkpoints
@pytest.mark.parametrize('model', MODELS)
def test_learns_planted_structure(model):
  # trained ranks depend on the cluster size (8), the untrained baseline on N.  DistMult cannot tell a tail cluster from
  # the head cluster's predecessor, so its trained MRR is about half the others'; it gets twice the entities, which
  # halves its baseline
  N, R = (800, 3) if model == 'distmult' else (400, 3)
  train, valid, test = synthetic_kg(N, R, 15 * N, seed=0)
  flt = kge_filter(torch.cat([train, valid, test], 1).to(DEV), N, R)
  eng = KgeEngine(N, R, model=model, hidden_channels=32, num_negatives=16, batch_size=512, lr=0.05, seed=0,
                  device=DEV)
  eng.warmup_and_capture()
  _, mrr0, hits0 = eng.test(*test, k=10, filter=flt)
  g = torch.Generator().manual_seed(0)
  for _ in range(80):
    perm = torch.randperm(train.size(1), generator=g)
    for b in range(0, train.size(1), 512):
      eng.train_step(train[:, perm[b:b + 512]].contiguous().to(DEV))
  _, mrr1, hits1 = eng.test(*test, k=10, filter=flt)
  assert hits1 >= 10 * hits0 and mrr1 >= 10 * mrr0, (hits0, hits1, mrr0, mrr1)


@pytest.mark.parametrize('model', MODELS)
def test_state_dict_round_trip(model):
  a = _engine(model)
  a.warmup_and_capture()
  for step in range(3):
    a.train_step(_triples(300, 7, 64, seed=step).to(DEV))
  sd = a.state_dict()
  names = {'transe': {'node_emb.weight', 'rel_emb.weight'}, 'distmult': {'node_emb.weight', 'rel_emb.weight'},
           'complex': {'node_emb.weight', 'node_emb_im.weight', 'rel_emb.weight', 'rel_emb_im.weight'},
           'rotate': {'node_emb.weight', 'node_emb_im.weight', 'rel_emb.weight'}}[model]
  assert set(sd['model']) == names
  assert all(v.shape == (300 if k.startswith('node') else 7, 32) for k, v in sd['model'].items())
  b = _engine(model)                       # the seed keys the negatives; the tables and counters come from sd
  b.warmup_and_capture()
  b.load_state_dict(sd)
  q = _triples(300, 7, 50, seed=99)
  assert torch.equal(a.score(*q), b.score(*q))
  trip = _triples(300, 7, 64, seed=42).to(DEV)
  a.train_step(trip)
  b.train_step(trip)
  torch.cuda.synchronize()
  assert torch.equal(a.negatives, b.negatives)
  torch.testing.assert_close(a.ent, b.ent, rtol=1e-5, atol=1e-6)


# ---------------------------------------------------------------------------------------------- bindings, example
def test_binding_argument_errors(native):
  eng = _engine('complex', use_cuda_graph=False)
  ent, rel = eng.ent, eng.rel
  ids = torch.zeros(4, dtype=torch.int64, device=DEV)
  cases = [
    lambda: native.kge_score(2, ent.double(), rel, ids, ids, ids, 1.0, 1),           # dtype
    lambda: native.kge_score(2, ent[:, :24], rel, ids, ids, ids, 1.0, 1),             # width
    lambda: native.kge_score(2, ent, rel[:, :8], ids, ids, ids, 1.0, 1),              # relation width
    lambda: native.kge_score(5, ent, rel, ids, ids, ids, 1.0, 1),                     # model
    lambda: native.kge_score(2, ent, rel, ids.cpu(), ids, ids, 1.0, 1),               # device
    lambda: native.kge_score(2, ent, rel, ids.int(), ids, ids, 1.0, 1),               # id dtype
    lambda: native.kge_score(2, ent, rel, ids[:3], ids, ids, 1.0, 1),                 # shape
    lambda: native.kge_score(2, ent, rel, ids + 300, ids, ids, 1.0, 1),               # entity id
    lambda: native.kge_score(2, ent, rel, ids, ids - 1, ids, 1.0, 1),                 # relation id
    lambda: native.kge_rank(2, ent, rel, ids, ids, ids, True, ids.float(), 1.0, 1),   # keys dtype
    lambda: native.kge_rank(2, ent, rel, ids, ids, ids, True, None, 1.0, 3),          # p
    lambda: native.kge_rank(2, ent, rel, ids, ids, ids, True, None, 1.0, 1, -1),      # splits
    lambda: native.kge_negatives(eng.count, 64, 3, 300, 0, eng.state[2:3], eng.negatives[:, :2]),
    lambda: native.kge_negatives(eng.count.float(), 64, 3, 300, 0, eng.state[2:3], eng.negatives),
    lambda: native.kge_negatives(eng.count, 64, 3, 0, 0, eng.state[2:3], eng.negatives),
    lambda: native.kge_loss_grad(2, eng.trip[:2], eng.count, eng.negatives, ent, rel, 1.0, 1, eng.grad_ent,
                                 eng.grad_rel, eng.touched_ent, eng.touched_rel, eng.loss),
    lambda: native.kge_loss_grad(2, eng.trip, eng.count, eng.negatives, ent, rel, 1.0, 1, eng.grad_rel,
                                 eng.grad_rel, eng.touched_ent, eng.touched_rel, eng.loss),
    lambda: native.kge_loss_grad(2, eng.trip, eng.count, eng.negatives, ent, rel, 1.0, 1, eng.grad_ent,
                                 eng.grad_rel, eng.touched_rel, eng.touched_rel, eng.loss),
    lambda: native.kge_loss_grad(2, eng.trip, eng.count, eng.negatives[:10], ent, rel, 1.0, 1, eng.grad_ent,
                                 eng.grad_rel, eng.touched_ent, eng.touched_rel, eng.loss),
    lambda: native.kge_loss_grad(2, eng.trip, eng.count, eng.negatives, ent, rel, 1.0, 1, eng.grad_ent,
                                 eng.grad_rel, eng.touched_ent, eng.touched_rel, eng.loss.double()),
    lambda: native.kge_sparse_adam(ent, eng.grad_ent, eng.exp_avg_rel, eng.exp_avg_sq_ent, eng.touched_ent,
                                   eng.state[1:2], 0.01, 0.9, 0.999, 1e-8),
    lambda: native.kge_sparse_adam(ent, eng.grad_ent, eng.exp_avg_ent, eng.exp_avg_sq_ent, eng.touched_ent,
                                   eng.state[1:2], -1.0, 0.9, 0.999, 1e-8),
    lambda: native.kge_sparse_adam(ent.cpu(), eng.grad_ent, eng.exp_avg_ent, eng.exp_avg_sq_ent, eng.touched_ent,
                                   eng.state[1:2], 0.01, 0.9, 0.999, 1e-8),
  ]
  for i, f in enumerate(cases):
    with pytest.raises(RuntimeError):
      f()
      pytest.fail(f'case {i} did not raise')


def test_engine_argument_errors_on_use():
  eng = _engine('transe', use_cuda_graph=False)
  with pytest.raises(ValueError):
    eng.train_step(torch.zeros(3, 65, dtype=torch.int64))
  with pytest.raises(ValueError):
    eng.train_step(torch.zeros(2, 4, dtype=torch.int64))
  with pytest.raises(ValueError):
    eng.rank([0], [0], [0], mode='both')


def test_example_runs():
  out = subprocess.run([sys.executable, os.path.join(ROOT, 'examples', 'kge.py'), '--model', 'rotate', '--epochs', '2',
                        '--num-nodes', '200', '--num-relations', '3', '--num-triples', '2000',
                        '--hidden-channels', '16'], capture_output=True, text=True, cwd=ROOT, timeout=600)
  assert out.returncode == 0, out.stderr[-2000:]
  assert 'valid' in out.stdout and 'test' in out.stdout and 'Hits@10' in out.stdout, out.stdout
