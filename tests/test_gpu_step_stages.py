"""Every stage of a real GraphSAGE, link-prediction and R-SAGE training step against float64, over consecutive steps.

The kernel tests check each kernel on hand-built batches.  Here the engines run their public `train_step` (eager,
captured into a CUDA graph, or pipelined) and every stage of the step is then recomputed in float64 from that stage's
actual inputs, as the step left them in the engine's buffers: the aggregation from the arena's ELL hops and the source
rows, the linear layer from the aggregation operand and the pre-step bf16 weights, the loss from the logits, the
weight and input gradients from dPre and the operands, the gather backward / scatter from dA, Adam from the pre-step
parameters, moments and the step's gradient.  Because every stage is fed its real inputs, its bound is the kernel
test's bound (tests/helpers.py) and errors do not compound, so a wiring error (a dropped hop, a block credited to the
wrong type, a stale row, a missing weight decay) stands out.

Each configuration runs four steps with batches of bs, about bs / 3 (padded with -1), 1 and bs seeds, so that steps 2
and 3 run far below the previous step's row counts, on top of its rows: rows [T, cap) of dPre must be exactly zero
(the split-K weight-gradient GEMM reads dPre up to the next 64-row k-block past T).

Adam is checked against torch.optim.Adam(weight_decay=wd) semantics in float64 with the fp32 values of lr, beta1,
beta2, eps and wd that the kernel receives; its bound follows the fp32 roundings of the update (u = 2^-24 per
operation, one u for each bias correction).

Negative controls apply the same checks to perturbed copies of a real step's buffers and show that each check
rejects the defect it exists for.  `-s` prints the worst error / bound ratio per stage, configuration and step.
"""
import math

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.data import dequantize_mxfp8, quantize_mxfp8
from graphlearn_for_pytorch_b200.models import GraphSageEngine, GraphSageLinkEngine, HeteroSageEngine
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges
from helpers import (Ratios, _batches, _check_adam, _check_grads, _check_linear, _check_softmax, _ell_edges, _f32,
                     _snapshot, _table, _wgrad_ratio, bound_ratio, colsum_ratio, gather_ref, mean_ref, sum_bound)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


# --------------------------------------------------------------------------- stages shared by the engines
# --------------------------------------------------------------------------- GraphSageEngine / GraphSageLinkEngine
def _sage_stages(R, eng, snap, parity, X, Xself, labels, controls):
  """Every stage of the step that trained arena `parity`.  X: fp32/bf16 feature table indexed by global id (the
  de-quantised table for MXFP8), Xself: its bf16 rows as the self half holds them."""
  torch.cuda.synchronize()
  ar, L = eng._arenas[parity], eng.L
  c = ar.counters[:L + 2].tolist()
  W = lambda l: eng.W(l, snap['p16'])
  b = lambda l: eng.b(l, snap['p16'])
  gscale = 1.0 / (1.0 - eng.dropout)
  nodes = ar.nodes
  Ts = [None] + [min(c[L - l + 1], eng.Z[l].shape[0]) for l in range(1, L + 1)]
  for l in range(1, L + 1):
    nh = L - l + 1
    A, T, d = eng._A(l, parity), Ts[l], eng.dims_in[l - 1]
    # aggregation: mean over the hops 0..nh-1 of the feature rows (l = 1) or of Z[l-1]; self half bit-exact
    tgt, src = _ell_edges(lambda h: ar.ell[h], ar.deg, c, nh, eng.cap_rows, eng.fanouts)
    keep = tgt < T
    tgt, src = tgt[keep], src[keep]
    if l == 1:
      ref, bound = mean_ref(X, tgt, nodes[src], ar.deg[:T])
      self_ok = torch.equal(A[:T, d:], Xself[nodes[:T]])
    else:
      assert src.numel() == 0 or int(src.max()) < eng.Z[l - 1].shape[0], f'layer {l}: a source row past Z[{l - 1}]'
      ref, bound = mean_ref(eng.Z[l - 1], tgt, src, ar.deg[:T])
      self_ok = torch.equal(A[:T, d:], eng.Z[l - 1][:T])
    R.check(f'agg{l}', bound_ratio(A[:T, :d], ref, bound))
    R.exact(f'self{l}', self_ok)
    if controls and l == 1:
      bad = A[:T, :d].clone()
      bad[c[nh - 1]:T] = 0                                   # layer 1 without its deepest hop
      assert bound_ratio(bad, ref, bound) > 1.0, 'the aggregation check must reject a dropped hop'
    # linear: bf16(act(A W^T + b)) with the pre-step weights; hidden layers then run inverted dropout
    keep, scale = None, 1.0
    if eng.dropout > 0 and l < L:
      ones = torch.ones_like(eng.Z[l])
      eng.nat.dropout_bf16(ones, ar.counters, nh, eng.dropout, eng.seed, l, snap['step'])
      keep, scale = ones[:T] != 0, _f32(gscale)
    _check_linear(R, f'Z{l}', A, W(l), b(l), eng.Z[l], T, l < L, keep, scale)
  # loss
  boff, bn = eng._b_off[L - 1]
  n0 = Ts[L]
  if isinstance(eng, GraphSageLinkEngine):
    _check_link_loss(R, eng, ar, parity, n0, eng.g32[boff:boff + bn])
  else:
    _check_softmax(R, eng.Z[L], eng.C, labels, nodes, n0, eng.dPre[L], eng.g32[boff:boff + bn], eng.loss,
                   eng.correct)
  # backward, layer by layer
  for l in range(L, 0, -1):
    nh = L - l + 1
    A, T, d = eng._A(l, parity), Ts[l], eng.dims_in[l - 1]
    off, n, k = eng._w_off[l - 1]
    gW = eng.g32[off:off + n * k].view(n, k)
    _check_grads(R, l, gW, eng.dPre[l], A, W(l), eng.dA[l] if l > 1 else None, T)
    if l == L:
      R.exact('dW pad rows', bool((gW[eng.C:] == 0).all()))
    if controls and T + 64 <= A.shape[0]:
      # a dPre tail left from the previous, larger batch would add its products with the stale A rows
      prev = snap['dPre'][l]
      bad = gW + (prev[T:T + 64].float().t() @ A[T:T + 64].float())
      assert bool(prev[T:T + 64].any()), 'the control needs a larger previous batch'
      assert _wgrad_ratio(bad, eng.dPre[l], A, T) > 1.0, 'the weight-gradient check must reject a stale dPre tail'
    if l > 1:
      S = min(c[nh + 1], eng.dPre[l - 1].shape[0])
      tgt, src = _ell_edges(lambda h: ar.ell[h], ar.deg, c, nh, eng.cap_rows, eng.fanouts)
      dP = eng.dPre[l - 1]
      ref, bound = gather_ref(eng.dA[l], eng.hidden, eng.Z[l - 1], tgt, src, ar.deg, T, S, dP.shape[0], gscale)
      R.check(f'dPre{l - 1}', bound_ratio(dP, ref, bound))
      pboff, pn = eng._b_off[l - 2]
      R.check(f'db{l - 1}', colsum_ratio(eng.g32[pboff:pboff + pn], dP, S))
      if controls and eng.dropout > 0:
        bad = (dP.float() / _f32(gscale)).to(torch.bfloat16)
        assert bound_ratio(bad, ref, bound) > 1.0, 'the gather check must reject a backward without the dropout scale'
  for l in range(1, L + 1):
    R.exact(f'dPre{l} tail', bool((eng.dPre[l][Ts[l]:] == 0).all()))
  _check_adam(R, eng, snap, eng.wd, controls and eng.wd > 0)
  for l in range(1, L + 1):
    if eng.fused_ok[l]:
      R.exact(f'w_packed{l}', torch.equal(eng.w_packed[l].view(torch.int16),
                                          eng.nat.pack_weight(eng.W(l)).flatten().view(torch.int16)))


def _check_link_loss(R, eng, ar, parity, R_rows, bias_grad):
  """Mean BCE-with-logits over the valid (source, target) pairs of arena.seed_local; dZ32 against autograd, dPre[L]
  its bf16 cast, rows past the batch zero."""
  P, B, C, L = eng.P, eng.pos_bs, eng.C, eng.L
  sl = ar.seed_local
  valid = (sl[:P] >= 0) & (sl[P:] >= 0)
  R.exact('n_pairs', int(eng._n_pairs[parity].item()) == int(valid.sum()))
  Zd = eng.Z[L][:, :C].double().requires_grad_(True)
  ls, lt = sl[:P].long()[valid], sl[P:].long()[valid]
  y = (torch.arange(P, device=DEV) < B).double()[valid]
  s = (Zd[ls] * Zd[lt]).sum(-1)
  ref = F.binary_cross_entropy_with_logits(s, y)
  ref.backward()
  R.check('loss', abs(eng.loss.item() - ref.item()) / (1e-4 * max(1.0, ref.item())))
  R.exact('correct', int(eng.correct.item()) == int(((s > 0).double() == y).sum()))
  g = Zd.grad
  R.check('dZ32', bound_ratio(eng._dZ32[:R_rows, :C], g[:R_rows], 1e-4 * g[:R_rows].abs() + 1e-6))
  R.exact('dPre cast', torch.equal(eng.dPre[L][:R_rows].view(torch.int16),
                                   eng._dZ32[:R_rows].to(torch.bfloat16).view(torch.int16)))
  R.check('db_last', colsum_ratio(bias_grad, eng.dPre[L], R_rows))


def _sage_graph(N, E, seed):
  ei = rmat_edges(N, E // 2, seed=seed)
  ei = torch.cat([ei, ei.flip(0)], 1)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=N)
  return topo, glt.data.Graph(topo, 'CUDA', 0)


SAGE_CASES = {
    # name: engine options (in_dim, hidden, classes, fanouts, ...), check the negative controls
    'eager-wd': dict(dims=(128, 256, 47), fanouts=[5, 4, 3], weight_decay=5e-4),
    'captured-fused-dropout-wd': dict(dims=(128, 256, 47), fanouts=[5, 4, 3], graph=True, dropout=0.5,
                                      weight_decay=5e-4, controls=True),
    'pipelined-captured-unfused': dict(dims=(128, 256, 47), fanouts=[5, 4, 3], graph=True, pipeline=True,
                                       use_fused=False, dropout=0.3),
    'L1': dict(dims=(128, 256, 47), fanouts=[10]),
    'L4-32-1024-8': dict(dims=(32, 1024, 8), fanouts=[4, 3, 3, 2], dropout=0.3),
    'wide-1024-768-300': dict(dims=(1024, 768, 300), fanouts=[5, 4], bs=128),
    'mxfp8': dict(dims=(128, 256, 47), fanouts=[5, 4, 3], mxfp8=True),
    'calibrated-overflow': dict(dims=(128, 128, 47), fanouts=[6, 5, 4], calibrated=True),
}


@pytest.mark.parametrize('name', list(SAGE_CASES))
def test_sage_step_stages_match_fp64(native, name):
  cfg = dict(SAGE_CASES[name])
  (in_dim, hidden, C), bs = cfg.pop('dims'), cfg.pop('bs', 256)
  N = 12000
  topo, graph = _sage_graph(N, 120000, seed=len(name))
  g = torch.Generator().manual_seed(7)
  X = torch.randn(N, in_dim, generator=g).to(DEV)
  labels = torch.randint(0, C, (N,), generator=g).to(DEV)
  if cfg.pop('mxfp8', False):
    q = quantize_mxfp8(X)
    X = dequantize_mxfp8(q, in_dim)
    ut, fmt = _table(q), 'mxfp8'
  else:
    X = X.to(torch.bfloat16)
    ut, fmt = _table(X), 'bf16'
  Xself = X.to(torch.bfloat16)
  captured, controls, calibrated = cfg.pop('graph', False), cfg.pop('controls', False), cfg.pop('calibrated', False)
  eng = GraphSageEngine(graph, ut._table(), labels, in_dim=in_dim, num_nodes=N, batch_size=bs, hidden=hidden,
                        num_classes=C, device=DEV, use_cuda_graph=captured, seed=3, feature_format=fmt,
                        calibration_seeds=torch.arange(N) if calibrated else None, calibration_margin=0.6,
                        check_every=0 if calibrated else 64, **cfg)
  assert eng.calibrated == calibrated
  if captured:
    eng.warmup_and_capture(n_eager=1)
  dpre = lambda: [None] + [eng.dPre[l].clone() for l in range(1, eng.L + 1)]
  batches = _batches(bs, N, g)
  steps = []
  if eng.pipeline:
    eng.train_step(batches[0])                               # samples batch 0 only
    for i in range(1, len(batches) + 1):
      snap = _snapshot(eng, dpre)
      eng.train_step(batches[i]) if i < len(batches) else eng.flush()
      steps.append((snap, 1 - eng._cur if i < len(batches) else eng._cur))
      _run_sage_checks(eng, name, i - 1, steps[-1], X, Xself, labels, controls)
  else:
    for i, seeds in enumerate(batches):
      snap = _snapshot(eng, dpre)
      eng.train_step(seeds)
      _run_sage_checks(eng, name, i, (snap, 0), X, Xself, labels, controls)
  if calibrated:
    assert eng.overflow_count() > 0, 'the calibrated engine must drop neighbours past its capacities'


def _run_sage_checks(eng, name, i, step, X, Xself, labels, controls):
  snap, parity = step
  R = Ratios(f'{name} step {i}')
  _sage_stages(R, eng, snap, parity, X, Xself, labels, controls and i == 1)
  R.show()


LINK_CASES = {
    'link-fused-dropout-captured': dict(use_fused=True, graph=True),
    'link-unfused-dropout-wd': dict(use_fused=False, weight_decay=5e-4),
}


@pytest.mark.parametrize('name', list(LINK_CASES))
def test_link_step_stages_match_fp64(native, name):
  cfg = dict(LINK_CASES[name])
  N, B, Fdim = 8000, 96, 64
  topo, graph = _sage_graph(N, 100000, seed=5)
  X = torch.randn(N, Fdim, generator=torch.Generator().manual_seed(1)).to(DEV).to(torch.bfloat16)
  ut = _table(X)
  captured = cfg.pop('graph', False)
  eng = GraphSageLinkEngine(graph, ut._table(), Fdim, N, fanouts=[5, 4], batch_size=B, hidden=128, out_channels=64,
                            neg_ratio=2, device=DEV, use_cuda_graph=captured, seed=5, dropout=0.5, **cfg)
  if captured:
    eng.warmup_and_capture(n_eager=1)
  dpre = lambda: [None] + [eng.dPre[l].clone() for l in range(1, eng.L + 1)]
  rows = torch.repeat_interleave(torch.arange(N), topo.indptr[1:] - topo.indptr[:-1])
  ei = torch.stack([rows, topo.indices.long().cpu()])
  g = torch.Generator().manual_seed(2)
  for i, n in enumerate((B, 7, 1, B)):
    pairs = ei[:, torch.randperm(ei.shape[1], generator=g)[:n]].to(DEV)
    snap = _snapshot(eng, dpre)
    eng.train_step(pairs)
    R = Ratios(f'{name} (fused layers {eng.fused_ok[1:]}) step {i} ({n} pairs)')
    _sage_stages(R, eng, snap, 0, X, X, None, False)
    R.show()


# --------------------------------------------------------------------------- HeteroSageEngine
def _hetero_stages(R, eng, snap, feats, controls):
  """Every (layer, destination type) stage of the R-SAGE step just taken.  feats: {type index: bf16 table}."""
  torch.cuda.synchronize()
  ar, L, H = eng.arena, eng.L, eng.hidden
  NT = len(eng.ntypes)
  cnt = ar.counters.tolist()
  ctr = [cnt[t * 8:t * 8 + 8] for t in range(NT)]
  p16 = lambda name: snap['p16'][eng.param_index[name][0]:][:math.prod(eng.param_index[name][1])].view(
      *eng.param_index[name][1])
  grad = lambda name: eng.param(name, grad=True)
  # the arena's COO of hops < L, to cross-check the edges read from the ELL blocks
  coo_nodes, coo_rows, coo_cols, _, nn, ne = ar.to_coo()

  def rel_edges(r, nh):
    t = eng.kt[r]
    return _ell_edges(lambda h: ar.ell_of(r, h), ar.deg_of(r), ctr[t], nh, eng.cap_rows[t], eng.fan[r][:nh])

  for r in range(len(eng.edge_types)):
    tgt, src = rel_edges(r, L)
    E = sum(ne[r][:L])
    key = lambda a, b: torch.sort(a.long() * (1 << 32) + b.long()).values
    R.exact('ell = coo', torch.equal(key(tgt, src), key(coo_cols[r][:E], coo_rows[r][:E])))

  def T_of(l, t):
    return min(ctr[t][L - l + 1], eng.A[l][t].shape[0])

  for l in range(1, L + 1):
    nh = L - l + 1
    for t in eng.targets[l]:
      A, T = eng.A[l][t], T_of(l, t)
      offs, self_col = eng.col[l][t]
      deg_blocks = {}
      for j, r in enumerate(eng.in_rel[l][t]):
        s = eng.nt[r]
        tgt, src = rel_edges(r, nh)
        keep = tgt < T
        tgt, src = tgt[keep], src[keep]
        d = eng._width_in(l, s)
        if l == 1:
          ref, bound = mean_ref(feats[s], tgt, ar.nodes_of(s)[src], ar.deg_of(r)[:T])
        else:
          assert src.numel() == 0 or int(src.max()) < eng.Z[l - 1][s].shape[0], f'layer {l}: a source row past Z'
          ref, bound = mean_ref(eng.Z[l - 1][s], tgt, src, ar.deg_of(r)[:T])
        R.check(f'agg{l}', bound_ratio(A[:T, offs[j]:offs[j] + d], ref, bound))
        deg_blocks[j] = (ref, bound, d)
      if controls:
        # two same-width relation blocks swapped
        same = [(a, b) for a in deg_blocks for b in deg_blocks if a < b and deg_blocks[a][2] == deg_blocks[b][2]]
        if same:
          a, b = same[0]
          ref, bound, d = deg_blocks[a]
          assert bound_ratio(A[:T, offs[b]:offs[b] + d], ref, bound) > 1.0, 'swapped relation blocks must be rejected'
      d_t = eng._width_in(l, t)
      Xt = feats[t][ar.nodes_of(t)[:T]] if l == 1 else eng.Z[l - 1][t][:T]
      R.exact(f'self{l}', torch.equal(A[:T, self_col:self_col + d_t], Xt))
      _check_linear(R, f'Z{l}', A, p16(('W', l, t)), p16(('b', l, t)), eng.Z[l][t], T, l < L)
  st = eng.tid[eng.seed_type]
  _check_softmax(R, eng.Z[L][st], eng.C, eng.labels, ar.nodes_of(st), T_of(L, st), eng.dPre[L][st],
                 grad(('b', L, st)), eng.loss, eng.correct)
  for l in range(L, 0, -1):
    nh = L - l + 1
    for t in eng.targets[l]:
      T = T_of(l, t)
      _check_grads(R, l, grad(('W', l, t)), eng.dPre[l][t], eng.A[l][t], p16(('W', l, t)),
                   eng.dA[l][t] if l > 1 else None, T)
      R.exact(f'dPre{l} tail', bool((eng.dPre[l][t][T:] == 0).all()))
    if l == 1:
      break
    # dH[l-1][s]: the scatter of every relation out of s (its dA mean block over the target's degree), plus the
    # self block of s's own rows
    for s in eng.targets[l - 1]:
      dH = eng.dH[l - 1][s]
      S = min(ctr[s][nh + 1], dH.shape[0])
      ref = torch.zeros(S, H, dtype=torch.float64, device=DEV)
      ab, n = torch.zeros_like(ref), torch.zeros(S, dtype=torch.float64, device=DEV)
      parts = []
      for t in eng.targets[l]:
        offs, self_col = eng.col[l][t]
        T, dA = T_of(l, t), eng.dA[l][t].double()
        for j, r in enumerate(eng.in_rel[l][t]):
          if eng.nt[r] != s:
            continue
          tgt, src = rel_edges(r, nh)
          keep = (tgt < T) & (src < S)
          tgt, src = tgt[keep], src[keep]
          terms = dA[tgt, offs[j]:offs[j] + H] / ar.deg_of(r).double()[tgt].unsqueeze(1)
          part = torch.zeros_like(ref).index_add_(0, src, terms)
          parts.append(part)
          ref += part
          ab.index_add_(0, src, terms.abs())
          n += torch.bincount(src, minlength=S).double()
        if t == s:
          m = min(T, S)
          ref[:m] += dA[:m, self_col:self_col + H]
          ab[:m] += dA[:m, self_col:self_col + H].abs()
          n[:m] += 1
      bound = sum_bound(n.unsqueeze(1), ab)
      R.check(f'dH{l - 1}', bound_ratio(dH[:S], ref, bound))
      if controls and parts and bool(parts[0].any()):
        # one relation's scatter credited to another source type: missing from this one
        assert bound_ratio(dH[:S].double() - parts[0], ref, bound) > 1.0, 'a misdirected scatter must be rejected'
      dP, Z = eng.dPre[l - 1][s], eng.Z[l - 1][s]
      exp = torch.where(Z[:S] > 0, dH[:S], torch.zeros_like(dH[:S])).to(torch.bfloat16)
      R.exact(f'dPre{l - 1}', torch.equal(dP[:S].view(torch.int16), exp.view(torch.int16)))
      R.check(f'db{l - 1}', colsum_ratio(grad(('b', l - 1, s)), dP, S))
  _check_adam(R, eng, snap, eng.wd, controls and eng.wd > 0)


def _rand_edges(n_src, n_dst, E, g, hubs=True):
  """E random (src, dst) edges; a few hub destinations and sources."""
  src = torch.randint(0, n_src, (E,), generator=g)
  dst = torch.randint(0, n_dst, (E,), generator=g)
  if hubs:
    dst[:E // 20] = 3 % n_dst
    src[E // 20:E // 10] = 5 % n_src
  return torch.stack([src, dst])


def _schema(name, g):
  """(edges {etype: [2, E]}, sizes, widths, seed type, engine options) of each schema."""
  if name == 'igbh':
    sizes = {'paper': 3000, 'author': 2000, 'institute': 60, 'fos': 40}
    e = {('paper', 'cites', 'paper'): _rand_edges(3000, 3000, 15000, g),
         ('paper', 'written_by', 'author'): _rand_edges(3000, 2000, 8000, g),
         ('author', 'affiliated_to', 'institute'): _rand_edges(2000, 60, 3000, g),
         ('paper', 'topic', 'fos'): _rand_edges(3000, 40, 6000, g)}
    for (a, rel, b) in list(e):
      if a != b:
        e[(b, 'rev_' + rel, a)] = e[(a, rel, b)].flip(0)
    return e, sizes, {'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128}, 'paper', \
        dict(fanouts=[4, 3, 2], hidden=192, num_classes=19, weight_decay=5e-4)
  if name in ('user-item-out', 'user-item-out-L4'):
    sizes = {'user': 2500, 'item': 1500}
    e = {('user', 'buys', 'item'): _rand_edges(2500, 1500, 12000, g),
         ('item', 'also', 'item'): _rand_edges(1500, 1500, 6000, g)}
    e[('item', 'rev_buys', 'user')] = e[('user', 'buys', 'item')].flip(0)
    fan = [4, 3] if name == 'user-item-out' else [3, 3, 2, 2]
    return e, sizes, {'user': 64, 'item': 128}, 'user', dict(fanouts=fan, hidden=128, num_classes=10, edge_dir='out')
  if name == 'fanout-dict-zero':
    sizes = {'a': 2000, 'b': 1500, 'c': 800}
    e = {('b', 'ba', 'a'): _rand_edges(1500, 2000, 9000, g), ('a', 'ab', 'b'): _rand_edges(2000, 1500, 9000, g),
         ('c', 'ca', 'a'): _rand_edges(800, 2000, 5000, g), ('a', 'ac', 'c'): _rand_edges(2000, 800, 5000, g)}
    fan = {et: [3, 3, 2] for et in e}
    fan[('c', 'ca', 'a')] = [4, 0, 0]                        # c feeds a at hop 0 only
    return e, sizes, {'a': 64, 'b': 64, 'c': 128}, 'a', dict(fanouts=fan, hidden=64, num_classes=12,
                                                               weight_decay=5e-4)
  if name == 'self-only-type':
    sizes = {'a': 2000, 'b': 1200, 'c': 900}
    e = {('b', 'ba', 'a'): _rand_edges(1200, 2000, 8000, g), ('c', 'ca', 'a'): _rand_edges(900, 2000, 6000, g)}
    return e, sizes, {'a': 64, 'b': 64, 'c': 128}, 'a', dict(fanouts=[4, 3], hidden=64, num_classes=7)
  if name in ('parallel-relations', 'parallel-relations-L1'):
    sizes = {'u': 1800, 'v': 2200}
    e = {('u', 'r1', 'v'): _rand_edges(1800, 2200, 9000, g), ('u', 'r2', 'v'): _rand_edges(1800, 2200, 4000, g),
         ('v', 'back', 'u'): _rand_edges(2200, 1800, 7000, g)}
    fan = [4, 3, 2] if name == 'parallel-relations' else [5]
    return e, sizes, {'u': 64, 'v': 64}, 'v', dict(fanouts=fan, hidden=64, num_classes=9)
  raise KeyError(name)


HETERO_CASES = ['igbh', 'user-item-out', 'fanout-dict-zero', 'self-only-type', 'parallel-relations',
                'parallel-relations-L1', 'user-item-out-L4']


@pytest.mark.parametrize('name', HETERO_CASES)
def test_hetero_step_stages_match_fp64(native, name):
  g = torch.Generator().manual_seed(len(name))
  edges, sizes, widths, seed_type, opts = _schema(name, g)
  edge_dir = opts.get('edge_dir', 'in')
  graphs, tables, feats, keep = {}, {}, {}, []
  for et, ei in edges.items():
    if edge_dir == 'in':
      topo = glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=sizes[et[2]])
    else:
      topo = glt.data.Topology(ei.to(DEV), layout='CSR', num_nodes=sizes[et[0]])
    graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
  for t, n in sizes.items():
    x = torch.randn(n, widths[t], generator=g).to(DEV).to(torch.bfloat16)
    ut = _table(x)
    keep.append(ut)
    tables[t], feats[t] = ut._table(), x
  labels = torch.randint(0, opts['num_classes'], (sizes[seed_type],), generator=g).to(DEV)
  bs = 192
  eng = HeteroSageEngine(graphs, tables, labels, widths, sizes, seed_type, batch_size=bs, lr=5e-3, seed=1,
                         device=DEV, use_cuda_graph=(name == 'igbh'), **opts)
  if name == 'self-only-type':
    assert any(not eng.in_rel[1][t] for t in eng.targets[1]), 'the schema must hold a self-only destination type'
  if name == 'fanout-dict-zero':
    assert any(0 in f for f in eng.fan)
  if name == 'igbh':
    eng.warmup_and_capture(n_eager=1)
    assert eng._graph is not None
  fidx = {eng.tid[t]: feats[t] for t in feats}
  dpre = lambda: None
  controls = name in ('parallel-relations', 'igbh')
  for i, seeds in enumerate(_batches(bs, sizes[seed_type], g)):
    snap = _snapshot(eng, dpre)
    eng.train_step(seeds)
    R = Ratios(f'{name} step {i}')
    _hetero_stages(R, eng, snap, fidx, controls and i == 1)
    R.show()
