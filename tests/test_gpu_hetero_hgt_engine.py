"""HeteroHgtEngine (device-resident HGT step) and its attention kernels (csrc/cuda/hgt.cu).

Kernels: `hgt_attention` and `hgt_attention_bwd` on hand-built ELL batches with 1, 2 and 4 relations into one type,
each with its own fan-outs (rows of degree 0, 1 and k with a k = 512 hub, -1 slots, three hops, rows with neighbours in
one relation only and rows with none), at heads 1 to 128 and head widths D from 8 to 256, with equal scores and scores
near 100 (where an unshifted exp overflows), against float64 autograd with explicit error bounds; and once with 8
relations x 128 heads, the most per-(relation, head) prior partials the backward reduces in shared memory.

Engine: one step against an fp32 PyTorch recomputation of the HGT model from the arena's COO on the SAME sampled batch,
rounding to bf16 where the engine stores bf16; the same logits as `models.HGTConv` loaded with the engine's weights;
graph replay, training progress, state_dict round trip, evaluation and constructor rejections.
"""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from helpers import (add_isolated_papers, bf16_ulp, bound_ratio, hgt_alpha_rel, hgt_bwd_tol, hgt_score_err,
                     weighted_sum_bound)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
EPS32 = 2.0 ** -23
ROWS = [3, 50, 400]                                     # target rows per hop
FANS = [(512, 7, 3), (64, 5, 2), (16, 9, 4), (2, 3, 6),  # per relation: k per hop (relation 0 has the hub)
        (32, 4, 2), (8, 6, 3), (128, 2, 5), (3, 8, 1)]
N_SRC = [600, 300, 450, 100, 250, 500, 350, 150]


# --------------------------------------------------------------------------- kernels against float64
def _structure(R, seed):
  """Per relation r, per-hop ELL blocks over its sources [0, N_SRC[r]).  Row 0 of every hop has no neighbour in any
  relation; row 1 has degree 1 and row 2 degree k; row 3 of hops 1 and 2 has neighbours in relation 0 only.  About 10%
  of the slots below a row's degree are -1; slots past the degree hold valid ids that must not be read."""
  g = torch.Generator().manual_seed(seed)
  cum = [0]
  for n in ROWS:
    cum.append(cum[-1] + n)
  degs, ells = [], []
  for r in range(R):
    dr, er = [], []
    for h, rows in enumerate(ROWS):
      k = FANS[r][h]
      deg = torch.randint(0, k + 1, (rows,), generator=g)
      deg[:3] = torch.tensor([0, 1, k])
      if r > 0 and h > 0:
        deg[3] = 0
      elif h > 0:
        deg[3] = max(1, k // 2)
      e = torch.randint(0, N_SRC[r], (rows, k), generator=g)
      e[torch.rand(rows, k, generator=g) < 0.1] = -1
      e[2, :] = torch.randint(0, N_SRC[r], (k,), generator=g)
      er.append(e.to(torch.int32))
      dr.append(deg.to(torch.int32))
    degs.append(torch.cat(dr))
    ells.append(er)
  return cum, degs, ells


def _edges(cum, deg, ells, r):
  tg, sr, slot = [], [], []
  for h, rows in enumerate(ROWS):
    k = FANS[r][h]
    e = ells[h].long()
    m = (torch.arange(k).unsqueeze(0) < deg[cum[h]:cum[h + 1]].long().unsqueeze(1)) & (e >= 0)
    tg.append((torch.arange(rows).unsqueeze(1) + cum[h]).expand(rows, k)[m])
    sr.append(e[m])
    slot.append(m)
  return torch.cat(tg).to(DEV), torch.cat(sr).to(DEV), slot


def _counters(vals):
  c = torch.zeros(16, dtype=torch.int32)
  c[:len(vals)] = torch.tensor(vals, dtype=torch.int32)
  return c.to(DEV)


# (heads, D): H = heads * D from 64 to 1024, D in {8, 16, 24, 32, 48, 64, 128, 256}.  Up to 8 heads a lane owns at
# most one head's softmax statistics; 64 and 128 heads exceed the 32 lanes of a row, so each lane owns 2 or 4 heads.
SHAPES = [(1, 64), (1, 256), (2, 32), (4, 48), (8, 24), (8, 8), (4, 256), (8, 128),
          (16, 8), (32, 16), (64, 8), (128, 8)]


@pytest.mark.parametrize('scores', ['normal', 'equal', 'large'])
@pytest.mark.parametrize('R', [1, 2, 4])
@pytest.mark.parametrize('heads,D', SHAPES)
def test_hgt_attention_kernels_match_fp64(native, heads, D, R, scores):
  _attention_case(native, heads, D, R, scores)


@pytest.mark.parametrize('scores', ['normal', 'large'])
def test_hgt_attention_kernels_8_relations_128_heads(native, scores):
  """8 relations x 128 heads of width 8: the backward's shared prior partials s_prior[kHgtMaxRel * 128] are full."""
  _attention_case(native, 128, 8, 8, scores)


def _attention_case(native, heads, D, R, scores):
  H = heads * D
  cum, degs, ells = _structure(R, seed=H + heads + R)
  T = cum[-1]
  g = torch.Generator().manual_seed(H * 7 + heads + R)
  qq = torch.randn(T + 5, R * H, generator=g)
  if scores == 'equal':
    qq.zero_()
  qq = qq.to(torch.bfloat16).to(DEV)
  kv = [torch.randn(N_SRC[r], 3 * H, generator=g).to(torch.bfloat16).to(DEV) for r in range(R)]
  if scores == 'large':      # |score| up to ~100: exp of an unshifted score overflows fp32 above 88.7
    prior = [(33.0 + torch.rand(heads, generator=g)).to(DEV) for _ in range(R)]
  else:
    prior = [(1.0 + 0.3 * torch.randn(heads, generator=g)).to(DEV) for _ in range(R)]
  ctr = _counters(cum)
  ell_d = [[e.flatten().to(DEV) for e in ells[r]] for r in range(R)]
  ks = [list(FANS[r][:3]) for r in range(R)]
  deg_d = [d.to(DEV) for d in degs]
  alpha = [[torch.full((rows * FANS[r][h] * heads,), 5.0, device=DEV) for h, rows in enumerate(ROWS)]
           for r in range(R)]
  U = torch.full((T + 5, R * H), 9.0, dtype=torch.bfloat16, device=DEV)
  native.hgt_attention(qq, U, heads, ctr, 3, kv, prior, ell_d, ks, deg_d, alpha)
  torch.cuda.synchronize()

  # ---- float64 reference from the bf16 inputs
  qd = qq[:T].double().requires_grad_(True)
  kvd = [x.double().requires_grad_(True) for x in kv]
  pd = [p.double().requires_grad_(True) for p in prior]
  scale = 1.0 / math.sqrt(D)
  E = [_edges(cum, degs[r], ells[r], r) for r in range(R)]
  sc, cabs, tgs = [], [], []
  for r in range(R):
    tg, sr, _ = E[r]
    q = qd[:, r * H:(r + 1) * H].reshape(T, heads, D)[tg]
    k = kvd[r][:, :H].reshape(-1, heads, D)[sr]
    sc.append((q * k).sum(-1) * pd[r] * scale)
    cabs.append((q.detach().abs() * k.detach().abs()).sum(-1) * scale)
    tgs.append(tg)
  s_all, tg_all = torch.cat(sc), torch.cat(tgs)
  m = torch.full((T, heads), -float('inf'), dtype=torch.float64, device=DEV).scatter_reduce(
      0, tg_all.unsqueeze(1).expand(-1, heads), s_all.detach(), 'amax', include_self=True)
  ex = torch.exp(s_all - m[tg_all])
  den = torch.zeros(T, heads, dtype=torch.float64, device=DEV).index_add(0, tg_all, ex)
  al = ex / den[tg_all]
  als = list(torch.split(al, [len(t) for t in tgs]))
  outs = []
  for r in range(R):
    tg, sr, _ = E[r]
    v = kvd[r][:, 2 * H:].reshape(-1, heads, D)[sr]
    outs.append(torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add(0, tg, (als[r].unsqueeze(-1) * v)
                                                                             .reshape(-1, H)))
  out = torch.cat(outs, 1)

  # alpha: every relation's slots, in the kernel's layout; the softmax spans all relations
  ga = []
  for r in range(R):
    slot = E[r][2]
    ga.append(torch.cat([alpha[r][h].view(rows, FANS[r][h], heads)[slot[h].to(DEV)] for h, rows in enumerate(ROWS)]))
  ga = torch.cat(ga)
  # score error: an fp32 dot of D terms times prior / sqrt(D), relative to the sum of |terms|
  pr_abs = torch.cat([pd[r].detach().abs().expand(len(tgs[r]), heads) for r in range(R)])
  serr = hgt_score_err(torch.cat(cabs), pr_abs, s_all.detach(), D)
  arel = hgt_alpha_rel(s_all.detach(), serr, tg_all, T)
  assert bound_ratio(ga, al.detach(), arel * al.detach() + 1e-30) <= 1.0
  # the softmax spans every relation: alpha sums to one per (row, head) over all of them (zero for isolated rows)
  tot = torch.zeros(T, heads, dtype=torch.float64, device=DEV).index_add(0, tg_all, ga.double())
  covered = torch.zeros(T, dtype=torch.bool, device=DEV)
  covered[tg_all] = True
  assert bool((tot[covered] - 1).abs().max() < 1e-5), 'alpha over all relations sums to one'
  assert bool((tot[~covered] == 0).all())
  assert int((~covered).sum()) >= 3
  if R > 1:
    only0 = covered.clone()
    for r in range(1, R):
      only0[E[r][0]] = False
    assert int(only0.sum()) > 0, 'rows with neighbours in one relation only'
  # output: one bf16 rounding of an fp32 sum of weighted terms
  ab = torch.cat([torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add(
      0, E[r][0], (als[r].detach().unsqueeze(-1) * kvd[r].detach()[:, 2 * H:].abs().reshape(-1, heads, D)[E[r][1]])
      .reshape(-1, H)) for r in range(R)], 1)
  kd = torch.stack([d.to(DEV) for d in degs]).sum(0).double().unsqueeze(1)
  arel_row = torch.zeros(T, heads, dtype=torch.float64, device=DEV).scatter_reduce(
      0, tg_all.unsqueeze(1).expand(-1, heads), arel, 'amax', include_self=True)
  arel_col = arel_row.repeat_interleave(D, 1).repeat(1, R)
  # (+ 2^-120 kd max|v|: alphas below fp32's normal range lose their precision, the float64 reference keeps it)
  vmax = max(float(x[:, 2 * H:].abs().max()) for x in kv)
  bound = weighted_sum_bound(out.detach(), ab, kd, arel=arel_col, floor=2.0 ** -120 * kd * vmax)
  assert bound_ratio(U[:T], out.detach(), bound) <= 1.0
  assert bool((U[:T][~covered] == 0).all()), 'a row without any neighbour aggregates nothing'

  # ---- backward
  dU = torch.randn(T, R * H, generator=g).to(torch.bfloat16).to(DEV)
  (out * dU.double()).sum().backward()
  dal = [[torch.full((2 * a.numel(),), 11.0, device=DEV) for a in alpha[r]] for r in range(R)]
  dkv = [torch.zeros(N_SRC[r], 2 * H, device=DEV) for r in range(R)]
  dprior = [torch.zeros(heads, device=DEV) for _ in range(R)]
  dqq = torch.full((T + 200, R * H), 9.0, dtype=torch.bfloat16, device=DEV)
  qq_pad = torch.cat([qq, torch.zeros(195, R * H, dtype=torch.bfloat16, device=DEV)])
  dU_pad = torch.cat([dU, torch.zeros(200, R * H, dtype=torch.bfloat16, device=DEV)])
  native.hgt_attention_bwd(dU_pad, qq_pad, dqq, heads, ctr, 3, kv, prior, ell_d, ks, deg_d, alpha, dal, dkv, dprior)
  torch.cuda.synchronize()
  Gd = dU.double()
  # |terms| of the score gradient: alpha (|dalpha| + sum alpha |dalpha|), each dalpha an fp32 dot of D terms
  dabs = []
  for r in range(R):
    tg, sr, _ = E[r]
    dabs.append((Gd[:, r * H:(r + 1) * H].abs().reshape(T, heads, D)[tg] *
                 kvd[r].detach()[:, 2 * H:].abs().reshape(-1, heads, D)[sr]).sum(-1))
  dabs = torch.cat(dabs)
  sabs = torch.zeros(T, heads, dtype=torch.float64, device=DEV).index_add(0, tg_all, al.detach() * dabs)
  term = al.detach() * (dabs + sabs[tg_all])
  tol = hgt_bwd_tol(D, kd.max().item() + 600, float(arel.max()))
  terms = list(torch.split(term, [len(t) for t in tgs]))
  for r in range(R):
    tg, sr, _ = E[r]
    pr = float(pd[r].detach().abs().max()) * scale
    tr = terms[r]
    # dqq: sum_j g k_j, bf16
    kab = kvd[r].detach()[:, :H].abs().reshape(-1, heads, D)[sr]
    b_q = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add(
        0, tg, (tr.unsqueeze(-1) * pr * kab).reshape(-1, H))
    ref_q = qd.grad[:, r * H:(r + 1) * H]
    assert bound_ratio(dqq[:T, r * H:(r + 1) * H], ref_q, bf16_ulp(ref_q) + tol * b_q + 1e-30) <= 1.0
    # dK: sum_i g qq_i (fp32 atomics), dV: sum_i alpha dU_i
    qab = qd.detach()[:, r * H:(r + 1) * H].abs().reshape(T, heads, D)[tg]
    b_k = torch.zeros(N_SRC[r], H, dtype=torch.float64, device=DEV).index_add(
        0, sr, (tr.unsqueeze(-1) * pr * qab).reshape(-1, H))
    assert bound_ratio(dkv[r][:, :H], kvd[r].grad[:, :H], tol * b_k + 1e-30) <= 1.0
    b_v = torch.zeros(N_SRC[r], H, dtype=torch.float64, device=DEV).index_add(
        0, sr, (als[r].detach().unsqueeze(-1) * Gd[:, r * H:(r + 1) * H].abs().reshape(T, heads, D)[tg]).reshape(-1, H))
    assert bound_ratio(dkv[r][:, H:], kvd[r].grad[:, 2 * H:], tol * b_v + 1e-30) <= 1.0
    # prior: sum over every slot of ds * c / sqrt(D)
    b_p = (tr * cabs[r]).sum(0)
    assert bound_ratio(dprior[r], pd[r].grad, (tol + len(tg) * EPS32) * b_p + 1e-30) <= 1.0
  assert bool((dqq[T:T + 128 - T % 128] == 0).all()), 'rows past the targets up to the next 128-row tile are zero'


def test_hgt_attention_rejects_too_many_relations(native):
  H, heads, R = 64, 2, 9
  qq = torch.zeros(128, R * H, dtype=torch.bfloat16, device=DEV)
  kv = [torch.zeros(128, 3 * H, dtype=torch.bfloat16, device=DEV)] * R
  prior = [torch.ones(heads, device=DEV)] * R
  ell = [[torch.zeros(4, dtype=torch.int32, device=DEV)]] * R
  deg = [torch.zeros(128, dtype=torch.int32, device=DEV)] * R
  alpha = [[torch.zeros(4 * heads, device=DEV)]] * R
  with pytest.raises(RuntimeError, match='1 to 8 relations'):
    native.hgt_attention(qq, torch.zeros_like(qq), heads, _counters([0, 1]), 1, kv, prior, ell, [[4]] * R, deg, alpha)


# --------------------------------------------------------------------------- engine
ISOLATED = 64


def _build(schema='mag', feat_dim=64, hidden=64, heads=2, classes=20, fan=(4, 3), bs=256, use_graph=False,
           papers=3000, lr=1e-2):
  """Synthetic MAG or IGBH plus ISOLATED extra papers that only send edges (in every relation out of 'paper'): they
  have no in-neighbour in any relation, so as targets they aggregate nothing, while their outputs still feed others."""
  from common import synthetic_igbh, synthetic_mag
  from graphlearn_for_pytorch_b200.models import HeteroHgtEngine
  if schema == 'mag':
    edges, _, labels, sizes = synthetic_mag(papers, papers // 2, 40, 30, feat_dim=8, num_classes=classes, seed=2)
  else:
    edges, _, labels, sizes = synthetic_igbh(papers, papers // 2, 50, 30, feat_dim=8, num_classes=classes, seed=2)
  g = torch.Generator().manual_seed(3)
  add_isolated_papers(edges, sizes, ISOLATED, g, {et: 3 for et in edges if et[0] == 'paper'})
  labels = torch.randint(0, classes, (sizes['paper'],), generator=g)
  dims = feat_dim if isinstance(feat_dim, dict) else {t: feat_dim for t in sizes}
  feats = {t: torch.randn(sizes[t], dims[t], generator=g) for t in sizes}
  graphs, tables, keep, fb = {}, {}, [], {}
  for et, ei in edges.items():
    topo = glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=sizes[et[2]])
    graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
  for nt, x in feats.items():
    fb[nt] = x.to(DEV).to(torch.bfloat16)
    ut = glt.data.UnifiedTensor(0, torch.bfloat16)
    ut.append_shared_tensor(fb[nt])
    tables[nt] = ut._table()
    keep.append(ut)
  eng = HeteroHgtEngine(graphs, tables, labels.to(DEV), feat_dim, sizes, 'paper', fanouts=list(fan), batch_size=bs,
                        hidden=hidden, heads=heads, num_classes=classes, edge_dir='in', lr=lr, seed=1, device=DEV,
                        use_cuda_graph=use_graph)
  eng._keep = keep
  return eng, fb, labels.to(DEV), sizes


def _seeds(eng, sizes, batch_seed=0):
  """Half of the isolated papers plus random papers."""
  n_old = sizes['paper'] - ISOLATED
  rnd = torch.randperm(n_old, generator=torch.Generator().manual_seed(batch_seed))[:eng.bs - ISOLATED // 2]
  return torch.cat([torch.arange(n_old, n_old + ISOLATED // 2), rnd]).to(DEV)


class _BfGrad(torch.autograd.Function):
  """Identity whose backward rounds the gradient to bf16 (where the engine stores a gradient in bf16)."""

  @staticmethod
  def forward(ctx, x):
    return x.view_as(x)

  @staticmethod
  def backward(ctx, g):
    return g.to(torch.bfloat16).float()


def _params(eng):
  """fp32 leaf copies of the parameters as the engine's GEMMs see them: the bf16 shadow, except prior and skip, which
  the kernels read from the fp32 master copy."""
  P = {}
  for k, (o, shape) in eng.param_index.items():
    src = eng.p32 if k[0] in ('prior', 'skip') else eng.p16
    P[k] = src[o:o + math.prod(shape)].view(*shape).float().clone().requires_grad_(True)
  return P


def _reference(eng, fb, labels):
  """fp32 recomputation of the HGT step from the arena's COO, rounding to bf16 where the engine stores bf16 (every
  GEMM output and activation, and the gradients the engine keeps in bf16)."""
  nodes, rows, cols, _, nn, ne = eng.arena.to_coo()
  L, nt, hd, H = eng.L, eng.nt, eng.heads, eng.hidden
  D = H // hd
  bf = lambda x: x.to(torch.bfloat16).float()   # noqa: E731
  P = _params(eng)
  x = {}
  for u in eng.in_types:
    pre = _BfGrad.apply(fb[eng.ntypes[u]][nodes[u]].float() @ P[('in_W', u)].t() + P[('in_b', u)])
    x[u] = bf(F.relu(pre))
  info = {'isolated': 0}
  for l in range(1, L + 1):
    nh = L - l + 1
    kqv = {u: _BfGrad.apply(bf(x[u] @ P[('kqv_W', l, u)].t() + P[('kqv_b', l, u)])) for u in eng.kqv_types[l]}
    out = {}
    for t in eng.targets[l]:
      T = sum(nn[t][:nh])
      q = kqv[t][:T, H:2 * H].reshape(T, hd, D)
      sc, msgs, dsts, srcs = [], [], [], []
      us = []
      covered = torch.zeros(T, dtype=torch.bool, device=DEV)
      for r in eng.in_rel[l][t]:
        E = sum(ne[r][:nh])
        src, dst = rows[r][:E].long(), cols[r][:E].long()
        covered[dst] = True
        qq = _BfGrad.apply(bf(torch.einsum('ihf,hdf->ihd', q, P[('att', l, r)])))
        k = kqv[nt[r]][:, :H].reshape(-1, hd, D)
        sc.append((qq[dst] * k[src]).sum(-1) * P[('prior', l, r)] / math.sqrt(D))
        dsts.append(dst)
        srcs.append(src)
      s = torch.cat(sc)
      dst_all = torch.cat(dsts)
      m = torch.full((T, hd), -float('inf'), device=DEV).scatter_reduce(
          0, dst_all.unsqueeze(1).expand(-1, hd), s.detach(), 'amax', include_self=True)
      ex = torch.exp(s - m[dst_all])
      den = torch.zeros(T, hd, device=DEV).index_add(0, dst_all, ex)
      al = ex / den[dst_all]
      agg = torch.zeros(T, H, device=DEV)
      for r, a, src, dst in zip(eng.in_rel[l][t], torch.split(al, [len(d) for d in dsts]), srcs, dsts):
        v = kqv[nt[r]][:, 2 * H:].reshape(-1, hd, D)
        u_r = torch.zeros(T, hd, D, device=DEV).index_add(0, dst, a.unsqueeze(-1) * v[src])
        u_r = _BfGrad.apply(bf(u_r))
        agg = agg + torch.einsum('ihd,hdf->ihf', u_r, P[('msg', l, r)]).reshape(T, H)
      agg = _BfGrad.apply(bf(agg))
      ge = _BfGrad.apply(bf(F.gelu(agg)))
      A = _BfGrad.apply(bf(ge @ P[('a_W', l, t)].t() + P[('a_b', l, t)]))
      sg = torch.sigmoid(P[('skip', l, t)])
      z = bf(sg * A + (1 - sg) * x[t][:T])
      info['isolated'] += int((~covered).sum())
      out[t] = _BfGrad.apply(z) if l == L else z
    x = out
  st = eng.tid[eng.seed_type]
  n0 = nn[st][0]
  logits = x[st][:n0] @ P[('head_W',)].t() + P[('head_b',)]
  loss = F.cross_entropy(logits[:, :eng.C], labels[nodes[st][:n0]])
  loss.backward()
  return float(loss), {k: v.grad for k, v in P.items()}, info


def _gradient_errors(eng, fb, labels, sizes, batch_seed=0):
  """One engine step on a seeded batch -> {kind: largest max|engine - ref| / max|ref| over the parameters of that
  kind}, and the reference's diagnostics."""
  eng._seeds.copy_(_seeds(eng, sizes, batch_seed))
  eng._sample()
  eng._forward()
  eng._backward()
  torch.cuda.synchronize()
  assert eng.overflow_count() == 0
  ref_loss, grads, info = _reference(eng, fb, labels)
  errs = {'loss': abs(float(eng.loss.item()) - ref_loss) / max(1.0, abs(ref_loss))}
  for k, r in grads.items():
    if r is None:
      continue
    o, shape = eng.param_index[k]
    got = eng.g32[o:o + math.prod(shape)].view(*shape)
    e = float((got - r).abs().max()) / max(float(r.abs().max()), 1e-6)
    errs[k[0]] = max(errs.get(k[0], 0.0), e)
  return errs, info


# prior and skip get a looser bound.  Their gradients are sums over every edge (prior) or every element (skip) of nearly
# cancelling terms: sum_j ds_ij vanishes per target because the softmax weights sum to one, and dZ (A - X) mixes signs.
# So one-ulp differences between the engine's bf16 activations (wgmma accumulation order) and the reference's show up
# amplified.  The largest ratios observed were 0.073 (skip, IGBH widths with three layers) and 0.015 (prior); every
# other kind stays below 0.013.
SUM_TOL = 0.15


def _assert_match(errs):
  assert errs.pop('loss') < 3e-2, errs
  bad = {k: e for k, e in errs.items() if not e < (SUM_TOL if k in ('prior', 'skip') else 6e-2)}
  assert not bad, bad
  assert set(errs) >= {'in_W', 'in_b', 'kqv_W', 'kqv_b', 'att', 'msg', 'prior', 'a_W', 'a_b', 'skip', 'head_W',
                       'head_b'}, errs


IGBH_WIDTHS = {'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128}


@pytest.mark.parametrize('schema,feat_dim,hidden,heads,classes,fan', [
    ('mag', 128, 64, 2, 20, (4, 3)),                  # the reference's model: hidden 64, 2 heads, 2 layers
    ('mag', 64, 64, 1, 20, (4, 3)),                   # one head
    ('mag', 128, 256, 8, 20, (4, 3)),                 # eight heads of 32
    ('igbh', IGBH_WIDTHS, 64, 2, 2983, (4, 3, 2)),    # IGBH per-type widths, three layers, 2983 classes
    ('mag', 128, 512, 8, 20, (4, 3)),                 # K/Q/V gradient rows of 192 vectors: two column chunks
    ('mag', 128, 704, 8, 20, (4, 3)),                 # 264 vectors: three chunks, the last of 8; heads of 88
], ids=['mag-64-h2', 'mag-64-h1', 'mag-256-h8', 'igbh_widths-64-h2-L3-2983', 'mag-512-h8', 'mag-704-h8'])
def test_hetero_hgt_engine_gradients_match_fp32(schema, feat_dim, hidden, heads, classes, fan):
  eng, fb, labels, sizes = _build(schema, feat_dim, hidden, heads, classes, fan)
  errs, info = _gradient_errors(eng, fb, labels, sizes)
  assert info['isolated'] > 0, info
  print('largest relative error per parameter kind:', {k: round(v, 4) for k, v in errs.items()})
  _assert_match(errs)


def test_hetero_hgt_engine_matches_hgtconv():
  """`models.HGTConv` loaded with the engine's weights (plus the input Linears and the head) gives the engine's seed
  logits on a batch where every destination type has edges."""
  from graphlearn_for_pytorch_b200.models import HGTConv
  eng, fb, labels, sizes = _build('mag', 128, 64, 2, 20, (4, 3))
  eng._seeds.copy_(torch.randperm(sizes['paper'] - ISOLATED, generator=torch.Generator().manual_seed(4))[:eng.bs]
                   .to(DEV))
  eng._sample()
  eng._forward()
  torch.cuda.synchronize()
  nodes, rows, cols, _, nn, ne = eng.arena.to_coo()
  L, H, hd = eng.L, eng.hidden, eng.heads
  P = {k: v.detach() for k, v in _params(eng).items()}
  names = list(eng.ntypes)
  x = {names[u]: F.relu(fb[names[u]][nodes[u]].float() @ P[('in_W', u)].t() + P[('in_b', u)]) for u in eng.in_types}
  for l in range(1, L + 1):
    nh = L - l + 1
    conv = HGTConv({t: H for t in names}, H, names, eng.edge_types, heads=hd).to(DEV)
    ei = {}
    for r, et in enumerate(eng.edge_types):
      if any(r in eng.in_rel[l][t] for t in eng.targets[l]):
        E = sum(ne[r][:nh])
        assert E > 0
        ei[et] = torch.stack([rows[r][:E].long(), cols[r][:E].long()])
    with torch.no_grad():
      for u in eng.kqv_types[l]:
        W, b = P[('kqv_W', l, u)], P[('kqv_b', l, u)]
        for i, lin in enumerate((conv.k, conv.q, conv.v)):
          lin[names[u]].weight.copy_(W[i * H:(i + 1) * H]); lin[names[u]].bias.copy_(b[i * H:(i + 1) * H])
      for t in eng.targets[l]:
        conv.a[names[t]].weight.copy_(P[('a_W', l, t)]); conv.a[names[t]].bias.copy_(P[('a_b', l, t)])
        conv.skip[names[t]].copy_(P[('skip', l, t)])
        for r in eng.in_rel[l][t]:
          key = '__'.join(eng.edge_types[r])
          conv.w_att[key].copy_(P[('att', l, r)]); conv.w_msg[key].copy_(P[('msg', l, r)])
          conv.prior[key].copy_(P[('prior', l, r)])
      x = conv(x, ei)
  st = eng.tid[eng.seed_type]
  n0 = nn[st][0]
  ref = x[eng.seed_type][:n0] @ P[('head_W',)].t() + P[('head_b',)]
  got = eng.logits[:n0].float()
  err = float((got[:, :eng.C] - ref[:, :eng.C]).abs().max()) / float(ref[:, :eng.C].abs().max())
  assert err < 3e-2, err


def test_hetero_hgt_engine_graph_replay_and_state_dict():
  eng, fb, labels, sizes = _build(use_graph=True)
  eng.warmup_and_capture(n_eager=1)
  assert eng._graph is not None and eng.kernels_per_step > 0
  seeds = _seeds(eng, sizes, 7)
  # the replayed graph computes the eager step (up to the order of fp32 atomics)
  saved = eng.state_dict()
  graph, eng._graph = eng._graph, None
  l_eager = float(eng.train_step(seeds).item())
  eng.load_state_dict(saved)
  eng._graph = graph
  l_graph = float(eng.train_step(seeds).item())
  assert abs(l_graph - l_eager) <= 1e-3 * max(1.0, abs(l_eager)), (l_graph, l_eager)
  # state_dict round trip: the same steps from the same state give the same losses
  s = eng.state_dict()
  run = lambda: [float(eng.train_step(_seeds(eng, sizes, 100 + i)).item()) for i in range(3)]   # noqa: E731
  first = run()
  eng.load_state_dict(s)
  second = run()
  assert all(abs(a - b) <= 1e-2 * max(1.0, abs(a)) for a, b in zip(first, second)), (first, second)
  eng.close()


def test_hetero_hgt_engine_trains_under_cuda_graph_and_evaluates():
  eng, fb, labels, sizes = _build(use_graph=True, classes=8)
  # learnable labels: a fixed function of the paper features
  w = torch.randn(fb['paper'].shape[1], 8, generator=torch.Generator().manual_seed(9)).to(DEV)
  eng.labels.copy_((fb['paper'].float() @ w).argmax(1))
  eng.warmup_and_capture(n_eager=1)
  g = torch.Generator().manual_seed(0)
  losses = []
  for i in range(60):
    losses.append(float(eng.train_step(torch.randperm(sizes['paper'], generator=g)[:eng.bs].to(DEV)).item()))
  assert all(l == l for l in losses)
  assert sum(losses[-10:]) / 10 < sum(losses[:10]) / 10 - 0.05, (losses[:5], losses[-5:])
  p_before = eng.p32.clone()
  l, c, n = eng.evaluate_batch(torch.arange(eng.bs, device=DEV))
  assert n == eng.bs and 0 <= c <= n and l == l
  assert torch.equal(eng.p32, p_before)
  eng.close()


def test_hetero_hgt_engine_diagonal_blocks_only():
  """Only the per-head diagonal blocks of the relation transforms are parameters: the flat buffer holds heads * D * D
  entries per relation and transform, and an Adam step moves nothing else."""
  eng, fb, labels, sizes = _build(heads=2)
  D = eng.hidden // eng.heads
  for k, (o, shape) in eng.param_index.items():
    if k[0] in ('att', 'msg'):
      assert tuple(shape) == (eng.heads, D, D)
  eng.train_step(_seeds(eng, sizes, 1))
  torch.cuda.synchronize()
  used = torch.zeros(eng.p32.numel(), dtype=torch.bool, device=DEV)
  for k, (o, shape) in eng.param_index.items():
    used[o:o + math.prod(shape)] = True
  assert bool((eng.m[~used] == 0).all()) and bool((eng.p32[~used] == 0).all())


@pytest.mark.parametrize('kw', [
    dict(feat_dim=96),                                                       # in_dim not a multiple of 64
    dict(feat_dim={'paper': 64, 'author': 64, 'institution': 64, 'field_of_study': 40}),
    dict(hidden=96),
    dict(hidden=2048),
    dict(hidden=192, heads=5),                                               # heads does not divide hidden
    dict(heads=16),                                                          # D = 4
])
def test_hetero_hgt_engine_rejects_unsupported_widths(kw):
  with pytest.raises(ValueError, match='in_dim|hidden|heads'):
    _build(papers=1000, **kw)


def test_hetero_hgt_engine_rejects_schemas_the_kernels_cannot_run():
  from graphlearn_for_pytorch_b200.models import HeteroHgtEngine
  sizes = {'paper': 500, 'a': 100}
  g = torch.Generator().manual_seed(0)

  def graph(n_src, n_dst):
    ei = torch.stack([torch.randint(0, n_src, (2000,), generator=g), torch.randint(0, n_dst, (2000,), generator=g)])
    return glt.data.Graph(glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=n_dst), 'CUDA', 0)
  keep, tables = [], {}
  for t, n in sizes.items():
    ut = glt.data.UnifiedTensor(0, torch.bfloat16)
    ut.append_shared_tensor(torch.zeros(n, 64, dtype=torch.bfloat16, device=DEV))
    keep.append(ut)
    tables[t] = ut._table()
  labels = torch.zeros(500, dtype=torch.int64, device=DEV)
  # nine relations into 'paper'
  graphs = {('paper', f'r{i}', 'paper'): graph(500, 500) for i in range(9)}
  with pytest.raises(ValueError, match='at most 8'):
    HeteroHgtEngine(graphs, tables, labels, 64, sizes, 'paper', fanouts=[2, 2], batch_size=64, device=DEV)
  # 'a' is a message source at layer 1 but receives nothing, so it cannot be a layer-1 target of its own hop
  graphs = {('a', 'to', 'paper'): graph(100, 500)}
  with pytest.raises(ValueError, match='no incoming relation'):
    HeteroHgtEngine(graphs, tables, labels, 64, sizes, 'paper', fanouts=[2, 2], batch_size=64, device=DEV)
