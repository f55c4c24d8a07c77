"""HeteroGatEngine (device-resident R-GAT step) and its attention kernels (csrc/cuda/gat.cu).

Kernels: `gat_scores`, `gat_aggregate`, `gat_backward` and `gat_score_bwd` on hand-built ELL batches (rows of degree 0,
1 and k with a k = 512 hub, -1 slots, three hops) at heads 1 to 8 and head widths C from 8 to 256, with equal scores
and scores near 100 (where an unshifted exp overflows), against float64 autograd with explicit error bounds.

Engine: one step against an fp32 PyTorch recomputation of the reference's IGBH R-GAT (examples/igbh/rgnn.py) from the
arena's COO on the SAME sampled batch, rounding to bf16 where the engine stores bf16, with dropout through the engine's
own mask; graph replay, training progress, state_dict round trip, evaluation without dropout and width rejections.
"""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from helpers import (GAT_ISOLATED_EDGES, add_isolated_papers, bf16_ulp, bound_ratio, colsum_bound, gat_alpha_bound,
                     gat_dscore_tol, gat_score_bound, score_bwd_bound, softmax_seg, weighted_sum_bound)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
EPS32 = 2.0 ** -23
HOPS = [(3, 512), (50, 7), (400, 3)]          # (rows, k): a hub hop, then two ordinary hops
N_SRC = 600


# --------------------------------------------------------------------------- kernels against float64
def _structure(seed):
  """Per-hop ELL blocks over sources [0, N_SRC): the first rows of every hop have degree 0, 1 and k; about 10% of the
  slots below a row's degree are -1; slots past the degree hold valid ids that must not be read."""
  g = torch.Generator().manual_seed(seed)
  cum, degs, ells = [0], [], []
  for rows, k in HOPS:
    deg = torch.randint(0, k + 1, (rows,), generator=g)
    deg[:3] = torch.tensor([0, 1, k])
    e = torch.randint(0, N_SRC, (rows, k), generator=g)
    e[torch.rand(rows, k, generator=g) < 0.1] = -1
    e[2, :] = torch.randint(0, N_SRC, (k,), generator=g)   # one full row without holes
    ells.append(e.to(torch.int32))
    degs.append(deg.to(torch.int32))
    cum.append(cum[-1] + rows)
  return cum, torch.cat(degs), ells


def _edges(cum, deg, ells):
  tg, sr = [], []
  for h, (rows, k) in enumerate(HOPS):
    e = ells[h].long()
    m = (torch.arange(k).unsqueeze(0) < deg[cum[h]:cum[h + 1]].long().unsqueeze(1)) & (e >= 0)
    tg.append((torch.arange(rows).unsqueeze(1) + cum[h]).expand(rows, k)[m])
    sr.append(e[m])
  return torch.cat(tg).to(DEV), torch.cat(sr).to(DEV)


def _counters(vals):
  c = torch.zeros(16, dtype=torch.int32)
  c[:len(vals)] = torch.tensor(vals, dtype=torch.int32)
  return c.to(DEV)


# (heads, C): H = heads * C from 64 to 1024, C in {8, 16, 24, 48, 128, 256}.  Up to 8 heads a lane owns at most one
# head's softmax statistics; 64 and 128 heads exceed the 32 lanes of a row, so each lane owns 2 or 4 heads.
SHAPES = [(1, 128), (1, 256), (2, 128), (4, 48), (8, 24), (8, 8), (4, 256), (8, 128),
          (16, 8), (32, 16), (64, 8), (128, 8)]


@pytest.mark.parametrize('scores', ['normal', 'equal', 'large'])
@pytest.mark.parametrize('heads,C', SHAPES)
def test_gat_kernels_match_fp64(native, heads, C, scores):
  H = heads * C
  cum, deg, ells = _structure(seed=H + heads)
  T = cum[-1]
  tg, sr = _edges(cum, deg, ells)
  g = torch.Generator().manual_seed(H * 7 + heads)
  Ps = torch.randn(N_SRC, H, generator=g).to(torch.bfloat16).to(DEV)
  Pd = torch.randn(T + 5, H, generator=g).to(torch.bfloat16).to(DEV)
  att_s, att_d = torch.randn(H, generator=g), torch.randn(H, generator=g)
  if scores == 'equal':
    att_s.zero_(); att_d.zero_()
  elif scores == 'large':      # |score| up to ~100: exp of an unshifted score overflows fp32 above 88.7
    att_s *= 100.0 / (C ** 0.5 * 3); att_d *= 100.0 / (C ** 0.5 * 3)
  att_s, att_d = att_s.to(torch.bfloat16).to(DEV), att_d.to(torch.bfloat16).to(DEV)
  ctr_s, ctr_t = _counters([N_SRC]), _counters(cum)
  as_ = torch.full((N_SRC, heads), 7.0, device=DEV)
  ad = torch.full((T + 5, heads), 7.0, device=DEV)
  zero = torch.full((N_SRC, heads), 3.0, device=DEV)
  # sources: rows < ctr_s[0]; targets: rows < ctr_t[3]
  native.gat_scores(Ps, att_s, as_, ctr_s, 0, Pd, att_d, ad, ctr_t, 3, zero=zero, heads=heads)
  ell = [e.flatten().to(DEV) for e in ells]
  ks = [k for _, k in HOPS]
  deg_d = deg.to(DEV)
  alpha = [torch.full((rows * k * heads,), 5.0, device=DEV) for rows, k in HOPS]
  Z = torch.full((T + 5, H), 9.0, dtype=torch.bfloat16, device=DEV)
  native.gat_aggregate(Ps, as_, ad, heads, ctr_t, 3, ell, ks, deg_d, alpha, Z=Z)
  torch.cuda.synchronize()
  assert bool((zero == 0).all())
  # float64 reference from the bf16 inputs
  Psd = Ps.double().requires_grad_(True)
  Pdd = Pd[:T].double().requires_grad_(True)
  asd_, add_ = att_s.double().requires_grad_(True), att_d.double().requires_grad_(True)
  a_s = (Psd.view(-1, heads, C) * asd_.view(heads, C)).sum(-1)
  a_d = (Pdd.view(-1, heads, C) * add_.view(heads, C)).sum(-1)
  a_s.retain_grad(); a_d.retain_grad()
  # scores: fp32 dot of C terms
  for got, ref, P, att in ((as_, a_s, Psd, asd_), (ad[:T], a_d, Pdd, add_)):
    ab = (P.detach().abs().view(-1, heads, C) * att.detach().abs().view(heads, C)).sum(-1)
    assert bound_ratio(got, ref.detach(), gat_score_bound(ab, C)) <= 1.0
  raw = a_s[sr] + a_d[tg]
  e = F.leaky_relu(raw, 0.2)
  al = softmax_seg(e, tg, T)
  out = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add_(
      0, tg, (al.unsqueeze(-1) * Psd[sr].view(-1, heads, C)).view(-1, H))
  # alpha: relative error of the fp32 exp of (score - max), |score| * 2^-22 with margin
  kmask = [((torch.arange(k).unsqueeze(0) < deg[cum[h]:cum[h + 1]].long().unsqueeze(1)) & (ells[h].long() >= 0))
           for h, (rows, k) in enumerate(HOPS)]
  ga = torch.cat([alpha[h].view(rows, k, heads)[kmask[h].to(DEV)] for h, (rows, k) in enumerate(HOPS)], 0)
  emax = float(e.detach().abs().max()) + 1.0
  assert bound_ratio(ga.abs(), al.detach(), gat_alpha_bound(al.detach(), emax)) <= 1.0
  assert bool(((ga < 0) | ((ga == 0) & torch.signbit(ga))).eq(raw.detach() <= 0).all()), 'sign bit of alpha'
  # output: one bf16 rounding of an fp32 sum of deg weighted terms
  ab = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add_(
      0, tg, (al.detach().unsqueeze(-1) * Psd.detach()[sr].abs().view(-1, heads, C)).view(-1, H))
  kd = deg.to(DEV).double().unsqueeze(1)
  bound = weighted_sum_bound(out.detach(), ab, kd, arel=64 * EPS32 * emax)
  assert bound_ratio(Z[:T], out.detach(), bound) <= 1.0
  assert bool((Z[0] == 0).all())                          # degree-0 row without bias: exactly zero

  # ---- backward
  G = torch.randn(T, H, generator=g).to(torch.bfloat16).to(DEV)
  (out * G.double()).sum().backward()
  dal = [torch.full_like(a, 11.0) for a in alpha]
  dP = torch.zeros(N_SRC, H, device=DEV)
  da_src = torch.zeros(N_SRC, heads, device=DEV)
  da_dst = torch.full((T + 5, heads), 13.0, device=DEV)
  native.gat_backward(G, Ps, heads, ctr_t, 3, ell, ks, deg_d, alpha, dal, dP, da_src, da_dst)
  # destination scores as a separate projection
  g_as, g_ad = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
  dPs = torch.full((N_SRC, H), 9.0, dtype=torch.bfloat16, device=DEV)
  dPd = torch.full((T + 5, H), 9.0, dtype=torch.bfloat16, device=DEV)
  da_src_k, da_dst_k = da_src.clone(), da_dst.clone()
  native.gat_score_bwd(Ps, dP, da_src, att_s, g_as, dPs, ctr_s, 0, da_dst, att_d, g_ad, ctr_t, 3, P_dst=Pd,
                       dPb_dst=dPd, heads=heads)
  torch.cuda.synchronize()
  assert bool((dP == 0).all()), 'gat_score_bwd re-zeroes the fp32 source rows'
  # score gradients: terms |alpha| * (|dalpha| + |sum alpha dalpha|), each dalpha an fp32 dot of C terms
  Gd = G.double()
  dalpha_abs = (Gd[tg].abs().view(-1, heads, C) * Psd.detach()[sr].abs().view(-1, heads, C)).sum(-1)
  sabs = torch.zeros(T, heads, dtype=torch.float64, device=DEV).index_add_(0, tg, al.detach() * dalpha_abs)
  term = al.detach() * (dalpha_abs + sabs[tg])
  tol = gat_dscore_tol(C, emax, 600)
  ds_abs_src = torch.zeros(N_SRC, heads, dtype=torch.float64, device=DEV).index_add_(0, sr, term)
  ds_abs_dst = torch.zeros(T, heads, dtype=torch.float64, device=DEV).index_add_(0, tg, term)
  assert bound_ratio(da_src_k, a_s.grad, tol * ds_abs_src + 1e-30) <= 1.0
  assert bound_ratio(da_dst_k[:T], a_d.grad, tol * ds_abs_dst + 1e-30) <= 1.0
  # projection gradients (bf16): alpha G scatter + score terms
  agg_abs = torch.zeros(N_SRC, H, dtype=torch.float64, device=DEV).index_add_(
      0, sr, (al.detach().unsqueeze(-1) * Gd[tg].abs().view(-1, heads, C)).view(-1, H))
  src_abs = agg_abs + (ds_abs_src.unsqueeze(-1) * att_s.double().abs().view(heads, C)).view(N_SRC, H)
  # (+ 1e-30: alphas below fp32's range flush to zero, the float64 reference keeps them)
  assert bound_ratio(dPs, Psd.grad, bf16_ulp(Psd.grad) + tol * src_abs + 1e-30) <= 1.0
  dst_abs = (ds_abs_dst.unsqueeze(-1) * att_d.double().abs().view(heads, C)).view(T, H)
  assert bound_ratio(dPd[:T], Pdd.grad, bf16_ulp(Pdd.grad) + tol * dst_abs + 1e-30) <= 1.0
  assert bool((dPd[T:] == 0).all()), 'rows past the targets up to the next 128-row tile are zero'
  # attention vector gradients: fp32 column sums over every row
  gs_abs = (ds_abs_src.unsqueeze(-1) * Psd.detach().abs().view(-1, heads, C)).view(-1, H).sum(0)
  gd_abs = (ds_abs_dst.unsqueeze(-1) * Pdd.detach().abs().view(-1, heads, C)).view(-1, H).sum(0)
  assert bound_ratio(g_as, asd_.grad, (tol + 2000 * EPS32) * gs_abs + 1e-30) <= 1.0
  assert bound_ratio(g_ad, add_.grad, (tol + 2000 * EPS32) * gd_abs + 1e-30) <= 1.0


@pytest.mark.parametrize('heads,C', [(4, 48), (2, 128)])
def test_gat_score_bwd_folded_destination(native, heads, C):
  """A relation between rows of one type: the targets are the first rows of the source projection and their score
  gradient is folded into the same bf16 rows."""
  H = heads * C
  g = torch.Generator().manual_seed(5)
  n, T = 700, 300
  P = torch.randn(n, H, generator=g).to(torch.bfloat16).to(DEV)
  att_s = torch.randn(H, generator=g).to(torch.bfloat16).to(DEV)
  att_d = torch.randn(H, generator=g).to(torch.bfloat16).to(DEV)
  dP = torch.randn(n, H, generator=g).to(DEV)
  da_s, da_d = torch.randn(n, heads, generator=g).to(DEV), torch.randn(T, heads, generator=g).to(DEV)
  ref = dP.double() + (da_s.double().unsqueeze(-1) * att_s.double().view(heads, C)).view(n, H)
  ref[:T] += (da_d.double().unsqueeze(-1) * att_d.double().view(heads, C)).view(T, H)
  gs = (da_s.double().unsqueeze(-1) * P.double().view(n, heads, C)).view(n, H).sum(0)
  gd = (da_d.double().unsqueeze(-1) * P[:T].double().view(T, heads, C)).view(T, H).sum(0)
  out = torch.full((n + 60, H), 9.0, dtype=torch.bfloat16, device=DEV)
  g_as, g_ad = torch.zeros(H, device=DEV), torch.zeros(H, device=DEV)
  dP_in = torch.cat([dP, torch.zeros(60, H, device=DEV)])
  Pin = torch.cat([P, torch.zeros(60, H, dtype=torch.bfloat16, device=DEV)])
  native.gat_score_bwd(Pin, dP_in, torch.cat([da_s, torch.zeros(60, heads, device=DEV)]), att_s, g_as, out,
                       _counters([n]), 0, da_d, att_d, g_ad, _counters([T]), 0, heads=heads)
  torch.cuda.synchronize()
  terms = dP.double().abs() + (da_s.double().abs().unsqueeze(-1) * att_s.double().abs().view(heads, C)).view(n, H)
  terms[:T] += (da_d.double().abs().unsqueeze(-1) * att_d.double().abs().view(heads, C)).view(T, H)
  assert bound_ratio(out[:n], ref, score_bwd_bound(ref, terms)) <= 1.0
  assert bool((out[n:] == 0).all())
  ab_s = (da_s.double().abs().unsqueeze(-1) * P.double().abs().view(n, heads, C)).view(n, H).sum(0)
  ab_d = (da_d.double().abs().unsqueeze(-1) * P[:T].double().abs().view(T, heads, C)).view(T, H).sum(0)
  zero = torch.zeros(H, device=DEV)
  assert bound_ratio(g_as, gs, colsum_bound(ab_s.unsqueeze(0), zero, n) + 1e-30) <= 1.0
  assert bound_ratio(g_ad, gd, colsum_bound(ab_d.unsqueeze(0), zero, T) + 1e-30) <= 1.0


@pytest.mark.parametrize('H,heads', [(64, 1), (192, 4), (1024, 8)])
def test_gat_kernels_reject_unsupported_widths(native, H, heads):
  P = torch.zeros(128, H, dtype=torch.bfloat16, device=DEV)
  att = torch.zeros(H, dtype=torch.bfloat16, device=DEV)
  out = torch.zeros(128, heads, device=DEV)
  native.gat_scores(P, att, out, _counters([1]), 0, heads=heads)      # accepted
  for bad_heads in (3, 2 * H // 8) if H % 3 else (5, 2 * H // 8):
    with pytest.raises(RuntimeError, match='heads'):
      native.gat_scores(P, att, torch.zeros(128, bad_heads, device=DEV), _counters([1]), 0, heads=bad_heads)
  for bad_H in (96, 2048):
    Pb = torch.zeros(128, bad_H, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match='multiple of 64'):
      native.gat_scores(Pb, torch.zeros(bad_H, dtype=torch.bfloat16, device=DEV), out, _counters([1]), 0, heads=1)


# --------------------------------------------------------------------------- engine
ISOLATED = 64


def _build(feat_dim=64, hidden=64, heads=4, classes=19, dropout=0.0, fan=(4, 3, 2), bs=256, use_graph=False,
           papers=4000):
  """Synthetic IGBH plus ISOLATED extra papers with outgoing edges only (cites -> old papers, written_by -> authors):
  they have no in-neighbour in any relation, so as targets their pre-activation is exactly the (zero) bias sum, while
  their outputs still feed other targets."""
  from common import synthetic_igbh
  from graphlearn_for_pytorch_b200.models import HeteroGatEngine
  edges, feats, labels, sizes = synthetic_igbh(papers, papers // 2, 50, 30, feat_dim=64, num_classes=classes, seed=2)
  g = torch.Generator().manual_seed(3)
  add_isolated_papers(edges, sizes, ISOLATED, g, GAT_ISOLATED_EDGES)
  labels = {'paper': torch.cat([labels['paper'], torch.randint(0, classes, (ISOLATED,), generator=g)])}
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
  eng = HeteroGatEngine(graphs, tables, labels['paper'].to(DEV), feat_dim, sizes, 'paper', fanouts=list(fan),
                        batch_size=bs, hidden=hidden, heads=heads, num_classes=classes, dropout=dropout, edge_dir='in',
                        lr=5e-3, seed=1, device=DEV, use_cuda_graph=use_graph)
  eng._keep = keep
  return eng, fb, labels['paper'].to(DEV), sizes


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


def _score_signs(eng, l, r, t, nh, nn):
  """Per COO edge of relation r (hops in order, target rows in order, ELL slots below the degree) and head: the
  sign bit of the alpha the aggregation saved, i.e. whether the kernel's score took the 0.2 branch."""
  ells, ks = eng._rel_ell(r, nh)
  deg = eng.arena.deg_of(r)
  out, c = [], 0
  for h in range(nh):
    n, k = nn[t][h], ks[h]
    a = eng.alpha[(l, r)][h][:n * k * eng.heads].view(n, k, eng.heads)
    m = torch.arange(k, device=DEV).unsqueeze(0) < deg[c:c + n].long().unsqueeze(1)
    out.append(torch.signbit(a[m]))
    c += n
  return torch.cat(out)


def _reference(eng, fb, labels):
  """fp32 recomputation of the R-GAT step from the arena's COO, rounding to bf16 where the engine stores bf16 --
  activations, projections, and the gradients of the layer outputs and projections -- and applying the engine's
  dropout mask (regenerated with `dropout_bf16` from the same Philox key).

  Both leaky-ReLU branches are taken from the engine: a hidden layer's from its output Z (the kernel keeps Z > 0 <=>
  pre > 0 where the mask keeps the element), an attention score's from the sign bit of its saved alpha (set where
  the kernel's score is <= 0).  A value within rounding of zero can fall on the other side of it in the reference's
  fp32 recomputation from its own bf16 projections; its gradient would then differ 100-fold (slope 1 against 0.01)
  or 5-fold (1 against 0.2), which dominates the comparison of a whole weight row or attention vector.
  info['leaky_flips'] counts those elements."""
  nat = glt.ops.require_native()
  nodes, rows, cols, _, nn, ne = eng.arena.to_coo()
  L, nt, hd, H = eng.L, eng.nt, eng.heads, eng.hidden
  C = H // hd
  bf = lambda x: x.to(torch.bfloat16).float()   # noqa: E731
  P = {k: eng.param(k).float().requires_grad_(True) for k in eng.param_index}
  x = {t: fb[eng.ntypes[t]][nodes[t]].float() for t in range(len(eng.ntypes))}
  info = {'isolated_zero_pre': 0, 'leaky_flips': 0}
  for l in range(1, L + 1):
    nh = L - l + 1
    out = {}
    for t in eng.targets[l]:
      T = sum(nn[t][:nh])
      pre = torch.zeros(T, H, device=DEV)
      covered = torch.zeros(T, dtype=torch.bool, device=DEV)
      for r in eng.in_rel[l][t]:
        E = sum(ne[r][:nh])
        src, dst = rows[r][:E], cols[r][:E]
        covered[dst] = True
        Wd = P[('W_dst', l, r)] if ('W_dst', l, r) in P else P[('W_src', l, r)]
        hs = _BfGrad.apply(bf(x[nt[r]] @ P[('W_src', l, r)].t()))
        gd = _BfGrad.apply(bf(x[t][:T] @ Wd.t()))
        a_s = (hs.view(-1, hd, C) * P[('att_src', l, r)].view(hd, C)).sum(-1)
        a_d = (gd.view(-1, hd, C) * P[('att_dst', l, r)].view(hd, C)).sum(-1)
        raw = a_s[src] + a_d[dst]
        neg = _score_signs(eng, l, r, t, nh, nn)
        info['leaky_flips'] += int((neg != (raw.detach() <= 0)).sum())
        e = torch.where(neg, 0.2 * raw, raw)
        m = torch.full((T, hd), -float('inf'), device=DEV).scatter_reduce(
            0, dst.unsqueeze(1).expand(-1, hd), e.detach(), 'amax', include_self=True)
        ex = torch.exp(e - m[dst])
        den = torch.zeros(T, hd, device=DEV).index_add(0, dst, ex)
        al = ex / den[dst]
        pre = pre + torch.zeros(T, H, device=DEV).index_add(0, dst, (al.unsqueeze(-1) * hs[src].view(-1, hd, C))
                                                             .view(-1, H))
        pre = pre + P[('bias', l, r)]
      pre = _BfGrad.apply(pre)
      if l < L:
        ones = torch.ones_like(eng.Z[l][t])
        if eng.dropout > 0:
          nat.dropout_bf16(ones, eng.arena.counters[t * 8:t * 8 + 8], nh, eng.dropout, eng.seed, l, eng.step_dev)
        pos = eng.Z[l][t][:T] > 0
        info['leaky_flips'] += int(((ones[:T] != 0) & (pos != (pre.detach() > 0))).sum())
        z = torch.where(pos, pre, 0.01 * pre)
        if eng.dropout > 0:
          z = z * ones[:T].float()
        info['isolated_zero_pre'] += int(((~covered) & (pre.detach() == 0).all(1)).sum())
        out[t] = bf(z)
      else:
        out[t] = bf(pre)
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
    e = float((eng.param(k, grad=True) - r).abs().max()) / max(float(r.abs().max()), 1e-6)
    errs[k[0]] = max(errs.get(k[0], 0.0), e)
  return errs, info


# The attention-vector gradients get a looser bound.  They are sums of nearly cancelling terms: for att_dst,
# sum_j dscore_ij vanishes except through the leaky-ReLU slope, because the softmax weights sum to one.  So the one-ulp
# differences between the engine's bf16 projections (wgmma accumulation order) and the reference's show up amplified.
# The largest ratios observed were 0.061 (att_src) and 0.098 (att_dst), both at the IGBH widths, while the reference
# took both leaky-ReLU branches from its own fp32 values.  Since it takes them from the engine (see _reference), every
# kind stays below 0.01 at every width here, up to hidden 1024 with 16 heads.
ATT_TOL = 0.15


def _assert_match(errs):
  assert errs.pop('loss') < 3e-2, errs
  bad = {k: e for k, e in errs.items() if not e < (ATT_TOL if k.startswith('att') else 6e-2)}
  assert not bad, bad
  assert set(errs) >= {'W_src', 'att_src', 'att_dst', 'bias', 'head_W', 'head_b'}, errs


@pytest.mark.parametrize('feat_dim,hidden,heads,classes', [
    (64, 64, 4, 19),                                                           # uniform widths: one W per relation
    ({'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128}, 192, 4, 19),  # C = 48, shared and separate W
    (64, 64, 1, 2983),                                                         # one head, IGBH's 2983 classes
    (128, 256, 8, 19),                                                         # eight heads of 32
    (128, 512, 16, 19),                                                        # sixteen heads of 32
    (128, 1024, 8, 19),                                                        # the widest hidden width
], ids=['uniform-64-64-h4', 'igbh_widths-192-h4', '64-64-h1-2983', '128-256-h8', 'hidden-512-h16',
        'hidden-1024-h8'])
def test_hetero_gat_engine_gradients_match_fp32(feat_dim, hidden, heads, classes):
  eng, fb, labels, sizes = _build(feat_dim, hidden, heads, classes)
  errs, info = _gradient_errors(eng, fb, labels, sizes)
  if isinstance(feat_dim, dict):
    assert 'W_dst' in errs
  print('largest relative error per parameter kind:', {k: round(v, 4) for k, v in errs.items()},
        f"leaky-ReLU branches the fp32 recomputation would take the other way: {info['leaky_flips']}")
  _assert_match(errs)


def test_hetero_gat_engine_dropout_uses_its_mask():
  """dropout 0.5: the gradients match a recomputation with the engine's own mask, including targets without any
  in-neighbour, whose pre-activation is exactly 0 (their gradient is 0.01 G / (1 - p), not 0)."""
  eng, fb, labels, sizes = _build(dropout=0.5)
  errs, info = _gradient_errors(eng, fb, labels, sizes)
  assert info['isolated_zero_pre'] > 0, info
  print('largest relative error per parameter kind:', {k: round(v, 4) for k, v in errs.items()})
  _assert_match(errs)


def test_hetero_gat_engine_graph_replay_and_state_dict():
  """Without dropout: the sampler assigns a batch's local ids in arrival order, and the dropout mask is keyed by
  local row, so with dropout two runs of one batch drop different nodes."""
  eng, fb, labels, sizes = _build(dropout=0.0, use_graph=True)
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


def test_hetero_gat_engine_trains_under_cuda_graph_and_evaluates_without_dropout():
  eng, fb, labels, sizes = _build(dropout=0.5, use_graph=True)
  eng.warmup_and_capture(n_eager=1)
  # training progress over 60 steps
  g = torch.Generator().manual_seed(0)
  losses = []
  for i in range(60):
    losses.append(float(eng.train_step(torch.randperm(sizes['paper'], generator=g)[:eng.bs].to(DEV)).item()))
  assert all(l == l for l in losses)
  assert sum(losses[-10:]) / 10 < sum(losses[:10]) / 10 - 0.05, (losses[:5], losses[-5:])
  # evaluation: forward only, no dropout (a dropped activation would be an exact zero)
  p_before = eng.p32.clone()
  l, c, n = eng.evaluate_batch(torch.arange(eng.bs, device=DEV))
  assert n == eng.bs and 0 <= c <= n and l == l
  assert torch.equal(eng.p32, p_before) and eng._training
  pt = eng.tid['paper']
  valid = int(eng._ctr[pt][eng.L].item())
  zero_frac = float((eng.Z[1][pt][:valid] == 0).float().mean())
  assert zero_frac < 0.05, zero_frac
  eng.close()


@pytest.mark.parametrize('feat_dim,hidden,heads', [
    (96, 64, 4),                                                     # in_dim not a multiple of 64
    ({'paper': 64, 'author': 64, 'institute': 64, 'fos': 40}, 64, 4),
    (64, 96, 4),
    (64, 2048, 4),
    (64, 192, 5),                                                    # heads does not divide hidden
    (64, 64, 16),                                                    # C = 4
])
def test_hetero_gat_engine_rejects_unsupported_widths(feat_dim, hidden, heads):
  with pytest.raises(ValueError, match='in_dim|hidden|heads'):
    _build(feat_dim=feat_dim, hidden=hidden, heads=heads, papers=1000)
