"""Shared fixtures: tiny self-describing graphs (feature row v == [v]*dim)."""
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.utils.synthetic import id_features, ring_graph, rmat_edges


def ring_dataset(num_nodes=40, dim=16, graph_mode='CPU', edge_dir='out', with_gpu=False, device=None,
                 split_ratio=0.0, weights=False):
  ei = ring_graph(num_nodes)
  ds = glt.data.Dataset(edge_dir=edge_dir)
  w = (torch.arange(ei.shape[1], dtype=torch.float32) % 3 + 1.0) if weights else None
  ds.init_graph(ei, edge_weights=w, graph_mode=graph_mode, device=device, num_nodes=num_nodes)
  ds.init_node_features(id_features(num_nodes, dim), with_gpu=with_gpu, split_ratio=split_ratio, device=device)
  ds.init_edge_features(id_features(ei.shape[1], 4), with_gpu=with_gpu, device=device)
  ds.init_node_labels(torch.arange(num_nodes))
  return ds


def rmat_csr(num_nodes=2000, num_edges=40000, seed=0):
  ei = rmat_edges(num_nodes, num_edges, seed=seed)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=num_nodes)
  return ei, topo


def adjacency_sets(topo):
  ptr, ind = topo.indptr.tolist(), topo.indices.tolist()
  return [set(ind[ptr[i]:ptr[i + 1]]) for i in range(len(ptr) - 1)]


def canonical_edges(out):
  """Set of (global src, global dst) pairs of a SamplerOutput."""
  node = out.node.cpu()
  return set(zip(node[out.row.cpu()].tolist(), node[out.col.cpu()].tolist()))


# --------------------------------------------------------------------------- error bounds of GPU kernels
def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
  """Spacing of bf16 numbers at |x| (float64): 2^(e - 7) for |x| in [2^e, 2^(e+1)); the smallest normal spacing at 0."""
  x = x.double().abs()
  _, e = torch.frexp(x)                     # x = m * 2^e, m in [0.5, 1)
  return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e - 8), torch.full_like(x, 2.0 ** -133))


def gemm_bound(ref: torch.Tensor, absprod: torch.Tensor, k: int, bf16_out: bool = True) -> torch.Tensor:
  """Largest error of a bf16 GEMM with fp32 accumulation over a contraction of length k: k * 2^-22 * (|A| . |W|^T)
  (fp32 summation with margin for truncating adders), plus one bf16 ulp of the result for a bf16 output.  `ref` and
  `absprod` are float64; for a split-K fp32 output (`bf16_out=False`) only the summation term applies."""
  b = float(k) * 2.0 ** -22 * absprod.double()
  return b + bf16_ulp(ref) if bf16_out else b


EPS32 = 2.0 ** -23


def sum_bound(n, abs_sum: torch.Tensor) -> torch.Tensor:
  """Largest error of an fp32 sum of n terms (in any order, each term rounded once): (n + 1) * 2^-23 * sum|terms|."""
  n = n.double() if torch.is_tensor(n) else float(n)
  return (n + 1) * EPS32 * abs_sum.double()


def mean_ref(X: torch.Tensor, tgt: torch.Tensor, src: torch.Tensor, deg: torch.Tensor):
  """float64 mean aggregation sum_{edges t <- s} X[s] / deg[t] over the T = deg.numel() targets, and its error bound:
  one bf16 ulp of the mean, plus the fp32 sum of deg rows and the multiplication by the fp32 1/deg; rows of degree 0
  must be exactly 0."""
  Xd = X.double()
  T, d = deg.numel(), X.shape[1]
  s = torch.zeros(T, d, dtype=torch.float64, device=X.device).index_add_(0, tgt, Xd[src])
  a = torch.zeros(T, d, dtype=torch.float64, device=X.device).index_add_(0, tgt, Xd[src].abs())
  dg = deg.to(X.device).double().unsqueeze(1)
  ref = s / dg.clamp(min=1)
  bound = torch.where(dg > 0, bf16_ulp(ref) + (dg + 2) * EPS32 * a / dg.clamp(min=1), torch.zeros_like(ref))
  return ref, bound


def gather_ref(dA, d, Z, tgt, src, deg, T, S, cap_src, gscale):
  """float64 dPre of sage_gather_bwd (dPre[s] = relu'(Z[s]) * gscale * (dA[s, d:] if s < T + sum_{t <- s} dA[t, :d] /
  deg[t])) and its error bound, from the exact bf16 operands and the edges (tgt, src) of the layer's hops; the bound is
  0 (exact) on masked elements and on rows in [S, cap_src)."""
  dev = dA.device
  keep = (tgt < T) & (src < S)
  tgt, src = tgt[keep], src[keep]
  inv = (1.0 / deg.float()).double()                   # fp32 1/deg, as the kernel computes it
  dAd = dA.double()
  terms = dAd[tgt, :d] * inv[tgt].unsqueeze(1)
  ref = torch.zeros(cap_src, d, dtype=torch.float64, device=dev)
  ab = torch.zeros_like(ref)
  m = min(T, S)
  ref[:m] = dAd[:m, d:]
  ab[:m] = dAd[:m, d:].abs()
  ref.index_add_(0, src, terms)
  ab.index_add_(0, src, terms.abs())
  n = torch.bincount(src, minlength=cap_src).double()
  n[:m] += 1
  g = float(torch.tensor(gscale, dtype=torch.float32))
  live = (torch.arange(cap_src, device=dev) < S).unsqueeze(1)
  mask = live & (Z[:cap_src] > 0) if Z is not None else live.expand(cap_src, d)
  ref = torch.where(mask, ref * g, torch.zeros_like(ref))
  bound = torch.where(mask, bf16_ulp(ref) + g * sum_bound((n + 2).unsqueeze(1), ab),torch.zeros_like(ref))
  return ref, bound


def colsum_ratio(colsum: torch.Tensor, X: torch.Tensor, S: int, init: float = 0.0) -> float:
  """Error / bound of fp32 column sums (bias gradients) of the first S rows of X accumulated onto `init`."""
  x = X[:S].double()
  return bound_ratio(colsum, x.sum(0) + init, sum_bound(S, x.abs().sum(0) + abs(init)))


def bound_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
  """max |got - ref| / bound over all elements (<= 1 when every element lies within its bound; 0-bound elements
  must match exactly)."""
  err = (got.double() - ref.double()).abs()
  if err.numel() == 0:
    return 0.0
  exact = bound <= 0
  if bool((err[exact] > 0).any()):
    return float('inf')
  return float((err[~exact] / bound[~exact]).max()) if bool((~exact).any()) else 0.0


# --------------------------------------------------------------------------- per-stage checks of a real training step
DEV = torch.device('cuda', 0)
U = 2.0 ** -24


class Ratios(object):
  """Worst error / bound per stage of one step; `check` asserts each ratio <= 1 as it is recorded."""

  def __init__(self, tag):
    self.tag, self.r = tag, {}

  def check(self, stage, ratio):
    self.r[stage] = max(self.r.get(stage, 0.0), ratio)
    assert ratio <= 1.0, f'{self.tag}: {stage} error / bound = {ratio}'

  def exact(self, stage, ok):
    self.check(stage, 0.0 if ok else float('inf'))

  def show(self):
    print(f'{self.tag}: ' + ', '.join(f'{k} {v:.3f}' for k, v in self.r.items()))


def _f32(x):
  return float(torch.tensor(x, dtype=torch.float32))


def _batches(bs, N, g):
  """Seed batches of bs, about bs / 3, 1 and bs nodes (the small ones padded with -1 by train_step)."""
  return [torch.randperm(N, generator=g)[:n].to(DEV) for n in (bs, max(1, bs // 3), 1, bs)]


def _ell_edges(ell_of, deg, ctr, nh, caps, ks):
  """(target, source) of the ELL hops 0..nh-1: frontier rows of hop h are [ctr[h], ctr[h+1]) clamped to the hop's
  capacity, slots inside the row's degree, sources >= 0.  A hop of fan-out 0 has no ELL block; its rows must have
  degree 0."""
  tg, sr = [], []
  for h in range(nh):
    k = ks[h]
    n = max(0, min(ctr[h + 1] - ctr[h], caps[h]))
    if n == 0:
      continue
    if k == 0:
      assert not bool(deg[ctr[h]:ctr[h] + n].any()), f'rows of hop {h} (fan-out 0) must have degree 0'
      continue
    e = ell_of(h).view(-1, k)[:n].long()
    m = (torch.arange(k, device=DEV).unsqueeze(0) < deg[ctr[h]:ctr[h] + n].long().unsqueeze(1)) & (e >= 0)
    tg.append((torch.arange(n, device=DEV).unsqueeze(1) + ctr[h]).expand(n, k)[m])
    sr.append(e[m])
  empty = torch.zeros(0, dtype=torch.int64, device=DEV)
  return torch.cat(tg + [empty]), torch.cat(sr + [empty])


def _check_linear(R, stage, A, W, b, Z, T, relu, keep=None, scale=1.0):
  """Z[:T] against bf16(act(A W^T + b)) (then inverted dropout with mask `keep`)."""
  Ad, Wd = A[:T].double(), W.double()
  ref = Ad @ Wd.t() + b.double()
  bound = gemm_bound(ref, Ad.abs() @ Wd.abs().t() + b.double().abs(), A.shape[1])
  if relu:
    ref = ref.clamp(min=0)
  if keep is not None:
    ref = torch.where(keep, ref * scale, torch.zeros_like(ref))
    bound = torch.where(keep, bound * scale + bf16_ulp(ref), torch.zeros_like(ref))
  R.check(stage, bound_ratio(Z[:T], ref, bound))


def _wgrad_ratio(gW, dPre, A, T):
  Pd, Ad = dPre[:T].double(), A[:T].double()
  return bound_ratio(gW, Pd.t() @ Ad, gemm_bound(None, Pd.abs().t() @ Ad.abs(), T, bf16_out=False))


def _check_grads(R, stage, gW, dPre, A, W, dA, T):
  """dW = dPre[:T]^T A[:T] (split-K fp32) and, when dA is given, dA[:T] = bf16(dPre[:T] W)."""
  R.check(f'dW{stage}', _wgrad_ratio(gW, dPre, A, T))
  if dA is not None:
    Pd, Wd = dPre[:T].double(), W.double()
    ref = Pd @ Wd
    R.check(f'dA{stage}', bound_ratio(dA[:T], ref, gemm_bound(ref, Pd.abs() @ Wd.abs(), W.shape[0])))


def _check_softmax(R, Z, C, labels, nodes, n0, dPre, bias_grad, loss, correct):
  xs = Z[:n0, :C].double()
  lab = labels[nodes[:n0]]
  ref_loss = F.cross_entropy(xs, lab)
  R.check('loss', abs(loss.item() - ref_loss.item()) / (1e-4 * max(1.0, ref_loss.item())))
  mx = xs.max(1, keepdim=True).values
  first = torch.where(xs == mx, torch.arange(C, device=DEV), C).min(1).values
  R.exact('correct', int(correct.item()) == int((first == lab).sum()))
  ref = (torch.softmax(xs, 1) - F.one_hot(lab, C).double()) / n0
  R.check('dlogits', bound_ratio(dPre[:n0, :C], ref, bf16_ulp(ref) + 1e-4 / n0))
  R.exact('dlogits pad', bool((dPre[:n0, C:] == 0).all()))
  R.check('db_last', colsum_ratio(bias_grad, dPre, n0))


def _adam_ref(p, g, m, v, t, lr, wd, b1=0.9, b2=0.999, eps=1e-8):
  """float64 torch.optim.Adam(weight_decay=wd) update from fp32 state, with the fp32 constants the kernel receives,
  and the bounds of its fp32 evaluation: 2u per rounded sum of products, one u for each bias correction."""
  lr, wd, b1, b2, eps = (_f32(x) for x in (lr, wd, b1, b2, eps))
  p, g, m, v = p.double(), g.double(), m.double(), v.double()
  gi = g + wd * p
  e_g = 2 * U * (g.abs() + (wd * p).abs())
  m1 = b1 * m + (1 - b1) * gi
  v1 = b2 * v + (1 - b2) * gi * gi
  e_m = 2 * U * (b1 * m.abs() + (1 - b1) * gi.abs()) + (1 - b1) * e_g
  e_v = 3 * U * (b2 * v + (1 - b2) * gi * gi) + (1 - b2) * 2 * gi.abs() * e_g
  c1, c2 = 1 - b1 ** t, 1 - b2 ** t
  M, V = m1 / c1, v1 / c2
  dM = e_m / c1 + M.abs() * 2 * U
  dV = e_v / c2 + V * 2 * U
  S = V.sqrt()
  dS = torch.minimum(dV.sqrt(), dV / (2 * S).clamp(min=1e-300)) + U * S
  D = S + eps
  upd = M / D
  dU = dM / D + M.abs() * (dS + U * D) / (D * D) + U * upd.abs()
  p1 = p - lr * upd
  dP = lr * dU + 2 * U * (lr * upd.abs() + p1.abs())
  return (p1, m1, v1), (dP, e_m, e_v)


def _check_adam(R, eng, snap, wd, controls=False):
  t = int(snap['step'][0]) + 1
  (p1, m1, v1), (bp, bm, bv) = _adam_ref(snap['p32'], eng.g32, snap['m'], snap['v'], t, eng.lr, wd)
  R.check('adam p', bound_ratio(eng.p32, p1, bp))
  R.check('adam m', bound_ratio(eng.m, m1, bm))
  R.check('adam v', bound_ratio(eng.v, v1, bv))
  R.exact('p16', torch.equal(eng.p16.view(torch.int16), eng.p32.to(torch.bfloat16).view(torch.int16)))
  R.exact('step_dev', eng.step_dev.tolist() == [t, 0])
  ratios = {}
  if controls:
    # the same check rejects Adam without weight decay and Adam with t off by one
    (q, _, _), _ = _adam_ref(snap['p32'], eng.g32, snap['m'], snap['v'], t, eng.lr, 0.0)
    ratios['Adam without weight decay'] = bound_ratio(q.float(), p1, bp)
    assert ratios['Adam without weight decay'] > 1.0, 'the Adam check must reject an update without weight decay'
    (q, _, _), _ = _adam_ref(snap['p32'], eng.g32, snap['m'], snap['v'], t + 1, eng.lr, wd)
    ratios['Adam with t off by one'] = bound_ratio(q.float(), p1, bp)
    assert ratios['Adam with t off by one'] > 1.0, 'the Adam check must reject an update with t off by one'
  return ratios


def _snapshot(eng, dpre):
  s = {k: getattr(eng, k).clone() for k in ('p32', 'p16', 'm', 'v')}
  s['step'] = eng.step_dev.clone()
  s['dPre'] = dpre()
  return s


def _table(x):
  ut = glt.data.UnifiedTensor(0, x.dtype)
  ut.append_shared_tensor(x)
  return ut


GAT_ISOLATED_EDGES = {('paper', 'cites', 'paper'): 4, ('paper', 'written_by', 'author'): 3}   # per isolated paper


def add_isolated_papers(edges, sizes, n, g, per_node):
  """n extra papers that only send edges: per_node[etype] edges out of each new paper, for the relations named there,
  drawn from g in the order of `edges` (destinations: the old papers, or the relation's destination type).  As targets
  the new papers have no in-neighbour in any relation, while their outputs still feed other targets.  Returns the first
  new id (the old paper count); sizes['paper'] grows by n."""
  n_old = sizes['paper']
  new = torch.arange(n_old, n_old + n)
  for et in list(edges):
    k = per_node.get(et, 0)
    if k:
      n_dst = n_old if et[2] == 'paper' else sizes[et[2]]
      extra = torch.stack([new.repeat_interleave(k), torch.randint(0, n_dst, (k * n,), generator=g)])
      edges[et] = torch.cat([edges[et], extra], 1)
  sizes['paper'] = n_old + n
  return n_old


# --------------------------------------------------------------------------- float64 references of the attention kernels
# Shared by the kernel tests (hand-built buffers) and the step-stage test (a real step's buffers).  u = 2^-24 is fp32's
# unit roundoff, EPS32 = 2u.  The fp32 library functions are IEEE-accurate builds (expf, erff within 2 ulp):
#   sigmoid  1 / (1 + expf(-s)) is within 2^-22 of sigma(s); SIG_ERR = 2^-21 leaves a factor of two
#   gelu     1 + erff(x / sqrt 2) is within 2^-21 of 1 + erf(x / sqrt 2)
SIG_ERR = 2.0 ** -21
ERF_ERR = 2.0 ** -21


def softmax_seg(e, tg, T):
  """Segment softmax of e [E, heads] over the targets tg (float64)."""
  heads = e.shape[1]
  m = torch.full((T, heads), -float('inf'), dtype=e.dtype, device=e.device)
  m = m.scatter_reduce(0, tg.unsqueeze(1).expand(-1, heads), e, 'amax', include_self=True)
  ex = torch.exp(e - m[tg])
  den = torch.zeros(T, heads, dtype=e.dtype, device=e.device).index_add_(0, tg, ex)
  return ex / den[tg]


def colsum_bound(x, s0, n):
  """fp32 sum of n terms (the rows of x, float64) onto s0: (n + 2) EPS32 (sum |x| + |s0|), per column."""
  return (n + 2) * EPS32 * (x.abs().sum(0) + s0.double().abs())


def weighted_sum_bound(ref, ab, n, arel=0.0, bf16_out=True, floor=0.0):
  """An attention output sum_j alpha_j x_j of n fp32 terms: (n + 2) EPS32 sum alpha |x| for the summation, plus arel
  sum alpha |x| when the reference's alpha is float64 and the kernel's carries a relative error arel (0 when the
  reference reads the kernel's own alpha), one bf16 ulp for a bf16 result, and an absolute floor."""
  b = ((n + 2) * EPS32 + arel) * ab + floor
  return b + bf16_ulp(ref) if bf16_out else b


def gat_score_bound(ab, C):
  """gat_scores: an fp32 dot of C terms, against sum |terms| = ab."""
  return (C + 2) * EPS32 * ab + 1e-30


def gat_alpha_bound(al, emax):
  """gat_aggregate alpha: relative error of the fp32 exp of (score - max), |score| * 2^-22 with margin; emax is
  max |score| + 1."""
  return 64 * EPS32 * emax * al + 1e-30


def gat_dscore_tol(C, emax, n_terms):
  """Relative tolerance of the GAT score gradients (gat_backward's da_src / da_dst, and through them the projection
  gradients) against their terms alpha (|dalpha| + sum alpha |dalpha|): C for each fp32 dot dalpha, 64 emax for an
  alpha whose reference is float64 (0 when the reference reads the kernel's alpha), n_terms for the fp32 sums (the
  kernel tests' 600 covers their k = 512 hub; the step test passes its largest row degree plus source count)."""
  return (C + 64 * emax + n_terms) * EPS32


def score_bwd_bound(ref, terms):
  """gat_score_bwd's bf16 projection gradient dP + da att from its actual fp32 inputs: one bf16 ulp plus two fp32
  fmas over sum |terms|."""
  return bf16_ulp(ref) + 4 * EPS32 * terms + 1e-30


def act_bwd_ref(dH, Z, keep, scale):
  """gat_act_bwd: bf16(dH leaky'(Z) keep scale) and its bound (one bf16 ulp; every factor is exact in fp32)."""
  ref = dH.double() * torch.where(Z > 0, 1.0, 0.01).double() * keep.double() * scale
  return ref, bf16_ulp(ref)


def gelu64(x):
  return 0.5 * x * (1 + torch.erf(x / 2 ** 0.5))


def gelu_grad64(x):
  return 0.5 * (1 + torch.erf(x / 2 ** 0.5)) + x * torch.exp(-0.5 * x * x) / (2 * torch.pi) ** 0.5


def gelu_ref(x):
  """hgt_gelu forward from float64 X: Y = 0.5 x (1 + erf) errs by 0.5 |x| ERF_ERR plus u |Y|, twice over."""
  ref = gelu64(x)
  return ref, bf16_ulp(ref) + 2 * (0.5 * x.abs() * ERF_ERR + EPS32 * ref.abs())


def gelu_bwd_ref(x, gy):
  """hgt_gelu backward dY gelu'(X): 0.5 (1 + erf) errs by 2^-22, x 0.39894228 expf(-0.5 x x) by (0.5 x^2 + 7) u of
  itself, the sum and the product with dY by u each."""
  ref = gy * gelu_grad64(x)
  t1 = 0.5 * (1 + torch.erf(x / 2 ** 0.5))
  t2 = (x * torch.exp(-0.5 * x * x)).abs() / (2 * torch.pi) ** 0.5
  err = gy.abs() * (ERF_ERR / 2 + (0.5 * x * x + 7) * EPS32 / 2 * t2 + EPS32 * (t1 + t2))
  return ref, bf16_ulp(ref) + 2 * err


def gate_ref(a, x, sg):
  """hgt_gate forward sigma A + (1 - sigma) X."""
  ref = sg * a + (1 - sg) * x
  return ref, bf16_ulp(ref) + 2 * (SIG_ERR * (a.abs() + x.abs()) + EPS32 * (sg * a.abs() + (1 - sg) * x.abs()))


def gate_da_ref(gz, sg):
  """hgt_gate backward dA = bf16(sigma dZ)."""
  ref = sg * gz
  return ref, bf16_ulp(ref) + 2 * (SIG_ERR + EPS32 * sg) * gz.abs()


def gate_dx_ref(dx0, gz, sg):
  """hgt_gate backward dX += (1 - sigma) dZ in fp32."""
  ref = dx0 + (1 - sg) * gz
  return ref, SIG_ERR * gz.abs() + 2 * EPS32 * (dx0.abs() + 2 * (1 - sg) * gz.abs())


def skip_g_ref(s0, sg, t, n_terms):
  """hgt_gate's skip gradient s0 + sigma' sum t (t = dZ (A - X)): an fp32 sum whose longest chain of roundings has
  n_terms terms, onto s0, and sigma'(skip) within 2^-20 (two factors within SIG_ERR).  n_terms = T d is valid for any
  summation order (the kernel tests); the step test passes the kernel's own chain -- each thread's grid-stride share,
  a warp tree, the CTA's warps, one atomic per CTA -- which is much shorter and tight enough to see a sign error."""
  dsg = sg * (1 - sg)
  ref = s0.double() + dsg * t.sum()
  bound = (n_terms + 2) * EPS32 * (dsg * t.abs().sum() + s0.double().abs()) + 2 * SIG_ERR * t.abs().sum()
  return ref, bound


def block_images(att, msg):
  """hgt_blocks: the block-diagonal images att_img [R H, H] and msg_img [H, R H] of [R, heads, D, D] blocks."""
  R = att.shape[0]
  ref_a = torch.cat([torch.block_diag(*att[r]) for r in range(R)], 0)
  ref_m = torch.cat([torch.block_diag(*msg[r].transpose(1, 2)) for r in range(R)], 1)
  return ref_a, ref_m


def block_grads(att_d, msg_d, R, heads, D):
  """The diagonal blocks [R, heads, D, D] of the dense weight gradients att_d [R H, H] and msg_d [H, R H]."""
  blk_a = torch.diagonal(att_d.view(R, heads, D, heads, D), dim1=1, dim2=3).permute(0, 3, 1, 2)
  blk_m = torch.diagonal(msg_d.view(heads, D, R, heads, D), dim1=0, dim2=3).permute(1, 3, 2, 0)
  return blk_a, blk_m


def hgt_score_err(cabs, pr_abs, s, D):
  """Error of an hgt_attention score <qq, k> prior / sqrt(D): an fp32 dot of D terms (cabs = sum |terms| / sqrt(D))
  times |prior|, and the products."""
  return (D + 4) * EPS32 * cabs * pr_abs + 4 * EPS32 * s.abs()


def hgt_alpha_rel(s, serr, tg, T):
  """Relative error of every hgt_attention alpha (per edge and head): 64 EPS32 (max |s| + 1) for the exp of the
  shifted scores and twice the largest score error of the target row."""
  heads = s.shape[1]
  emax = float(s.abs().max()) + 1.0 if s.numel() else 1.0
  serr_row = torch.zeros(T, heads, dtype=torch.float64, device=s.device).scatter_reduce(
      0, tg.unsqueeze(1).expand(-1, heads), serr, 'amax', include_self=True)
  return 64 * EPS32 * emax + 2 * serr_row[tg]


def hgt_bwd_tol(D, n_terms, arel_max):
  """Relative tolerance of hgt_attention_bwd's dqq / dK / dV against their terms (D for each fp32 dot, n_terms for
  the fp32 sums, arel_max for an alpha whose reference is float64; 0 when the reference reads the kernel's alpha)."""
  return (n_terms + D) * EPS32 + arel_max
