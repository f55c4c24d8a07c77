"""The engine's SIMT kernels (csrc/cuda/sage.cu) at every width they accept, against float64 references.

The aggregation / scatter kernels pick their lane-group shape from the row width (GLT_DISPATCH_WIDTH: 4, 8, 16 or 32
lanes per row, 1, 2 or 4 vectors per lane), and the bias-gradient column sums have width-dependent paths.  Each test
builds the sampler's layout by hand -- per-hop ELL blocks, `deg`, cumulative counters, source rows -- so that every
edge case is placed on purpose: rows of degree 0, 1 and exactly k (one hub row with k = 512), ELL slots past the
degree holding valid ids that must not be read, three hops of different k, counters above the buffer capacity.

References are computed in float64 from the exact bf16 values the kernel reads, and every comparison is a bound:
one bf16 ulp for a bf16 result, n * 2^-23 * sum|terms| for an fp32 sum of n terms (tests/helpers.py).
"""
import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from helpers import bf16_ulp, bound_ratio, mean_ref, sum_bound

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
SENTINEL = 7.0

# both sides of every lane-group boundary of GLT_DISPATCH_WIDTH (8 columns = one 16-byte vector)
AGG_WIDTHS = [8, 32, 40, 64, 72, 128, 136, 256, 264, 512, 520, 1024]
# divisors of 2048 (bias gradient fused into the cast) and widths that are not
CAST_WIDTHS = [8, 64, 96, 192, 200, 384, 512, 768, 1024, 2048]
CLASSES = [8, 47, 172, 256, 300, 1000, 2983]
HOPS = [(3, 512), (50, 7), (400, 3)]          # (rows, k): a hub hop, then two ordinary hops


def _structure(n_src, seed):
  """Per-hop ELL blocks of HOPS over sources [0, n_src): first rows of each hop have degree 0, 1 and k; the slots past
  a row's degree hold valid ids (a kernel that reads them sums wrong rows)."""
  g = torch.Generator().manual_seed(seed)
  cum, degs, ells = [0], [], []
  for rows, k in HOPS:
    deg = torch.randint(0, k + 1, (rows,), generator=g)
    deg[:3] = torch.tensor([0, 1, k])
    ells.append(torch.randint(0, n_src, (rows, k), generator=g).to(torch.int32))
    degs.append(deg.to(torch.int32))
    cum.append(cum[-1] + rows)
  return cum, torch.cat(degs), ells


def _edges(cum, deg, ells, T):
  """(target, source) of every edge of the first T target rows."""
  tg, sr = [], []
  for h, (rows, k) in enumerate(HOPS):
    n = max(0, min(T, cum[h + 1]) - cum[h])
    if n == 0:
      continue
    e = ells[h][:n].long()
    m = torch.arange(k).unsqueeze(0) < deg[cum[h]:cum[h] + n].long().unsqueeze(1)
    tg.append((torch.arange(n).unsqueeze(1) + cum[h]).expand(n, k)[m])
    sr.append(e[m])
  return torch.cat(tg).to(DEV), torch.cat(sr).to(DEV)


def _counters(cum, total=None):
  c = torch.zeros(16, dtype=torch.int32)
  c[:len(cum)] = torch.tensor(cum, dtype=torch.int32)
  if total is not None:
    c[len(cum) - 1] = total
  return c.to(DEV)


def _args(cum, deg, ells):
  return [e.flatten().to(DEV) for e in ells], [k for _, k in HOPS], deg.to(DEV)


def _sources(n_src, d, seed, table):
  """bf16 source rows [n_src, d]; table=True also returns a UnifiedTensor holding them under a node-id map, its rows
  split between HBM and pinned host memory."""
  g = torch.Generator().manual_seed(seed)
  if not table:
    return (torch.randn(n_src, d, generator=g) * 2).to(torch.bfloat16).to(DEV), None, None
  n_glob = n_src + 97
  X = (torch.randn(n_glob, d, generator=g) * 2).to(torch.bfloat16)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(X[:n_glob // 2].to(DEV))
  ut.append_cpu_tensor(X[n_glob // 2:].clone())
  nodes = torch.randperm(n_glob, generator=g)[:n_src]
  return X[nodes].to(DEV), ut, nodes.to(DEV)


# --------------------------------------------------------------------------- aggregation
@pytest.mark.parametrize('block', [False, True])
@pytest.mark.parametrize('table', [False, True])
@pytest.mark.parametrize('d', AGG_WIDTHS)
def test_sage_aggregate_matches_fp64_mean(native, d, table, block):
  cum, deg, ells = _structure(600, seed=d)
  ell, ks, deg_d = _args(cum, deg, ells)
  X, ut, nodes = _sources(600, d, seed=d + 1, table=table)
  feat = ut._table() if table else None
  src_local = None if table else X
  ratio = 0.0
  # spare rows above the batch, then counters above the capacity (the kernel clamps to the buffer's rows)
  for cap, total in ((cum[-1] + 37, None), (cum[-1] - 20, cum[-1] + 1000)):
    ctr = _counters(cum, total)
    T = min(cum[-1] if total is None else total, cap)
    ld, mcol = (2 * d + 24, 16) if block else (2 * d, 0)
    out = torch.full((cap, ld), SENTINEL, dtype=torch.bfloat16, device=DEV)
    if block:
      native.sage_aggregate_block(feat, nodes, src_local, d, ctr, 3, ell, ks, deg_d, out, mcol)
    else:
      native.sage_aggregate(feat, nodes, src_local, d, ctr, 3, ell, ks, deg_d, out)
    torch.cuda.synchronize()
    tg, sr = _edges(cum, deg, ells, T)
    ref, bound = mean_ref(X, tg, sr, deg[:T])
    r = bound_ratio(out[:T, mcol:mcol + d], ref, bound)
    assert r <= 1.0, (d, table, block, cap, r)
    ratio = max(ratio, r)
    if not block:
      assert torch.equal(out[:T, d:], X[:T]), 'self half must be the source row, bit for bit'
    else:
      assert bool((out[:, :mcol] == SENTINEL).all()) and bool((out[:, mcol + d:] == SENTINEL).all())
    assert bool((out[T:] == SENTINEL).all()), 'rows at and above T must not be written'
  print(f'aggregate d={d} table={table} block={block}: max error / bound = {ratio:.3f}')


# --------------------------------------------------------------------------- scatter backward
@pytest.mark.parametrize('layout', ['rows', 'block'])
@pytest.mark.parametrize('d', AGG_WIDTHS)
def test_sage_scatter_matches_fp64_sum(native, d, layout):
  """rows: dA rows are [mean | self]; block: the mean and self blocks sit at offsets inside wider, padded rows."""
  n_src = 500                                  # ~1900 edges: sources are shared by many target rows
  cum, deg, ells = _structure(n_src, seed=d + 7)
  ell, ks, deg_d = _args(cum, deg, ells)
  g = torch.Generator().manual_seed(d)
  ratio = 0.0
  for cap, total in ((cum[-1] + 37, None), (cum[-1] - 20, cum[-1] + 1000)):
    ctr = _counters(cum, total)
    T = min(cum[-1] if total is None else total, cap)
    ld, mcol, scol = (2 * d + 32, 8, d + 24) if layout == 'block' else (2 * d, 0, d)
    dA = (torch.randn(cap, ld, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
    init = torch.randn(n_src, d, generator=g).to(DEV)
    dH = init.clone()
    native.sage_scatter_block(dA, d, mcol, ctr, 3, ell, ks, deg_d, dH)
    native.add_block_f32(dA, scol, d, ctr, 3, dH)
    torch.cuda.synchronize()
    tg, sr = _edges(cum, deg, ells, T)
    dAd = dA.double()
    dg = deg.to(DEV).double()
    terms = dAd[tg, mcol:mcol + d] / dg[tg].unsqueeze(1)
    ref = init.double().clone()
    ref[:T] += dAd[:T, scol:scol + d]
    ref.index_add_(0, sr, terms)
    a = init.double().abs()
    a[:T] += dAd[:T, scol:scol + d].abs()
    a.index_add_(0, sr, terms.abs())
    n = torch.ones(n_src, dtype=torch.float64, device=DEV)
    n[:T] += 1
    n += torch.bincount(sr, minlength=n_src).double()
    # fp32 summation of n terms (the initial value, the self term and one term per edge), each rounded once
    bound = sum_bound(n.unsqueeze(1), a)
    r = bound_ratio(dH, ref, bound)
    assert r <= 1.0, (d, layout, cap, r)
    ratio = max(ratio, r)
    untouched = n == 1
    assert torch.equal(dH[untouched], init[untouched]), 'rows without a term must keep their value'
  print(f'scatter d={d} layout={layout}: max error / bound = {ratio:.3f}')


# --------------------------------------------------------------------------- relu_bwd_cast
@pytest.mark.parametrize('prezeroed', [True, False])
@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('d', CAST_WIDTHS)
def test_relu_bwd_cast_bits_and_bias_gradient(native, d, relu, prezeroed):
  cap, T, gscale = 3000, 2777, 1.0 / (1.0 - 0.3)
  g = torch.Generator().manual_seed(d)
  dH = torch.randn(cap + 5, d, generator=g).to(DEV)
  Z = torch.randn(cap + 9, d, generator=g).to(torch.bfloat16).to(DEV)
  dPre = torch.full((cap, d), SENTINEL, dtype=torch.bfloat16, device=DEV)
  colsum = torch.zeros(d, device=DEV) if prezeroed else torch.full((d,), 3.0, device=DEV)
  ctr = _counters([0, 1000, T])
  native.relu_bwd_cast(dH, Z, ctr, 2, dPre, colsum, prezeroed, gscale, relu=relu)
  torch.cuda.synchronize()
  g32 = dH[:T] * torch.tensor(gscale, dtype=torch.float32, device=DEV)      # fp32 product, as in the kernel
  exp = torch.where(Z[:T] > 0, g32, torch.zeros_like(g32)) if relu else g32
  assert torch.equal(dPre[:T].view(torch.int16), exp.to(torch.bfloat16).view(torch.int16)), 'dPre must be bf16(mask dH s)'
  assert bool((dPre[T:] == 0).all()), 'rows in [T, cap) must be zero'
  x = dPre[:T].double()
  ref = x.sum(0)
  bound = sum_bound(T, x.abs().sum(0))
  r = bound_ratio(colsum, ref, bound)
  print(f'relu_bwd_cast d={d} relu={relu} prezeroed={prezeroed}: bias gradient error / bound = {r:.3f}')
  assert r <= 1.0, f'bias gradient (column sums of dPre) wrong at d={d}: error / bound = {r}'


# --------------------------------------------------------------------------- softmax_nll
@pytest.mark.parametrize('via_nodes', [False, True])
@pytest.mark.parametrize('C', CLASSES)
def test_softmax_nll_matches_fp64(native, C, via_nodes):
  ld = (C + 63) // 64 * 64
  cap, n0 = 320, 301                           # n0 is not a multiple of the 8 warps of a block
  g = torch.Generator().manual_seed(C)
  x = torch.randn(cap, ld, generator=g) * 2
  x[::2] = x[::2].round()                      # integer logits: ties for the arg-max
  logits = x.to(torch.bfloat16).to(DEV)
  if via_nodes:
    nodes = torch.randperm(5000, generator=g)[:cap].to(DEV)
    labels_all = torch.randint(0, C, (5000,), generator=g).to(DEV)
    y, label = None, labels_all[nodes]
  else:
    nodes = labels_all = None
    y = torch.randint(0, C, (cap,), generator=g).to(DEV)
    label = y
  loss = torch.full((1,), 5.0, device=DEV)
  correct = torch.full((1,), 99, dtype=torch.int32, device=DEV)
  colsum = torch.full((ld,), 3.0, device=DEV)
  dl = torch.full((cap, ld), SENTINEL, dtype=torch.bfloat16, device=DEV)
  ctr = _counters([0, n0])
  native.softmax_nll(logits, C, y, labels_all, nodes, ctr, loss, dl, correct, colsum, False)
  torch.cuda.synchronize()
  xs = logits[:n0, :C].double()
  lab = label[:n0]
  ref_loss = F.cross_entropy(xs, lab)
  assert abs(loss.item() - ref_loss.item()) <= 1e-4 * max(1.0, ref_loss.item()), (loss.item(), ref_loss.item())
  ref = (torch.softmax(xs, 1) - F.one_hot(lab, C).double()) / n0
  # one bf16 ulp, plus the fast exp / log of the kernel (relative error < 1e-5 of p and of 1 - p)
  r = bound_ratio(dl[:n0, :C], ref, bf16_ulp(ref) + 1e-4 / n0)
  assert r <= 1.0, ('dlogits', C, r)
  assert bool((dl[:n0, C:] == 0).all()) and bool((dl[n0:] == 0).all()), 'padding columns and rows >= n0 are zero'
  mx = xs.max(1, keepdim=True).values
  first = torch.where(xs == mx, torch.arange(C, device=DEV), C).min(1).values
  assert int(correct.item()) == int((first == lab).sum()), 'correct counts first-index arg-max hits'
  db = dl[:n0].double()
  rc = bound_ratio(colsum, db.sum(0), sum_bound(n0, db.abs().sum(0)))
  print(f'softmax_nll C={C} via_nodes={via_nodes}: dlogits error / bound = {r:.3f}, bias gradient {rc:.3f}')
  assert rc <= 1.0, f'bias gradient (column sums of dlogits) wrong at C={C}: error / bound = {rc}'


# --------------------------------------------------------------------------- colsum_bf16
@pytest.mark.parametrize('d', [8, 96, 200, 1000, 2048])
def test_colsum_bf16_matches_fp64(native, d):
  cap, T = 1100, 1001                          # 1001 is not a multiple of any rows-per-block (256 / (d / 8))
  X = torch.randn(cap, d, generator=torch.Generator().manual_seed(d)).to(torch.bfloat16).to(DEV)
  out = torch.full((d,), 3.0, device=DEV)
  native.colsum_bf16(X, _counters([0, 500, T]), 2, out)
  torch.cuda.synchronize()
  x = X[:T].double()
  r = bound_ratio(out, x.sum(0), sum_bound(T, x.abs().sum(0)))
  print(f'colsum_bf16 d={d}: error / bound = {r:.3f}')
  assert r <= 1.0, (d, r)


# --------------------------------------------------------------------------- limits and launch counts
def _captured_kernels(native, fn, *args):
  """Kernel nodes of a CUDA graph holding the one call fn(*args)."""
  g = torch.cuda.CUDAGraph(keep_graph=True)
  with torch.cuda.graph(g):
    fn(*args)
  return native.graph_node_counts(g.raw_cuda_graph())[0]


def test_bias_gradient_kernel_nodes(native):
  """The bias gradient is fused into the cast / loss kernel where it can be (d | 2048, ld <= 256) and takes one extra
  column-sum kernel elsewhere, counted on the kernel nodes of the captured call."""
  ctr = _counters([0, 10])
  for d in (64, 96, 256, 320, 2048):
    dH = torch.zeros(16, d, device=DEV)
    Z = torch.zeros(16, d, dtype=torch.bfloat16, device=DEV)
    n = _captured_kernels(native, native.relu_bwd_cast, dH, Z, ctr, 1, Z.clone(), torch.zeros(d, device=DEV), False,
                          1.0)
    assert n == (1 if 2048 % d == 0 else 2), (d, n)
    assert _captured_kernels(native, native.relu_bwd_cast, dH, Z, ctr, 1, Z.clone(), None, False, 1.0) == 1
  for ld in (64, 256, 320, 3008):
    lg = torch.zeros(16, ld, dtype=torch.bfloat16, device=DEV)
    y = torch.zeros(16, dtype=torch.int64, device=DEV)
    n = _captured_kernels(native, native.softmax_nll, lg, ld - 5, y, None, None, ctr, torch.zeros(1, device=DEV),
                          lg.clone(), None, torch.zeros(ld, device=DEV), False)
    assert n == (1 if ld <= 256 else 2), (ld, n)


@pytest.mark.parametrize('d', [1032, 2048])
def test_aggregation_kernels_reject_rows_wider_than_1024(native, d):
  ctr = _counters([0, 4])
  ell, ks, deg = [torch.zeros(4, dtype=torch.int32, device=DEV)], [1], torch.ones(4, dtype=torch.int32, device=DEV)
  src = torch.zeros(8, d, dtype=torch.bfloat16, device=DEV)
  A = torch.zeros(4, 2 * d, dtype=torch.bfloat16, device=DEV)
  dH = torch.zeros(8, d, device=DEV)
  calls = [lambda: native.sage_aggregate(None, None, src, d, ctr, 1, ell, ks, deg, A),
           lambda: native.sage_aggregate_block(None, None, src, d, ctr, 1, ell, ks, deg, A, 0),
           lambda: native.sage_scatter_block(A, d, 0, ctr, 1, ell, ks, deg, dH)]
  for call in calls:
    with pytest.raises(RuntimeError, match=r'multiple of 8 in \[8, 1024\]'):
      call()
  torch.cuda.synchronize()
  assert bool((A == 0).all()) and bool((dH == 0).all())
