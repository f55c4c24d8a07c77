"""LabelPropagation / CorrectAndSmooth on a 'CPU' graph (torch.sparse_csr_tensor matmuls) against float64
transcriptions of PyG's semantics written here over the COO edges (torch index_add), and the products example's --cs."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import CorrectAndSmooth, LabelPropagation

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- float64 reference (PyG's pseudo-code)
def ref_step_weights(n, rows, cols, norm):
  """Per-entry weight of A_norm for the CSR entries (rows[e] <- cols[e]); columns outside [0, n) weigh 0."""
  deg = torch.bincount(rows, minlength=n).double()
  inside = (cols >= 0) & (cols < n)
  c = torch.where(inside, cols, torch.zeros_like(cols))
  if norm == 'sym':
    d = torch.where(deg > 0, deg.pow(-0.5), torch.zeros_like(deg))
    w = d[rows] * d[c]
  else:
    w = torch.where(deg > 0, 1.0 / deg, torch.zeros_like(deg))[rows]
  return torch.where(inside, w, torch.zeros_like(w)), c


def ref_propagate(n, rows, cols, base, num_layers, alpha, norm, clamp=None, fixed=None):
  w, c = ref_step_weights(n, rows, cols, norm)
  base = base.double()
  out, res = base, (1 - alpha) * base
  for _ in range(num_layers):
    agg = torch.zeros_like(out).index_add_(0, rows, w.unsqueeze(1) * out[c])
    out = alpha * agg + res
    if clamp is not None:
      out = out.clamp(*clamp)
    if fixed is not None:
      out = torch.where(fixed.unsqueeze(1), base, out)
  return out


def ref_lp(n, rows, cols, y, num_layers, alpha, norm, mask=None):
  if y.dtype == torch.long:
    y = F.one_hot(y)
  y = y.double()
  out = y
  if mask is not None:
    out = torch.zeros_like(y)
    out[mask] = y[mask]
  return ref_propagate(n, rows, cols, out, num_layers, alpha, norm, clamp=(0., 1.))


def ref_correct(n, rows, cols, y_soft, y_true, mask, layers, alpha, autoscale, scale, norm):
  y_soft = y_soft.double()
  numel = int(mask.sum()) if mask.dtype == torch.bool else mask.numel()
  if y_true.dtype == torch.long:
    y_true = F.one_hot(y_true, y_soft.size(1))
  error = torch.zeros_like(y_soft)
  error[mask] = y_true.double() - y_soft[mask]
  if autoscale:
    sm = ref_propagate(n, rows, cols, error, layers, alpha, norm, clamp=(-1., 1.))
    sigma = error[mask].abs().sum() / numel
    s = sigma / sm.abs().sum(1, keepdim=True)
    s[s.isinf() | (s > 1000)] = 1.0
    return y_soft + s * sm
  fixed = torch.zeros(n, dtype=torch.bool, device=y_soft.device)
  fixed[mask] = True
  return y_soft + scale * ref_propagate(n, rows, cols, error, layers, alpha, norm, fixed=fixed)


def ref_smooth(n, rows, cols, y_soft, y_true, mask, layers, alpha, norm):
  if y_true.dtype == torch.long:
    y_true = F.one_hot(y_true, y_soft.size(1))
  y = y_soft.double().clone()
  y[mask] = y_true.double()
  return ref_propagate(n, rows, cols, y, layers, alpha, norm, clamp=(0., 1.))


# ---------------------------------------------------------------- graphs
def small_graph():
  """A directed graph with isolated nodes (7, 8), a duplicate edge (2 <- 0 twice) and self-loops (1, 4)."""
  ei = torch.tensor([[0, 0, 1, 1, 2, 2, 2, 3, 4, 4, 5, 6, 6],
                     [1, 3, 1, 2, 0, 0, 5, 6, 4, 0, 2, 5, 0]])
  return ei, 9


def rand_graph(n=60, e=300, seed=0):
  g = torch.Generator().manual_seed(seed)
  return torch.randint(0, n - 5, (2, e), generator=g), n     # the last 5 nodes are isolated


def cpu_graph(ei, n):
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=n)
  g = glt.data.Graph(topo, 'CPU')
  rows = torch.repeat_interleave(torch.arange(n), topo.indptr[1:] - topo.indptr[:-1])
  return g, rows, topo.indices.long()


def close(got, ref, tol=1e-4):
  assert got.dtype == torch.float32 and got.shape == ref.shape
  err = float((got.double() - ref).abs().max()) if ref.numel() else 0.0
  assert err <= tol * max(1.0, float(ref.abs().max())), err


# ---------------------------------------------------------------- tests
def test_orientation_rows_receive():
  """Row i receives from the columns of row i; the transposed graph gives a different answer here."""
  ei, n = small_graph()
  g, rows, cols = cpu_graph(ei, n)
  y = torch.tensor([0, 1, 2, 0, 1, 2, 0, 1, 2])
  got = LabelPropagation(3, 0.8)(y, g)
  close(got, ref_lp(n, rows, cols, y, 3, 0.8, 'sym'))
  gt, rt, ct = cpu_graph(ei.flip(0), n)
  assert (ref_lp(n, rt, ct, y, 3, 0.8, 'sym') - got.double()).abs().max() > 1e-2
  close(LabelPropagation(3, 0.8)(y, gt), ref_lp(n, rt, ct, y, 3, 0.8, 'sym'))


@pytest.mark.parametrize('norm', ['sym', 'row'])
@pytest.mark.parametrize('alpha', [0.0, 0.5, 0.8, 1.0])
@pytest.mark.parametrize('num_layers', [0, 50])
@pytest.mark.parametrize('graph', ['small', 'random'])
def test_label_propagation(norm, alpha, num_layers, graph):
  ei, n = small_graph() if graph == 'small' else rand_graph()
  g, rows, cols = cpu_graph(ei, n)
  gen = torch.Generator().manual_seed(1)
  y = torch.randint(0, 4, (n,), generator=gen)
  y[-1] = 3                                           # num_classes = y.max() + 1 = 4
  mask = torch.rand(n, generator=gen) < 0.5
  lp = LabelPropagation(num_layers, alpha, norm)
  close(lp(y, g), ref_lp(n, rows, cols, y, num_layers, alpha, norm))
  close(lp(y, g, mask), ref_lp(n, rows, cols, y, num_layers, alpha, norm, mask))
  idx = mask.nonzero().view(-1)
  close(lp(y, g, idx), ref_lp(n, rows, cols, y, num_layers, alpha, norm, mask))
  soft = torch.rand(n, 5, generator=gen)              # float rows
  close(lp(soft, g, idx), ref_lp(n, rows, cols, soft, num_layers, alpha, norm, mask))


@pytest.mark.parametrize('norm', ['sym', 'row'])
@pytest.mark.parametrize('index_mask', [False, True])
def test_correct_autoscale(norm, index_mask):
  """Autoscale with both rules: node 0 (masked, self-loop) has an error of 1e-6 per class, which node 1 receives,
  so their scale exceeds 1000; node 4 is isolated and unmasked, so its smoothed error is 0 and its scale inf."""
  ei = torch.tensor([[0, 1, 2, 3, 3, 5],
                     [0, 0, 2, 2, 1, 3]])
  n, C = 6, 3
  g, rows, cols = cpu_graph(ei, n)
  gen = torch.Generator().manual_seed(2)
  y_soft = torch.rand(n, C, generator=gen).softmax(-1)
  mask = torch.tensor([True, False, True, False, False, False])
  y_true = torch.tensor([1, 0])
  y_soft[0] = torch.tensor([-1e-6, 1 + 2e-6, -1e-6])
  m = mask.nonzero().view(-1) if index_mask else mask
  cs = CorrectAndSmooth(4, 0.9, 4, 0.8, autoscale=True)
  err = torch.zeros(n, C, dtype=torch.float64)
  err[mask] = F.one_hot(y_true, C).double() - y_soft[mask].double()
  sm = ref_propagate(n, rows, cols, err, 4, 0.9, norm, clamp=(-1., 1.))
  raw = err[mask].abs().sum() / 2 / sm.abs().sum(1)
  assert torch.isinf(raw[4]) and 1000 < raw[1] < math.inf and 1000 < raw[0] < math.inf
  got = cs.correct(y_soft, y_true, m, g, norm=norm)
  close(got, ref_correct(n, rows, cols, y_soft, y_true, mask, 4, 0.9, True, 1.0, norm))
  assert torch.equal(got[4], y_soft[4])               # scale 1 times a zero smoothed error


@pytest.mark.parametrize('norm', ['sym', 'row'])
def test_correct_fixed_scale_and_smooth(norm):
  ei, n = rand_graph(seed=3)
  g, rows, cols = cpu_graph(ei, n)
  C = 6
  gen = torch.Generator().manual_seed(4)
  y_soft = torch.rand(n, C, generator=gen).softmax(-1)
  mask = torch.rand(n, generator=gen) < 0.3
  y_true = torch.randint(0, C, (int(mask.sum()),), generator=gen)
  cs = CorrectAndSmooth(50, 1.0, 50, 0.8, autoscale=False, scale=20.0)
  corr = cs.correct(y_soft, y_true, mask, g, norm=norm)
  ref_c = ref_correct(n, rows, cols, y_soft, y_true, mask, 50, 1.0, False, 20.0, norm)
  close(corr, ref_c)
  close(cs.smooth(corr, y_true, mask, g, norm=norm),
        ref_smooth(n, rows, cols, corr, y_true, mask, 50, 0.8, norm))
  # float label rows of the masked nodes, index mask
  rows_true = F.one_hot(y_true, C).float()
  idx = mask.nonzero().view(-1)
  close(cs.smooth(y_soft, rows_true, idx, g, norm=norm),
        ref_smooth(n, rows, cols, y_soft, rows_true, mask, 50, 0.8, norm))


def test_products_recipe():
  """PyG's products recipe: correct with 'sym', then smooth with 'row'."""
  ei, n = rand_graph(n=80, e=500, seed=5)
  g, rows, cols = cpu_graph(ei, n)
  gen = torch.Generator().manual_seed(6)
  y_soft = torch.rand(n, 4, generator=gen).softmax(-1)
  idx = torch.randperm(n, generator=gen)[:20]
  y_true = torch.randint(0, 4, (20,), generator=gen)
  cs = CorrectAndSmooth(50, 1.0, 50, 0.8, autoscale=False, scale=20.0)
  got = cs.smooth(cs.correct(y_soft, y_true, idx, g, norm='sym'), y_true, idx, g, norm='row')
  ref = ref_correct(n, rows, cols, y_soft, y_true, idx, 50, 1.0, False, 20.0, 'sym')
  close(got, ref_smooth(n, rows, cols, ref.float(), y_true, idx, 50, 0.8, 'row'))


def test_argument_errors():
  ei, n = small_graph()
  g, _, _ = cpu_graph(ei, n)
  with pytest.raises(ValueError):
    LabelPropagation(3, 0.5, norm='col')
  with pytest.raises(ValueError):
    LabelPropagation(-1, 0.5)
  with pytest.raises(ValueError):
    LabelPropagation(3, math.nan)
  with pytest.raises(ValueError):
    LabelPropagation(3, 0.5)(torch.zeros(n, 2), g, torch.ones(n + 1, dtype=torch.bool))
  with pytest.raises(ValueError):
    LabelPropagation(3, 0.5)(torch.zeros(n + 2, 2), g)
  cs = CorrectAndSmooth(2, 0.5, 2, 0.5)
  with pytest.raises(ValueError):                     # y_true rows != masked rows
    cs.correct(torch.zeros(n, 2), torch.zeros(3, dtype=torch.long), torch.tensor([0, 1]), g)


def test_products_example_cs():
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  out = subprocess.run([sys.executable, 'examples/train_sage_products.py', '--mode', 'engine', '--cs', '--nodes', '3000',
                        '--edges', '30000', '--epochs', '1', '--batch', '256'],
                       cwd=ROOT, capture_output=True, text=True, timeout=600, env=env)
  assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
  lines = [l for l in out.stdout.splitlines() if 'test acc' in l]
  assert len(lines) == 2 and 'after C&S' in lines[1], out.stdout
