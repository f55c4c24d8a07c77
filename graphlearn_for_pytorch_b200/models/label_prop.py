"""Label propagation and Correct & Smooth (C&S; Huang et al., 2021) over the full graph, with PyG's semantics.

`LabelPropagation` and `CorrectAndSmooth` follow PyG's classes of the same names and mix the training labels back into
a node classifier's predictions over the graph.  Row i of the graph's CSR lists the nodes whose values flow into i (the
row the samplers and `inference()` read); duplicate edges count with their multiplicity and self-loops count as stored,
as PyG with `add_self_loops=False`.  With deg(v) the length of row v, two normalisations:

  'sym'  out_i = d_i * sum_{j in row(i)} d_j x_j,  d_v = deg(v)^-1/2   (PyG `gcn_norm(add_self_loops=False)`)
  'row'  out_i = 1 / deg(i) * sum_{j in row(i)} x_j                    (the D^-1 A of PyG's ogbn-products example)

A factor of a row with deg = 0 is 0, and column ids outside [0, num_rows) read as zero rows.

A `data.Graph` in mode 'CUDA' or 'ZERO_COPY' runs one sm_90a launch per iteration (csrc/cuda/label_prop.cu, up to 512
classes); a 'CPU' graph runs the same formulas as `torch.sparse_csr_tensor` matmuls.  Both compute in fp32.

Not supported: PyG's arbitrary `post_step` callables, edge weights (propagation is unweighted even when the Graph
carries weights) and heterogeneous graphs.
"""
import math
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from ..ops import require_native

NORMS = ('sym', 'row')


def _check_args(num_layers: int, alpha: float, norm: str):
  if norm not in NORMS:
    raise ValueError(f"norm must be one of {NORMS}, not {norm!r}")
  if int(num_layers) != num_layers or num_layers < 0:
    raise ValueError(f'num_layers must be an integer >= 0, not {num_layers}')
  if not math.isfinite(alpha):
    raise ValueError(f'alpha must be finite, not {alpha}')


def _device(graph) -> torch.device:
  return torch.device('cpu') if graph.mode == 'CPU' else torch.device('cuda', int(graph.device))


def _row_mask(mask: torch.Tensor, n: int, device) -> torch.Tensor:
  """`mask` (bool [n] or node ids) on `device`; raises ValueError on a bool mask of the wrong length."""
  mask = torch.as_tensor(mask).to(device)
  if mask.dtype == torch.bool:
    if mask.dim() != 1 or mask.numel() != n:
      raise ValueError(f'a bool mask needs one entry per node ({n}), got shape {tuple(mask.shape)}')
  elif mask.is_floating_point() or mask.dim() != 1:
    raise ValueError('mask must be a bool [num_nodes] tensor or a 1-D tensor of node ids')
  return mask


def sparse_adj(indptr: torch.Tensor, indices: torch.Tensor, norm: str) -> torch.Tensor:
  """A_norm as an fp32 `torch.sparse_csr_tensor` [n, n] on the CSR's device (columns outside [0, n) get weight 0)."""
  n = indptr.numel() - 1
  deg = indptr[1:] - indptr[:-1]
  degf = deg.to(torch.float32)
  col = indices.to(torch.int64)
  inside = (col >= 0) & (col < n)
  col = torch.where(inside, col, torch.zeros_like(col))
  if norm == 'sym':
    d = torch.where(deg > 0, degf.pow(-0.5), torch.zeros_like(degf))
    vals = torch.repeat_interleave(d, deg) * d[col]
  else:
    vals = torch.repeat_interleave(torch.where(deg > 0, 1.0 / degf, torch.zeros_like(degf)), deg)
  vals = torch.where(inside, vals, torch.zeros_like(vals))
  return torch.sparse_csr_tensor(indptr.to(torch.int64), col, vals, size=(n, n), check_invariants=False)


def propagate_sparse(adj: torch.Tensor, base: torch.Tensor, num_layers: int, alpha: float,
                     clamp: Optional[Tuple[float, float]] = None, fixed: Optional[torch.Tensor] = None) -> torch.Tensor:
  """The iteration of `propagate` as torch ops over `adj` (from `sparse_adj`), on base's device."""
  out = base
  res = (1 - alpha) * base
  for _ in range(num_layers):
    out = adj @ out
    out.mul_(alpha).add_(res)
    if clamp is not None:
      out.clamp_(*clamp)
    if fixed is not None:
      out = torch.where(fixed.unsqueeze(1), base, out)
  return out


def propagate(graph, base: torch.Tensor, num_layers: int, alpha: float, norm: str = 'sym',
              clamp: Optional[Tuple[float, float]] = None, fixed: Optional[torch.Tensor] = None) -> torch.Tensor:
  """num_layers iterations from out = base:
       out = post(alpha * A_norm out + (1 - alpha) * base),  post = clamp to `clamp`, then base on the rows of `fixed`
  base: fp32 [num_rows, C] on the graph's device; fixed: bool [num_rows] or None.  Returns fp32 [num_rows, C]."""
  _check_args(num_layers, alpha, norm)
  if base.dim() != 2 or base.size(0) != graph.row_count:
    raise ValueError(f'values need one row per graph node ({graph.row_count}), got shape {tuple(base.shape)}')
  if graph.mode == 'CPU':
    topo = graph.topo
    return propagate_sparse(sparse_adj(topo.indptr, topo.indices, norm), base, num_layers, alpha, clamp, fixed)
  n, c = base.shape
  cp = (c + 3) // 4 * 4
  padded = torch.zeros(n, cp, dtype=torch.float32, device=base.device)
  padded[:, :c] = base
  lo, hi = clamp if clamp is not None else (-math.inf, math.inf)
  out = require_native().label_prop(graph.graph_handler, padded, c, int(num_layers), float(alpha), norm, float(lo),
                                    float(hi), fixed)
  return out if cp == c else out[:, :c].contiguous()


class LabelPropagation(torch.nn.Module):
  """PyG's `LabelPropagation` (Zhu & Ghahramani, 2002) over a `data.Graph`:

    if y is int64 [N]: y = one_hot(y)            (num_classes = y.max() + 1)
    out = y;  if mask is not None: out = 0; out[mask] = y[mask]
    res = (1 - alpha) * out
    repeat num_layers: out = clamp(alpha * A_norm(out) + res, 0, 1)

  `norm` is 'sym' (PyG's, the default) or 'row' (see the module docstring).  `mask` is a bool [N] tensor or node ids.
  Returns fp32 [N, C] on the graph's device (the CPU for a 'CPU' graph).  PyG's `post_step` callable and edge weights
  are not supported.
  """

  def __init__(self, num_layers: int, alpha: float, norm: str = 'sym'):
    super().__init__()
    _check_args(num_layers, alpha, norm)
    self.num_layers, self.alpha, self.norm = int(num_layers), float(alpha), norm

  @torch.no_grad()
  def forward(self, y: torch.Tensor, graph, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    dev = _device(graph)
    y = y.to(dev)
    if y.dtype == torch.long and y.size(0) == y.numel():
      y = F.one_hot(y.view(-1))
    y = y.to(torch.float32)
    out = y
    if mask is not None:
      mask = _row_mask(mask, y.size(0), dev)
      out = torch.zeros_like(y)
      out[mask] = y[mask]
    return propagate(graph, out, self.num_layers, self.alpha, self.norm, clamp=(0., 1.))

  def extra_repr(self) -> str:
    return f'num_layers={self.num_layers}, alpha={self.alpha}, norm={self.norm!r}'


class CorrectAndSmooth(torch.nn.Module):
  """PyG's `CorrectAndSmooth` (Huang et al., 2021) over a `data.Graph`.

  `correct(y_soft, y_true, mask, graph, norm='sym')`: y_true holds the class ids of the masked rows, or float rows
  [numel, C].  error = 0; error[mask] = y_true - y_soft[mask]; then error is propagated num_correction_layers times
  with correction_alpha.
    autoscale=True:  each iteration clamps to [-1, 1]; sigma = |error[mask]|.sum() / numel, scale_i = sigma /
                     |smoothed_i|.sum(), scale_i = 1 where it is inf or > 1000; returns y_soft + scale * smoothed.
    autoscale=False: each iteration resets the masked rows to error; returns y_soft + self.scale * smoothed.
  `smooth(y_soft, y_true, mask, graph, norm='sym')`: y = y_soft; y[mask] = y_true; then y is propagated
  num_smoothing_layers times with smoothing_alpha, clamping to [0, 1].

  `mask` is a bool [N] tensor or node ids (numel = its number of True entries, or of ids).  Results are fp32 [N, C] on
  the graph's device.  PyG's ogbn-products recipe is `correct(..., norm='sym')` then `smooth(..., norm='row')` with 50
  layers each, alphas 1.0 / 0.8, autoscale=False and scale=20.  Edge weights are not supported.
  """

  def __init__(self, num_correction_layers: int, correction_alpha: float, num_smoothing_layers: int,
               smoothing_alpha: float, autoscale: bool = True, scale: float = 1.0):
    super().__init__()
    _check_args(num_correction_layers, correction_alpha, 'sym')
    _check_args(num_smoothing_layers, smoothing_alpha, 'sym')
    self.num_correction_layers, self.correction_alpha = int(num_correction_layers), float(correction_alpha)
    self.num_smoothing_layers, self.smoothing_alpha = int(num_smoothing_layers), float(smoothing_alpha)
    self.autoscale, self.scale = bool(autoscale), float(scale)

  @staticmethod
  def _inputs(graph, y_soft, y_true, mask):
    dev = _device(graph)
    y_soft = y_soft.to(dev, torch.float32)
    mask = _row_mask(mask, y_soft.size(0), dev)
    numel = int(mask.sum()) if mask.dtype == torch.bool else mask.numel()
    y_true = y_true.to(dev)
    if y_true.size(0) != numel:
      raise ValueError(f'y_true needs one row per masked node ({numel}), got {y_true.size(0)}')
    if y_true.dtype == torch.long and y_true.size(0) == y_true.numel():
      y_true = F.one_hot(y_true.view(-1), y_soft.size(-1))
    return y_soft, y_true.to(torch.float32), mask, numel

  @torch.no_grad()
  def correct(self, y_soft: torch.Tensor, y_true: torch.Tensor, mask: torch.Tensor, graph,
              norm: str = 'sym') -> torch.Tensor:
    y_soft, y_true, mask, numel = self._inputs(graph, y_soft, y_true, mask)
    error = torch.zeros_like(y_soft)
    error[mask] = y_true - y_soft[mask]
    if self.autoscale:
      smoothed = propagate(graph, error, self.num_correction_layers, self.correction_alpha, norm, clamp=(-1., 1.))
      sigma = error[mask].abs().sum() / numel
      scale = sigma / smoothed.abs().sum(dim=1, keepdim=True)
      scale[scale.isinf() | (scale > 1000)] = 1.0
      return y_soft + scale * smoothed
    fixed = torch.zeros(y_soft.size(0), dtype=torch.bool, device=y_soft.device)
    fixed[mask] = True
    smoothed = propagate(graph, error, self.num_correction_layers, self.correction_alpha, norm, fixed=fixed)
    return y_soft + self.scale * smoothed

  @torch.no_grad()
  def smooth(self, y_soft: torch.Tensor, y_true: torch.Tensor, mask: torch.Tensor, graph,
             norm: str = 'sym') -> torch.Tensor:
    y_soft, y_true, mask, _ = self._inputs(graph, y_soft, y_true, mask)
    y = y_soft.clone()
    y[mask] = y_true
    return propagate(graph, y, self.num_smoothing_layers, self.smoothing_alpha, norm, clamp=(0., 1.))

  def extra_repr(self) -> str:
    return (f'correct: num_layers={self.num_correction_layers}, alpha={self.correction_alpha}; '
            f'smooth: num_layers={self.num_smoothing_layers}, alpha={self.smoothing_alpha}; '
            f'autoscale={self.autoscale}, scale={self.scale}')
