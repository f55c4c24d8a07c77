#!/usr/bin/env python
"""Correct & Smooth over the products-shape graph: the label-propagation kernel against torch.sparse_csr_tensor SpMM.

  python benchmarks/bench_label_prop.py [--nodes 2449029 --edges 123718280 --classes 47 --layers 50 --rounds 3]

The graph is the symmetric RMAT graph of ogbn-products' shape (bench.py's generator, int32 column ids, duplicate edges
kept).  Each arm runs the propagations of PyG's ogbn-products C&S recipe on the same inputs (a random softmax
prediction and an 8 % train mask, about the products train split): the correction (norm 'sym', alpha 1.0, masked rows
reset after every iteration) then the smoothing (norm 'row', alpha 0.8, clamp to [0, 1]), --layers iterations each.

* kernel: `models.label_prop.propagate` on a 'CUDA' graph (one csrc/cuda/label_prop.cu launch per iteration);
* torch:  `models.label_prop.propagate_sparse`, the same formulas as torch ops (what a 'CPU' graph runs), on CUDA
          tensors, over an fp32 `torch.sparse_csr_tensor` built once outside the timing.

Arms alternate for --rounds rounds after one warm-up call each, device-timed with CUDA events.  Per iteration: time,
the bytes an iteration must move at minimum (`iteration_bytes`, from shapes) and that over the time.  Agreement is the
max abs difference between the arms' smoothed outputs.  The card name and power limit are read in the same run.  One
JSON line is printed, and appended to --record when given.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_inference import card  # noqa: E402


def iteration_bytes(n, e, c, idx_bytes, norm):
  """Least HBM traffic of one iteration: the CSR (indptr, column ids), one neighbour row per edge (row pitch c rounded
  up to 4 floats), t_j per edge ('sym'), the base rows read, the output rows written, and s_i per row."""
  cp = (c + 3) // 4 * 4
  return ((n + 1) * 8 + e * idx_bytes + e * cp * 4 + (e * 4 if norm == 'sym' else 0) + 2 * n * cp * 4 + n * 4)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--nodes', type=int, default=2_449_029)
  p.add_argument('--edges', type=int, default=123_718_280, help='directed edges (both directions of each RMAT edge)')
  p.add_argument('--classes', type=int, default=47)
  p.add_argument('--layers', type=int, default=50)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--seed', type=int, default=0)
  p.add_argument('--record', default=None, help='append the JSON line to this file')
  a = p.parse_args()
  import torch
  import torch.nn.functional as F
  import graphlearn_for_pytorch_b200 as glt
  from graphlearn_for_pytorch_b200.models.label_prop import propagate, propagate_sparse, sparse_adj
  from graphlearn_for_pytorch_b200.utils.synthetic import rmat_csr_shard
  assert torch.cuda.is_available(), 'bench_label_prop measures on a GPU'
  assert a.rounds >= 2
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  N, C, L = a.nodes, a.classes, a.layers
  shard = rmat_csr_shard(N, a.edges // 2, 0, N, seed=a.seed, device=dev, undirected=True)
  graph = glt.data.Graph.from_shards([shard], 0)
  E = int(shard['indices'].numel())
  adj = {norm: sparse_adj(shard['indptr'], shard['indices'], norm) for norm in ('sym', 'row')}

  g = torch.Generator(device=dev).manual_seed(a.seed + 1)
  y_soft = torch.randn(N, C, device=dev, generator=g).softmax(-1)
  mask = torch.rand(N, device=dev, generator=g) < 0.08
  y_true = F.one_hot(torch.randint(0, C, (int(mask.sum()),), device=dev, generator=g), C).float()
  error = torch.zeros_like(y_soft)
  error[mask] = y_true - y_soft[mask]

  def recipe(run):
    """C&S's two propagations (the correction's result feeds the smoothing, as in CorrectAndSmooth)."""
    corrected = y_soft + 20.0 * run(error, L, 1.0, 'sym', None, mask)
    y = corrected.clone()
    y[mask] = y_true
    return run(y, L, 0.8, 'row', (0., 1.), None)

  arms = {
    'kernel': lambda x, l, al, norm, cl, fx: propagate(graph, x, l, al, norm, clamp=cl, fixed=fx),
    'torch': lambda x, l, al, norm, cl, fx: propagate_sparse(adj[norm], x, l, al, clamp=cl, fixed=fx),
  }

  def timed(name):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = recipe(arms[name])
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)

  outs, ms = {}, {k: [] for k in arms}
  for name in arms:                      # warm-up: module loads, cuSPARSE set-up, allocator
    timed(name)
  for _ in range(a.rounds):
    for name in arms:
      outs[name], t = timed(name)
      ms[name].append(t)
  diff = float((outs['kernel'] - outs['torch']).abs().max())

  iters = 2 * L
  idx_bytes = shard['indices'].element_size()
  bytes_per_iter = (iteration_bytes(N, E, C, idx_bytes, 'sym') + iteration_bytes(N, E, C, idx_bytes, 'row')) / 2
  res = {}
  for name in arms:
    med = statistics.median(ms[name])
    per = med / iters
    res[name] = {'recipe_ms_median': med, 'recipe_ms_all': ms[name], 'per_iteration_ms': per,
                 'GB_per_s': bytes_per_iter / (per * 1e-3) / 1e9}
  rec = {
    'metric': 'C&S products recipe (50 sym-correction + 50 row-smoothing iterations), ms per iteration, median',
    'value': res['kernel']['per_iteration_ms'], 'unit': 'ms', 'rounds': a.rounds,
    'kernel': res['kernel'], 'torch': res['torch'],
    'torch_arm': 'models.label_prop.propagate_sparse on CUDA tensors: torch.sparse_csr_tensor fp32 SpMM + element-wise',
    'speedup_vs_torch': res['torch']['per_iteration_ms'] / res['kernel']['per_iteration_ms'],
    'bytes_per_iteration_model': bytes_per_iter,
    'max_abs_diff_kernel_vs_torch': diff,
    'graph': {'nodes': N, 'directed_edges': E, 'column_id_bytes': idx_bytes, 'classes': C, 'train_fraction': 0.08},
    'card': card(),
  }
  line = json.dumps(rec)
  print(line, flush=True)
  if a.record:
    os.makedirs(os.path.dirname(os.path.abspath(a.record)), exist_ok=True)
    with open(a.record, 'a') as f:
      f.write(line + '\n')
  if not diff <= 1e-3:
    sys.exit(f'the arms disagree: max abs difference {diff}')


if __name__ == '__main__':
  main()
