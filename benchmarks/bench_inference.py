#!/usr/bin/env python
"""Exact layer-wise full-neighbourhood inference (`GraphSageEngine.inference()`) on the products-shape graph.

  python benchmarks/bench_inference.py [--iters 5] [--train-steps 20] [bench.py options, e.g. --feat-format mxfp8]

The engine is built on one GPU by bench.py's `build_ours` (RMAT with the ogbn-products shape, 3 x SAGEConv, hidden
256) and trained for a few steps so that the weights are not the initial ones.  Then, in the same process:

* ours: device-timed `eng.inference()` (CUDA events, one warm-up call, then --iters timed calls), with per-layer
  times from events around each layer;
* torch: the same math from PyTorch building blocks -- `torch.sparse_csr_tensor` SpMM (fp32 mean weights 1/deg
  over the same CSR) + `torch.matmul` in bf16, the same aggregate-first / project-first order and bf16 rounding
  points -- timed in the same loop, alternating with ours;
* agreement: both arms' logits on 4096 random nodes (tolerance 5e-2, argmax agreement >= 99 %).

Derived numbers: edges/s (neighbour rows aggregated over all layers per second) and, per layer, the bytes the layer
must move at minimum (computed from shapes, `layer_bytes`) over its time.  The card name and power limit are read
in the same run.  One JSON line is printed and appended to --record.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (parse_args / build_ours of the headline benchmark)


def layer_bytes(eng, E, idx_bytes, feat_row_bytes):
  """Minimum HBM bytes per layer: CSR (indptr + column ids), one source row per edge, the self rows, the A chunk
  written and read back by the GEMM (aggregate-first) or the projection's input and P (project-first), the output."""
  N = eng._num_nodes
  csr = E * idx_bytes + (N + 1) * 8
  out = []
  for l in range(1, eng.L + 1):
    d, n = eng.dims_in[l - 1], eng.dims_out[l - 1]
    if eng._project_first(l):
      b = N * d * 2 + N * 2 * n * 2 + csr + E * n * 2 + N * n * 2 + N * n * 2
    else:
      row = feat_row_bytes if l == 1 else d * 2
      b = csr + E * row + N * row + 2 * N * 2 * d * 2 + N * n * 2
    out.append(b)
  return out


def torch_inference(eng, csr, feats):
  """The same layer-wise computation from PyTorch ops: fp32 CSR SpMM for the means, bf16 matmuls."""
  import torch
  H = feats
  for l in range(1, eng.L + 1):
    W, b = eng.W(l), eng.b(l)
    d, n = eng.dims_in[l - 1], eng.dims_out[l - 1]
    if eng._project_first(l):
      P = H @ torch.cat([W[:, :d], W[:, d:]], 0).t()
      Z = (torch.sparse.mm(csr, P[:, :n].float()) + P[:, n:].float() + b.float())
      del P
    else:
      mean = torch.sparse.mm(csr, H.float()).to(torch.bfloat16)
      Z = torch.addmm(b, torch.cat([mean, H], 1), W.t()).float()
      del mean
    if l < eng.L:
      Z = torch.relu(Z)
    H = Z.to(torch.bfloat16)
    del Z
  return H[:, :eng.C]


def card():
  import torch
  try:
    r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True, timeout=30)
    power = r.stdout.strip() or None
  except Exception as e:  # the number is still reported, without its power limit
    power = f'unavailable: {type(e).__name__}'
  return {'name': torch.cuda.get_device_name(0), 'power_limit': power}


def main():
  p = argparse.ArgumentParser(add_help=False)
  p.add_argument('--iters', type=int, default=5)
  p.add_argument('--train-steps', type=int, default=20)
  p.add_argument('--check-nodes', type=int, default=4096)
  p.add_argument('--no-torch', action='store_true', help='skip the torch arm (and with it the agreement check)')
  p.add_argument('--record', default=os.path.join(ROOT, 'profiles', 'bench_inference_h100.json'))
  own, rest = p.parse_known_args()
  args = bench.parse_args(rest + ['--gpus', '1'])
  import torch
  assert torch.cuda.is_available(), 'bench_inference measures on a GPU'
  assert own.iters >= 5
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  eng, pool = bench.build_ours(args, 0, 1, dev)
  seeds = bench.seed_batches(pool, own.train_steps, args.batch).to(dev)
  for i in range(own.train_steps):
    eng.train_step(seeds[i])
  eng.flush()
  torch.cuda.synchronize()
  _, ut, feats, shard = eng._keep
  indptr, indices = shard['indptr'], shard['indices']
  E = int(indices.numel())
  feat_row_bytes = int(feats.shape[1] * feats.element_size())

  # per-layer device time: events around every layer of the same call
  marks = []
  run_layer = eng._infer_layer

  def timed_layer(l, *a):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run_layer(l, *a)
    e1.record()
    marks.append((l, e0, e1))
  eng._infer_layer = timed_layer

  def time_call(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return out, e0.elapsed_time(e1)

  csr = None
  if not own.no_torch:
    assert args.feat_format == 'bf16', 'the torch arm reads bf16 features'
    deg = (indptr[1:] - indptr[:-1]).float()
    vals = (1.0 / deg.clamp(min=1)).repeat_interleave((indptr[1:] - indptr[:-1]))
    csr = torch.sparse_csr_tensor(indptr, indices.long(), vals, size=(eng._num_nodes, eng._num_nodes))
    del vals, deg

  ours_ms, torch_ms, layer_ms = [], [], {l: [] for l in range(1, eng.L + 1)}
  ours, ref = time_call(eng.inference)[0], None           # warm-up calls
  if csr is not None:
    ref = time_call(lambda: torch_inference(eng, csr, feats))[0]
  for _ in range(own.iters):
    del marks[:]
    ours, ms = time_call(eng.inference)
    ours_ms.append(ms)
    for l, e0, e1 in marks:
      layer_ms[l].append(e0.elapsed_time(e1))
    if csr is not None:
      ref, ms = time_call(lambda: torch_inference(eng, csr, feats))
      torch_ms.append(ms)
  eng._infer_layer = run_layer

  agreement = None
  if ref is not None:
    g = torch.Generator(device='cpu').manual_seed(args.seed + 11)
    ids = torch.randperm(eng._num_nodes, generator=g)[:own.check_nodes].to(dev)
    a, b = ours[ids].float(), ref[ids].float()
    argmax = float((a.argmax(1) == b.argmax(1)).float().mean())
    ok = bool(torch.allclose(a, b, rtol=5e-2, atol=5e-2)) and argmax >= 0.99
    agreement = {'nodes': int(ids.numel()), 'max_abs_diff': float((a - b).abs().max()), 'argmax_agree': argmax,
                 'tolerance': 'rtol 5e-2, atol 5e-2, argmax >= 0.99', 'pass': ok}

  med = statistics.median(ours_ms)
  lb = layer_bytes(eng, E, indices.element_size(), feat_row_bytes)
  layers = []
  for l in range(1, eng.L + 1):
    t = statistics.median(layer_ms[l])
    layers.append({'layer': l, 'order': 'project-first' if eng._project_first(l) else 'aggregate-first',
                   'dims': [eng.dims_in[l - 1], eng.dims_out[l - 1]], 'ms': t, 'bytes': lb[l - 1],
                   'GB_per_s': lb[l - 1] / (t * 1e-3) / 1e9})
  rec = {
    'metric': 'GraphSageEngine.inference() over all nodes (ms, device-timed, median)',
    'value': med, 'unit': 'ms', 'min_ms': min(ours_ms), 'max_ms': max(ours_ms), 'iters': own.iters,
    'edges_per_s': E * eng.L / (med * 1e-3), 'layers': layers, 'total_bytes': sum(lb),
    'graph': {'nodes': eng._num_nodes, 'directed_edges': E, 'column_id_bytes': indices.element_size()},
    'model': {'in_dim': eng.in_dim, 'hidden': eng.hidden, 'classes': eng.C, 'layers': eng.L,
              'train_steps_before': own.train_steps},
    'feature_format': args.feat_format,
    'torch': (None if csr is None else
              {'arm': 'torch.sparse_csr_tensor SpMM (fp32) + torch bf16 matmul, same order and rounding points',
               'median_ms': statistics.median(torch_ms), 'min_ms': min(torch_ms), 'max_ms': max(torch_ms)}),
    'agreement': agreement,
    'card': card(),
  }
  line = json.dumps(rec)
  print(line, flush=True)
  if own.record:
    os.makedirs(os.path.dirname(os.path.abspath(own.record)), exist_ok=True)
    with open(own.record, 'a') as f:
      f.write(line + '\n')
  if agreement is not None and not agreement['pass']:
    sys.exit(1)


if __name__ == '__main__':
  main()
