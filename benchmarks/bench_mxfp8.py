"""What MXFP8 feature tables buy on one GPU: the layer-1 kernels and the heterogeneous training step, bf16 vs MXFP8.

  python benchmarks/bench_mxfp8.py [--out profiles/bench_mxfp8_h100.json]

Three parts, all in one process, arms alternating inside every round, every shape warmed up, device events:

  kernels  `sage_aggregate` (layer 1) on real sampled batches (fan-out 15,10,5, batch 1024) from a bf16 table and from
           its MXFP8 twin, at the products width (d = 128) and at the IGBH paper width (d = 1024), with the table in
           HBM and in pinned host memory; `gather_into` vs `gather_mxfp8_into` on 400 k rows.  Bytes are counted from
           shapes (`agg_bytes`, `gather_bytes`: rows read x row bytes + bf16 output) and reported as achieved bytes/s.
  steps    HeteroSageEngine and HeteroGatEngine at the IGBH shape of benchmarks/bench_hetero_rgnn.py, ms per step.
  tables   bytes per node type in both formats (from shapes).

Needs a CUDA GPU; the byte model of the tables is printed first, without one.  The card's name, power limit and
maximum SM clock are read with nvidia-smi and stored beside the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))

from graphlearn_for_pytorch_b200.data.quantize import mxfp8_row_bytes   # noqa: E402


def row_bytes(d, fmt):
  return mxfp8_row_bytes(d) if fmt == 'mxfp8' else 2 * d


def agg_bytes(rows_read, targets, d, fmt):
  """sage_aggregate: every valid ELL slot and every target's own row is one table row; the output is bf16 [mean | self]."""
  return rows_read * row_bytes(d, fmt) + targets * 2 * d * 2


def gather_bytes(n, d, fmt):
  return n * row_bytes(d, fmt) + n * d * 2


def igbh_sizes(papers):
  return {'paper': papers, 'author': papers // 2, 'institute': max(papers // 400, 8), 'fos': max(papers // 1000, 8)}


def table_bytes(papers, d):
  return {t: {f: n * row_bytes(d, f) for f in ('bf16', 'mxfp8')} for t, n in igbh_sizes(papers).items()}


def card():
  r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                     capture_output=True, text=True, timeout=60)
  name, power, clock = [v.strip() for v in r.stdout.strip().split(',')]
  return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


def alternate(arms, rounds, iters):
  """{arm: median over rounds of the ms per call}, arms taking turns inside each round; one warm-up call per arm."""
  for fn in arms.values():
    fn()
  torch.cuda.synchronize()
  ms = {k: [] for k in arms}
  for _ in range(rounds):
    for k, fn in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(iters):
        fn()
      e1.record()
      torch.cuda.synchronize()
      ms[k].append(e0.elapsed_time(e1) / iters)
  return {k: (statistics.median(v), v) for k, v in ms.items()}


def tables_of(x, glt, host):
  """{'bf16': handle, 'mxfp8': handle} over the same values (x is de-quantised MXFP8, so the two tables are twins)."""
  out, keep = {}, []
  for fmt, rows in (('bf16', x), ('mxfp8', glt.data.quantize_mxfp8_chunked(x))):
    ut = glt.data.UnifiedTensor(0, rows.dtype)
    if host:
      ut.append_cpu_tensor(rows.cpu())
    else:
      ut.append_shared_tensor(rows)
    keep.append(ut)
    out[fmt] = ut._table()
  return out, keep


def kernel_arm(args, glt, nat, dev, d, nodes):
  from graphlearn_for_pytorch_b200.models import GraphSageEngine
  from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges
  fan = [15, 10, 5]
  ei = rmat_edges(nodes, nodes * 8, seed=0, device=dev)
  graph = glt.data.Graph(glt.data.Topology(torch.cat([ei, ei.flip(0)], 1), layout='CSR', num_nodes=nodes), 'CUDA', 0)
  g = torch.Generator(device=dev).manual_seed(1)
  x = torch.cat([glt.data.dequantize_mxfp8(glt.data.quantize_mxfp8(torch.randn(min(nodes, b0 + (1 << 18)) - b0, d, device=dev, generator=g)), d)
                 .to(torch.bfloat16) for b0 in range(0, nodes, 1 << 18)])
  results = []
  hbm, keep = tables_of(x, glt, host=False)
  # the engine only provides the sampler arena and a real batch; the aggregation is launched directly on both tables
  eng = GraphSageEngine(graph, hbm['bf16'], torch.zeros(nodes, dtype=torch.int64), in_dim=d, num_nodes=nodes,
                        fanouts=fan, batch_size=args.batch, hidden=64, num_classes=8, device=dev, use_fused=False,
                        use_cuda_graph=False)
  ar = eng.arena
  eng._seeds[0].copy_(torch.randperm(nodes, device=dev)[:args.batch])
  eng._sample()
  torch.cuda.synchronize()
  T = int(ar.counters[len(fan)].item())
  rows_read = T + sum(int((ar.ell[h][:(int(ar.counters[h + 1]) - int(ar.counters[h])) * fan[h]] >= 0).sum()) for h in range(len(fan)))
  A = eng.A[1]
  for where in ('hbm', 'pinned_host'):
    tabs, keep2 = (hbm, None) if where == 'hbm' else tables_of(x, glt, host=True)
    arms = {fmt: (lambda t=tabs[fmt]: nat.sage_aggregate(t, ar.nodes, None, d, ar.counters, len(fan), list(ar.ell[:len(fan)]),
                                                         fan, ar.deg, A)) for fmt in ('bf16', 'mxfp8')}
    for fmt, (ms, all_ms) in alternate(arms, args.rounds, args.iters if where == 'hbm' else max(args.iters // 4, 2)).items():
      b = agg_bytes(rows_read, T, d, fmt)
      results.append({'kernel': 'sage_aggregate', 'd': d, 'table': where, 'format': fmt, 'targets': T,
                      'rows_read': rows_read, 'bytes': b, 'ms': round(ms, 4), 'ms_rounds': [round(v, 4) for v in all_ms],
                      'GB_per_s': round(b / ms / 1e6, 1)})
    del tabs, keep2
  n = 400_000
  ids = torch.randint(0, nodes, (n,), device=dev)
  out = torch.empty(n, d, dtype=torch.bfloat16, device=dev)
  arms = {'bf16': lambda: hbm['bf16'].gather_into(ids, None, None, out),
          'mxfp8': lambda: hbm['mxfp8'].gather_mxfp8_into(ids, None, None, out, d)}
  for fmt, (ms, all_ms) in alternate(arms, args.rounds, args.iters).items():
    b = gather_bytes(n, d, fmt)
    results.append({'kernel': 'gather_into' if fmt == 'bf16' else 'gather_mxfp8_into', 'd': d, 'table': 'hbm',
                    'format': fmt, 'rows': n, 'bytes': b, 'ms': round(ms, 4), 'ms_rounds': [round(v, 4) for v in all_ms],
                    'GB_per_s': round(b / ms / 1e6, 1)})
  del eng, hbm, keep
  torch.cuda.empty_cache()
  return results


def step_arm(args, glt, dev):
  from common import synthetic_igbh
  from graphlearn_for_pytorch_b200.models import HeteroGatEngine, HeteroSageEngine
  sizes = igbh_sizes(args.papers)
  edges, feats, labels, _ = synthetic_igbh(sizes['paper'], sizes['author'], sizes['institute'], sizes['fos'],
                                           feat_dim=args.feat_dim, num_classes=19)
  graphs = {et: glt.data.Graph(glt.data.Topology(ei.to(dev), layout='CSC', num_nodes=sizes[et[2]]), 'CUDA', 0)
            for et, ei in edges.items()}
  tabs, keep = {'bf16': {}, 'mxfp8': {}}, []
  for t, x in feats.items():
    q = glt.data.quantize_mxfp8_chunked(x.to(dev))
    both, k = tables_of(glt.data.dequantize_mxfp8(q, args.feat_dim).to(torch.bfloat16), glt, host=False)
    keep.append(k)
    for fmt in tabs:
      tabs[fmt][t] = both[fmt]
  y = labels['paper'].to(dev)
  pool = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(3)).to(dev)
  kw = dict(fanouts=[15, 10, 5], batch_size=args.batch, hidden=512, num_classes=19, edge_dir='in', lr=1e-3, seed=1,
            device=dev, use_cuda_graph=True)
  results = []
  for name, cls, extra in (('HeteroSageEngine', HeteroSageEngine, {}), ('HeteroGatEngine', HeteroGatEngine, {'heads': 4})):
    engs = {fmt: cls(graphs, tabs[fmt], y, args.feat_dim, sizes, 'paper', feature_format=fmt, **kw, **extra) for fmt in tabs}
    step = {fmt: 0 for fmt in tabs}

    def run(fmt):
      i = step[fmt] = step[fmt] + 1
      return engs[fmt].train_step(pool[(i * args.batch) % (pool.numel() - args.batch):][:args.batch])
    for e in engs.values():
      e.warmup_and_capture(n_eager=1)
    for fmt in tabs:
      for _ in range(3):
        run(fmt)
    for fmt, (ms, all_ms) in alternate({fmt: (lambda f=fmt: run(f)) for fmt in tabs}, args.rounds, args.steps).items():
      results.append({'engine': name, 'format': fmt, 'ms_per_step': round(ms, 4),
                      'ms_per_step_rounds': [round(v, 4) for v in all_ms], 'kernels_per_step': engs[fmt].kernels_per_step,
                      'loss': float(engs[fmt].loss.item())})
    for e in engs.values():
      e.close()
    del engs
    torch.cuda.empty_cache()
  return results


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--papers', type=int, default=200_000, help='IGBH-shaped graph of the step arm (authors = papers / 2)')
  p.add_argument('--feat-dim', type=int, default=1024)
  p.add_argument('--batch', type=int, default=1024)
  p.add_argument('--rounds', type=int, default=5)
  p.add_argument('--iters', type=int, default=20, help='kernel launches per timed window')
  p.add_argument('--steps', type=int, default=30, help='training steps per timed window')
  p.add_argument('--products-nodes', type=int, default=2_000_000)
  p.add_argument('--out', default=None, help='also write the JSON result to this file')
  args = p.parse_args()
  result = {'metric': 'MXFP8 vs bf16 feature tables: layer-1 kernels (ms, achieved GB/s) and heterogeneous step (ms)',
            'table_bytes': table_bytes(args.papers, args.feat_dim),
            'row_bytes': {str(d): {f: row_bytes(d, f) for f in ('bf16', 'mxfp8')} for d in (128, args.feat_dim)}}
  print(json.dumps({'table_bytes': result['table_bytes'], 'row_bytes': result['row_bytes']}), flush=True)
  if not torch.cuda.is_available():
    sys.exit('bench_mxfp8.py measures on a CUDA GPU and found none')
  import graphlearn_for_pytorch_b200 as glt
  nat = glt.ops.require_native()
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  result['card'] = card()
  result['kernels'] = kernel_arm(args, glt, nat, dev, 128, args.products_nodes) + \
      kernel_arm(args, glt, nat, dev, args.feat_dim, args.papers)
  result['steps'] = step_arm(args, glt, dev)
  line = json.dumps(result)
  print(line, flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      f.write(json.dumps(result, indent=1) + '\n')


if __name__ == '__main__':
  main()
