#!/usr/bin/env python
"""Multi-label node-classification step (`GraphSageMultiLabelEngine`) against the 112-class node step and the eager
trainer, on the products-shape graph.

  python benchmarks/bench_multilabel.py [--steps 50] [--warmup 5] [--rounds 5] [--tasks 112] [bench.py options]

The graph and features come from bench.py's `build_ours` (RMAT with the ogbn-products shape, 2.45 M nodes,
123.7 M directed edges, 100-dim features padded to 128), with bench.py's defaults: 3 x SAGE (128 -> 256 -> 256 -> T),
fanout 15/10/5, batch 1024, calibrated arena, pipelined, unfused layer 1.  T = 112 is ogbn-proteins' task count.
Arms, in the same process, timed in alternating rounds on the same seed batches:

* node        GraphSageEngine with T classes (softmax cross-entropy), CUDA graphs;
* multilabel  GraphSageMultiLabelEngine with T tasks (sigmoid BCE, labels 30 % positive), same options;
* eager       GraphSageMultiLabelTrainer on the GPU: NeighborSampler + eager fp32 GraphSAGE + autograd BCE + Adam.

ms/step is device time (CUDA events around --steps steps after --warmup warm-up steps, synchronized at both ends),
the median over --rounds rounds.  `loss_kernel_us` is the in-situ device time of each engine's loss launch from
`profile_kernels` (an eager unpipelined step, events around each launch, mean of 10 steps), measured after the timed
rounds.  The card name and power limit are read in the same run.  One JSON line is printed and appended to --record.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402  (parse_args / build_ours / seed_batches of the headline benchmark)
from bench_inference import card  # noqa: E402


def main():
  p = argparse.ArgumentParser(add_help=False)
  p.add_argument('--steps', type=int, default=50)
  p.add_argument('--warmup', type=int, default=5)
  p.add_argument('--rounds', type=int, default=5)
  p.add_argument('--tasks', type=int, default=112)
  p.add_argument('--eager-steps', type=int, default=5, help='steps per round of the (slow) eager arm')
  p.add_argument('--no-eager', action='store_true', help='skip the eager arm')
  p.add_argument('--record', default=os.path.join(ROOT, 'profiles', 'bench_multilabel_h100.json'))
  own, rest = p.parse_known_args()
  args = bench.parse_args(rest + ['--gpus', '1', '--classes', str(own.tasks)])
  import torch
  from graphlearn_for_pytorch_b200.models import GraphSageMultiLabelEngine, GraphSageMultiLabelTrainer
  assert torch.cuda.is_available(), 'bench_multilabel measures on a GPU'
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  node_eng, pool = bench.build_ours(args, 0, 1, dev)
  graph, ut, feats, shard = node_eng._keep
  N, T, bs = args.nodes, own.tasks, args.batch
  fanouts = [int(x) for x in args.fanout.split(',')]
  g = torch.Generator(device=dev)
  g.manual_seed(args.seed + 5)
  labels = torch.rand(N, T, device=dev, generator=g) < 0.3
  ml_eng = GraphSageMultiLabelEngine(graph, ut._table(), labels, in_dim=node_eng.in_dim, num_nodes=N, fanouts=fanouts,
                                     batch_size=bs, hidden=args.hidden, lr=3e-3, seed=args.seed, device=dev,
                                     use_fused=False if args.no_fused or args.fused == 'off' else (
                                         True if args.fused == 'on' else 'auto'),
                                     use_cuda_graph=not args.no_graph,
                                     calibration_seeds=None if args.no_calibrate else pool,
                                     pipeline=not args.no_pipeline, feature_format=args.feat_format,
                                     dropout=args.dropout)
  engines = {'node': node_eng, 'multilabel': ml_eng}
  for eng in engines.values():
    eng.warmup_and_capture()
  n_batches = max(own.rounds * own.steps, own.warmup) + 1
  seeds = bench.seed_batches(pool, n_batches, bs).to(dev)

  arms = {name: (lambda i, eng=eng: eng.train_step(seeds[i % n_batches])) for name, eng in engines.items()}
  steps = {name: own.steps for name in arms}
  if not own.no_eager:
    tr = GraphSageMultiLabelTrainer(graph, feats, labels, in_dim=node_eng.in_dim, fanouts=fanouts, hidden=args.hidden,
                                    lr=3e-3, seed=args.seed, device=dev)
    arms['eager'] = lambda i: tr.train_step(seeds[i % n_batches])
    steps['eager'] = own.eager_steps

  for name, step in arms.items():
    for i in range(own.warmup):
      step(i)
  torch.cuda.synchronize()
  times = {name: [] for name in arms}
  for r in range(own.rounds):
    for name, step in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      e0.record()
      for i in range(steps[name]):
        step(own.warmup + r * steps[name] + i)
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / steps[name])
  for eng in engines.values():
    eng.flush()

  loss_us = {}
  for name, eng in engines.items():
    eng._graphs = []
    kt = eng.profile_kernels(seeds[:8], iters=10)
    loss_us[name] = {k: round(us, 2) for k, us in kt if k in ('softmax_nll', 'sigmoid_bce')}

  res = {}
  for name, t in times.items():
    med = statistics.median(t)
    res[name] = {'ms_per_step': med, 'min_ms': min(t), 'max_ms': max(t), 'steps_per_round': steps[name]}
    if name in engines:
      res[name].update(kernels_per_step=engines[name].kernels_per_step, loss_kernel_us=loss_us[name])
  res['node']['api'] = f'GraphSageEngine(num_classes={T}).train_step (softmax_nll)'
  res['multilabel']['api'] = f'GraphSageMultiLabelEngine({T} tasks).train_step (sigmoid_bce)'
  if 'eager' in res:
    res['eager']['api'] = 'GraphSageMultiLabelTrainer.train_step on the GPU (fp32 eager, autograd BCE, torch Adam)'
  rec = {
    'metric': 'GraphSAGE multi-label node-classification training step (ms/step, device-timed, median over rounds)',
    'value': res['multilabel']['ms_per_step'], 'unit': 'ms',
    'multilabel_over_node': res['multilabel']['ms_per_step'] / res['node']['ms_per_step'],
    'arms': res,
    'config': {'nodes': N, 'directed_edges': int(shard['indices'].numel()), 'in_dim': node_eng.in_dim,
               'hidden': args.hidden, 'tasks': T, 'fanout': fanouts, 'batch': bs, 'pipelined': not args.no_pipeline,
               'calibrated': not args.no_calibrate, 'layer1_fused': bool(node_eng.fused_ok[1]),
               'steps': own.steps, 'warmup': own.warmup, 'rounds': own.rounds},
    'card': card(),
  }
  line = json.dumps(rec)
  print(line, flush=True)
  if own.record:
    os.makedirs(os.path.dirname(os.path.abspath(own.record)), exist_ok=True)
    with open(own.record, 'a') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
