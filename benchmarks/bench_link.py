#!/usr/bin/env python
"""Link-prediction training step (`GraphSageLinkEngine`) against the eager link path, on the products-shape graph.

  python benchmarks/bench_link.py [--steps 30] [--warmup 5] [--rounds 3] [bench.py options, e.g. --fanout 15,10,5]

The graph and features come from bench.py's `build_ours` (RMAT with the ogbn-products shape, 2.45 M nodes,
123.7 M directed edges, 100-dim features padded to 128).  The workload is the link step of the reference's
unsupervised GraphSAGE examples: 3 x SAGEConv (128 -> 256 -> 256 -> 256), fanout 15/10/5, 1024 positive pairs per
step (uniform over the graph's edges) with k = 1 binary negatives each, mean BCE on the endpoint dot products, Adam.
Arms, in the same process, timed in alternating rounds:

* engine       GraphSageLinkEngine, CUDA graph, unpipelined;
* engine_pipe  the same, pipelined (sample b+1 || train b);
* eager        this library's LinkNeighborLoader on the GPU (NegativeSampling('binary', k)) + the eager GraphSAGE under
               bf16 autocast + torch.optim.Adam, same batch, fanout and ratio.

ms/step is device time (CUDA events around --steps steps after --warmup warm-up steps, synchronized at both ends),
the median over --rounds rounds.  The card name and power limit are read in the same run.  One JSON line is
printed and appended to --record.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402  (parse_args / build_ours of the headline benchmark)
from bench_inference import card  # noqa: E402


def edge_pairs(shard, n, generator):
  """n uniform edges [2, n] of a CSR shard (device tensors)."""
  import torch
  indptr, indices = shard['indptr'], shard['indices']
  e = torch.randint(0, indices.numel(), (n,), device=indptr.device, generator=generator)
  src = torch.searchsorted(indptr, e, right=True) - 1 + int(shard['row_begin'])
  return torch.stack([src, indices[e].long()])


def main():
  p = argparse.ArgumentParser(add_help=False)
  p.add_argument('--steps', type=int, default=30)
  p.add_argument('--warmup', type=int, default=5)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--neg-ratio', type=int, default=1)
  p.add_argument('--out-channels', type=int, default=256)
  p.add_argument('--no-eager', action='store_true', help='skip the eager arm')
  p.add_argument('--record', default=os.path.join(ROOT, 'profiles', 'bench_link_h100.json'))
  own, rest = p.parse_known_args()
  args = bench.parse_args(rest + ['--gpus', '1'])
  import torch
  import torch.nn.functional as F
  import graphlearn_for_pytorch_b200 as glt
  from graphlearn_for_pytorch_b200.models import GraphSAGE, GraphSageLinkEngine
  from graphlearn_for_pytorch_b200.sampler import NegativeSampling
  assert torch.cuda.is_available(), 'bench_link measures on a GPU'
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  node_eng, _ = bench.build_ours(args, 0, 1, dev)
  graph, ut, feats, shard = node_eng._keep
  in_dim = node_eng.in_dim
  del node_eng
  torch.cuda.empty_cache()
  N, B, k = args.nodes, args.batch, own.neg_ratio
  fanouts = [int(x) for x in args.fanout.split(',')]
  gen = torch.Generator(device=dev)
  gen.manual_seed(args.seed + 3)
  n_batches = max(own.steps, own.warmup) + 1
  batches = edge_pairs(shard, n_batches * B, gen).view(2, n_batches, B).permute(1, 0, 2).contiguous()

  arms, kernels, lib = {}, {}, {}
  for name, pipe in (('engine', False), ('engine_pipe', True)):
    eng = GraphSageLinkEngine(graph, ut._table(), in_dim, N, fanouts=fanouts, batch_size=B, hidden=args.hidden,
                              out_channels=own.out_channels, neg_ratio=k, lr=3e-3, seed=args.seed, device=dev,
                              use_fused=False if args.fused == 'off' else (True if args.fused == 'on' else 'auto'),
                              calibration_pairs=edge_pairs(shard, 64 * B, gen).cpu(), pipeline=pipe)
    eng.warmup_and_capture(n_eager=2)
    kernels[name], lib[name] = eng.kernels_per_step, eng.library_gemms_per_step

    def step(i, eng=eng):
      eng.train_step(batches[i % n_batches])
    arms[name] = step

  if not own.no_eager:
    ds = glt.data.Dataset(graph=graph)
    ds.init_node_features(feats.cpu(), with_gpu=True, split_ratio=1.0, device=0, dtype=torch.bfloat16)
    label_index = edge_pairs(shard, 100 * B, gen).cpu()
    loader = glt.loader.LinkNeighborLoader(ds, fanouts, edge_label_index=label_index, batch_size=B, shuffle=True,
                                           neg_sampling=NegativeSampling('binary', k), device=dev, seed=args.seed)
    torch.manual_seed(args.seed)
    model = GraphSAGE(in_dim, args.hidden, own.out_channels, len(fanouts)).to(dev)
    opt = torch.optim.Adam(model.parameters(), lr=3e-3)
    state = {'it': iter(loader)}

    def eager_step(i):
      try:
        b = next(state['it'])
      except StopIteration:
        state['it'] = iter(loader)
        b = next(state['it'])
      with torch.autocast('cuda', dtype=torch.bfloat16):
        h = model(b.x, b.edge_index, b.num_sampled_nodes, b.num_sampled_edges)
      eli = b.edge_label_index
      logit = (h[eli[0]].float() * h[eli[1]].float()).sum(-1)
      loss = F.binary_cross_entropy_with_logits(logit, b.edge_label.float())
      opt.zero_grad(set_to_none=True)
      loss.backward()
      opt.step()
    arms['eager'] = eager_step

  for step in arms.values():
    for i in range(own.warmup):
      step(i)
  torch.cuda.synchronize()
  times = {name: [] for name in arms}
  for r in range(own.rounds):
    for name, step in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      e0.record()
      for i in range(own.steps):
        step(r * own.steps + i)
      e1.record()
      torch.cuda.synchronize()
      times[name].append(e0.elapsed_time(e1) / own.steps)

  res = {}
  for name, t in times.items():
    med = statistics.median(t)
    res[name] = {'ms_per_step': med, 'min_ms': min(t), 'max_ms': max(t), 'positive_pairs_per_s': B / (med * 1e-3)}
    if name in kernels:
      res[name].update(kernels_per_step=kernels[name], library_gemms_per_step=lib[name])
  if 'eager' in res:
    res['eager']['api'] = ('LinkNeighborLoader(NegativeSampling binary) on the GPU + eager GraphSAGE (bf16 autocast) '
                           '+ torch Adam')
    res['eager']['library_gemms_per_step'] = 'all (cuBLAS under autocast)'
  rec = {
    'metric': 'GraphSAGE link-prediction training step (ms/step, device-timed, median over rounds)',
    'value': res['engine']['ms_per_step'], 'unit': 'ms',
    'arms': res,
    'config': {'nodes': N, 'directed_edges': int(shard['indices'].numel()), 'in_dim': in_dim, 'hidden': args.hidden,
               'out_channels': own.out_channels, 'layers': len(fanouts), 'fanout': fanouts, 'positive_pairs': B,
               'neg_ratio': k, 'seeds_per_step': 2 * (1 + k) * B, 'layer1': args.fused, 'steps': own.steps,
               'warmup': own.warmup, 'rounds': own.rounds},
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
