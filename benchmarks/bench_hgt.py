"""HGT on an OGB-MAG-sized heterogeneous graph: the device-resident `HeteroHgtEngine` against the hetero
`NeighborLoader` + an eager PyTorch model of the same math, in one call.

The model is the reference's examples/hetero/train_hgt_mag.py: hidden 64, 2 heads, 2 layers, fanout [10, 10], batch
1024, Adam lr 0.01.  The graph is `synthetic_mag` at roughly ogbn-mag's node counts (736,389 papers, 1,134,649
authors, 8,740 institutions, 59,965 fields; cites / writes / affiliated_with / has_topic made undirected), with 128-wide
bf16 features for every type.

  python benchmarks/bench_hgt.py --rounds 5

Arms:
  engine  HeteroHgtEngine: sampling, the HGT layers, loss, backward and Adam as one CUDA graph
  eager   hetero NeighborLoader on the GPU + per-type Linear + ReLU, `models.HGTConv` H -> H twice, a Linear head,
          under bf16 autocast with torch.optim.Adam

ms_per_step is device-timed (CUDA events around --steps steps), the median over --rounds rounds.  Launches per step:
the kernel, memset and memcpy nodes of the engine's captured step; for the eager arm, the CUDA kernels (and memcpy / memset operations) torch.profiler records
over --steps steps, divided by --steps.  `--profile` prints the engine's per-kernel device times to stderr.  The card
name and power limit are read in the same run.  One JSON line is printed.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))

MAG = dict(num_papers=736_389, num_authors=1_134_649, num_insts=8_740, num_fields=59_965)


def card():
  try:
    r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True, timeout=30)
    power = r.stdout.strip() or None
  except Exception as e:  # the number is still reported, without its power limit
    power = f'unavailable: {type(e).__name__}'
  return {'name': torch.cuda.get_device_name(0), 'power_limit': power}


def timed(step, args):
  for i in range(args.warmup):
    step(i)
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  rounds, k = [], args.warmup
  for _ in range(max(args.rounds, 1)):
    e0.record()
    for _ in range(args.steps):
      out = step(k)
      k += 1
    e1.record()
    torch.cuda.synchronize()
    rounds.append(e0.elapsed_time(e1) / args.steps)
  return statistics.median(rounds), rounds, out


def profiled_launches(step, args, start):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for i in range(args.steps):
      step(start + i)
    torch.cuda.synchronize()
  n = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
  return n / args.steps, prof


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--scale', type=float, default=1.0, help='fraction of ogbn-mag node counts')
  p.add_argument('--feat-dim', type=int, default=128)
  p.add_argument('--classes', type=int, default=349)
  p.add_argument('--batch', type=int, default=1024)
  p.add_argument('--hidden', type=int, default=64)
  p.add_argument('--heads', type=int, default=2)
  p.add_argument('--steps', type=int, default=20)
  p.add_argument('--warmup', type=int, default=3)
  p.add_argument('--rounds', type=int, default=5)
  p.add_argument('--profile', action='store_true', help="print the engine's per-kernel device times to stderr")
  args = p.parse_args()
  import graphlearn_for_pytorch_b200 as glt
  from common import synthetic_mag
  from graphlearn_for_pytorch_b200.models import HGTConv, HeteroHgtEngine
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  fan = [10, 10]
  counts = {k: max(int(v * args.scale), 64) for k, v in MAG.items()}
  edges, feats, _, sizes = synthetic_mag(**counts, feat_dim=args.feat_dim, num_classes=args.classes)
  y = torch.randint(0, args.classes, (sizes['paper'],), generator=torch.Generator().manual_seed(5))
  pool = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(3))
  result = {'metric': 'HGT ogbn-mag-shape training step (device-timed ms/step, median over rounds)',
            'card': card(), 'nodes': sizes, 'edges': {'/'.join(k): int(v.shape[1]) for k, v in edges.items()},
            'feat_dim': args.feat_dim, 'hidden': args.hidden, 'heads': args.heads, 'layers': 2, 'fanout': fan,
            'batch': args.batch, 'classes': args.classes, 'steps': args.steps, 'rounds': args.rounds}

  # ---- engine
  graphs, tables, keep = {}, {}, []
  for et, ei in edges.items():
    graphs[et] = glt.data.Graph(glt.data.Topology(ei.to(dev), layout='CSC', num_nodes=sizes[et[2]]), 'CUDA', 0)
  for t, x in feats.items():
    ut = glt.data.UnifiedTensor(0, torch.bfloat16)
    ut.append_shared_tensor(x.to(dev).to(torch.bfloat16))
    keep.append(ut)
    tables[t] = ut._table()
  eng = HeteroHgtEngine(graphs, tables, y.to(dev), args.feat_dim, sizes, 'paper', fanouts=fan, batch_size=args.batch,
                        hidden=args.hidden, heads=args.heads, num_classes=args.classes, edge_dir='in', lr=0.01,
                        seed=1, device=dev)
  eng.warmup_and_capture(n_eager=1)
  pool_d = pool.to(dev)

  def seeds_of(i):
    return pool_d[(i * args.batch) % (pool_d.numel() - args.batch):][:args.batch]
  ms, rounds, loss = timed(lambda i: eng.train_step(seeds_of(i)), args)
  nodes, _ = eng.batch_sizes()
  result['engine'] = {'ms_per_step': ms, 'ms_per_step_rounds': rounds, 'launches_per_step': eng.kernels_per_step,
                      'loss': float(loss.item()), 'nodes_per_batch': {k: sum(v) for k, v in nodes.items()},
                      'dropped_neighbours': eng.overflow_count(),
                      'path': 'HeteroHgtEngine: grouped hetero sampling arena + wgmma GEMMs + hgt.cu attention, '
                              'one CUDA graph'}
  if args.profile:
    _, prof = profiled_launches(lambda i: eng.train_step(seeds_of(i)), args, 10_000)
    print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=30), file=sys.stderr)
  eng.close()
  del eng, graphs, tables, keep
  torch.cuda.empty_cache()

  # ---- eager: hetero NeighborLoader + the same math under bf16 autocast
  ds = glt.data.Dataset()
  ds.init_graph(edges, graph_mode='CUDA', num_nodes=sizes, device=0)
  ds.init_node_features(feats, split_ratio=1.0, with_gpu=True, device=0)
  ds.init_node_labels({'paper': y})
  loader = glt.loader.NeighborLoader(ds, fan, ('paper', pool), batch_size=args.batch, shuffle=True, drop_last=True,
                                     device=dev)
  names = list(sizes)

  class Model(torch.nn.Module):
    def __init__(self, etypes):
      super().__init__()
      self.inp = torch.nn.ModuleDict({t: torch.nn.Linear(args.feat_dim, args.hidden) for t in names})
      self.convs = torch.nn.ModuleList([HGTConv({t: args.hidden for t in names}, args.hidden, names, etypes,
                                                heads=args.heads) for _ in range(2)])
      self.head = torch.nn.Linear(args.hidden, args.classes)

    def forward(self, x, ei):
      x = {t: F.relu(self.inp[t](v)) for t, v in x.items()}
      for conv in self.convs:
        x = conv(x, ei)
      return self.head(x['paper'])

  it = {'it': iter(loader)}

  def next_batch():
    try:
      return next(it['it'])
    except StopIteration:
      it['it'] = iter(loader)
      return next(it['it'])
  first = next_batch()
  model = Model(list(first.edge_index_dict.keys())).to(dev)
  opt = torch.optim.Adam(model.parameters(), lr=0.01)

  def step(i):
    b = next_batch()
    bs = b['paper'].batch_size
    with torch.autocast('cuda', dtype=torch.bfloat16):
      out = model(b.x_dict, b.edge_index_dict)[:bs]
    loss = F.cross_entropy(out.float(), b['paper'].y[:bs].to(dev))
    opt.zero_grad(); loss.backward(); opt.step()
    return loss
  ms_e, rounds_e, loss_e = timed(step, args)
  launches, _ = profiled_launches(step, args, 0)
  result['eager'] = {'ms_per_step': ms_e, 'ms_per_step_rounds': rounds_e, 'launches_per_step': launches,
                     'loss': float(loss_e.detach()),
                     'path': 'hetero NeighborLoader (graph_mode CUDA, features in HBM) + per-type Linear/ReLU + '
                             'models.HGTConv x2 + Linear head, bf16 autocast, torch.optim.Adam'}
  result['engine_speedup'] = ms_e / result['engine']['ms_per_step']
  print(json.dumps(result), flush=True)


if __name__ == '__main__':
  main()
