"""BASELINE config 4: R-GNN (R-SAGE) on an IGBH-shaped heterogeneous graph (paper / author / institute / fos with
cites, written_by, affiliated_to, topic + reverse relations; reference examples/igbh/dataset.py:153-166,
examples/igbh/train_rgnn_multi_gpu.py:80-142: fanout 15,10,5, batch 1024, hidden 512, 3 layers, edge_dir 'in').

  python benchmarks/bench_hetero_rgnn.py --papers 1000000 --feat-dim 1024            # device-resident engine
  python benchmarks/bench_hetero_rgnn.py --model rgat                                 # R-GAT engine (HeteroGatEngine)
  python benchmarks/bench_hetero_rgnn.py --path loader                                # hetero NeighborSampler + eager RGNN
  python benchmarks/bench_hetero_rgnn.py --impl reference                             # unmodified reference, same box
  torchrun --nproc-per-node 8 --master-addr 127.0.0.1 benchmarks/bench_hetero_rgnn.py --papers 10000000

N GPUs (torchrun): every relation is range-partitioned over the GPUs by the node type its rows belong to and sampled
through peer-HBM reads; features are partitioned per node type and gathered in place over NVLink.  The engine path
is data-parallel: one engine per rank, the gradient all-reduce is a peer-HBM read fused into the Adam kernel.

Prints ONE JSON line on rank 0; device-timed (CUDA events), max over ranks.
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))

p = argparse.ArgumentParser()
p.add_argument('--impl', default='ours', choices=['ours', 'reference'])
p.add_argument('--path', default='engine', choices=['engine', 'loader'])
p.add_argument('--papers', type=int, default=200_000)
p.add_argument('--feat-dim', type=int, default=1024)
p.add_argument('--hidden', type=int, default=512)
p.add_argument('--classes', type=int, default=19)
p.add_argument('--batch', type=int, default=1024)
p.add_argument('--fanout', default='15,10,5')
p.add_argument('--steps', type=int, default=30)
p.add_argument('--warmup', type=int, default=3)
p.add_argument('--model', default='rsage', choices=['rsage', 'rgat'])
p.add_argument('--heads', type=int, default=4, help='attention heads of --model rgat')
p.add_argument('--rounds', type=int, default=1, help='timed windows of --steps steps (ms_per_step is their median)')
p.add_argument('--cap-limit', type=int, default=1 << 21)
p.add_argument('--feat-format', default='bf16', choices=['bf16', 'mxfp8'],
               help='engine path: feature storage of every node type (mxfp8 = e4m3 + UE8M0/32 block scales, '
                    'de-quantised inside the kernels that read the tables)')
p.add_argument('--device-gen', action='store_true', help='generate the graph / feature shards on the GPU')
args = p.parse_args()
rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
local = int(os.environ.get('LOCAL_RANK', 0))
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
if world > 1:
  os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
  dist.init_process_group('nccl', device_id=dev)
fan = [int(v) for v in args.fanout.split(',')]
METRIC = 'R-GNN igbh-shape training throughput (seed nodes/s, device-timed, max over ranks)'


def igbh_graph():
  from common import synthetic_igbh
  return synthetic_igbh(args.papers, args.papers // 2, max(args.papers // 400, 8), max(args.papers // 1000, 8),
                        feat_dim=args.feat_dim, num_classes=args.classes)


def igbh_graph_device():
  """Same schema generated ON THE DEVICE for large shapes (>= millions of papers, multi-GPU): every rank draws the
  same edge lists (same seed), features are generated per rank for its own row range only, labels are random
  (throughput runs).  -> (edges on device, feature shard generator, labels, sizes)."""
  n = {'paper': args.papers, 'author': args.papers // 2, 'institute': max(args.papers // 400, 8),
       'fos': max(args.papers // 1000, 8)}
  g = torch.Generator(device=dev)
  g.manual_seed(0)

  def rnd(ns, nd, e):
    return torch.stack([torch.randint(0, ns, (e,), device=dev, generator=g),
                        torch.randint(0, nd, (e,), device=dev, generator=g)])
  cites = rnd(n['paper'], n['paper'], n['paper'] * 8)
  written = rnd(n['paper'], n['author'], n['paper'] * 3)
  affil = rnd(n['author'], n['institute'], n['author'] * 2)
  topic = rnd(n['paper'], n['fos'], n['paper'] * 2)
  edges = {('paper', 'cites', 'paper'): torch.cat([cites, cites.flip(0)], 1),
           ('paper', 'written_by', 'author'): written, ('author', 'rev_written_by', 'paper'): written.flip(0),
           ('author', 'affiliated_to', 'institute'): affil, ('institute', 'rev_affiliated_to', 'author'): affil.flip(0),
           ('paper', 'topic', 'fos'): topic, ('fos', 'rev_topic', 'paper'): topic.flip(0)}

  def feat_shard(nt, lo, hi):
    gg = torch.Generator(device=dev)
    gg.manual_seed(100 + rank * 7 + sorted(n).index(nt))
    out = torch.empty(hi - lo, args.feat_dim, dtype=torch.bfloat16, device=dev)
    for b0 in range(0, hi - lo, 1 << 20):
      b1 = min(hi - lo, b0 + (1 << 20))
      out[b0:b1] = torch.randn(b1 - b0, args.feat_dim, device=dev, generator=gg).to(torch.bfloat16)
    return out
  labels = {'paper': torch.randint(0, args.classes, (n['paper'],), device=dev, generator=g)}
  return edges, feat_shard, labels, n


ROUND_MS = []


def timed(step):
  """Milliseconds of args.steps steps (the median of args.rounds windows; every window is in ROUND_MS)."""
  for i in range(args.warmup):
    step(i)
  torch.cuda.synchronize()
  if world > 1:
    dist.barrier()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  k = args.warmup
  for _ in range(max(args.rounds, 1)):
    e0.record()
    for i in range(args.steps):
      out = step(k)
      k += 1
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
      dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    ROUND_MS.append(float(ms.item()))
  return sorted(ROUND_MS)[len(ROUND_MS) // 2], out


def emit(ms, extra):
  if rank == 0:
    print(json.dumps(dict({'metric': METRIC, 'value': args.steps * args.batch * world / (ms / 1e3), 'unit': 'samples/s',
                           'n_gpus': world, 'ms_per_step': ms / args.steps, 'steps': args.steps, 'model': args.model,
                           'papers': args.papers, 'feat_dim': args.feat_dim, 'hidden': args.hidden, 'fanout': fan,
                           'batch': args.batch, 'impl': args.impl, 'feature_format': args.feat_format,
                           'ms_per_step_rounds': [m / args.steps for m in ROUND_MS]}, **extra)), flush=True)


def run_reference():
  """Unmodified reference (baseline/_ref): hetero Dataset + NeighborLoader + a plain-PyTorch R-SAGE with the same
  math as the engine (sum over relations of mean-aggregated neighbours + self, ReLU), fp32, HBM-resident."""
  sys.path.insert(0, os.path.join(ROOT, 'baseline', 'shims'))
  sys.path.insert(0, os.path.join(ROOT, 'baseline', '_ref'))
  import graphlearn_torch as rglt
  edges, feats, labels, sizes = igbh_graph()
  ds = rglt.data.Dataset(edge_dir='in')
  ds.init_graph(edge_index=edges, graph_mode='CUDA', device=local)
  ds.init_node_features(node_feature_data=feats, split_ratio=1.0, device_group_list=[rglt.data.DeviceGroup(0, [local])],
                        device=local)
  ds.init_node_labels(node_label_data=labels)
  pool = torch.randperm(args.papers, generator=torch.Generator().manual_seed(3))[rank::world]
  loader = rglt.loader.NeighborLoader(ds, fan, ('paper', pool), batch_size=args.batch, shuffle=True, drop_last=True,
                                      device=dev)
  ntypes = list(sizes)
  etypes = list(edges)

  class RSage(torch.nn.Module):
    def __init__(self):
      super().__init__()
      self.layers = torch.nn.ModuleList()
      for l in range(len(fan)):
        i = args.feat_dim if l == 0 else args.hidden
        o = args.hidden if l < len(fan) - 1 else args.classes
        self.layers.append(torch.nn.ModuleDict({
          'rel': torch.nn.ModuleDict({'__'.join(et): torch.nn.Linear(i, o, bias=False) for et in etypes}),
          'self': torch.nn.ModuleDict({t: torch.nn.Linear(i, o) for t in ntypes})}))

    def forward(self, x, ei):
      for l, layer in enumerate(self.layers):
        out = {t: layer['self'][t](h) for t, h in x.items()}
        for et, e in ei.items():
          s, d = et[0], et[2]
          if s not in x or d not in x or e.numel() == 0:
            continue
          agg = torch.zeros(x[d].shape[0], x[s].shape[1], device=dev).index_add_(0, e[1], x[s][e[0]])
          deg = torch.zeros(x[d].shape[0], device=dev).index_add_(0, e[1], torch.ones(e.shape[1], device=dev))
          out[d] = out[d] + layer['rel']['__'.join(et)](agg / deg.clamp(min=1).unsqueeze(1))
        x = {t: F.relu(h) for t, h in out.items()} if l < len(self.layers) - 1 else out
      return x['paper']

  model = RSage().to(dev)
  if world > 1:
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local])
  opt = torch.optim.Adam(model.parameters(), lr=1e-3)
  it = {'it': iter(loader)}

  def step(i):
    try:
      b = next(it['it'])
    except StopIteration:
      it['it'] = iter(loader)
      b = next(it['it'])
    x = {t: b[t].x for t in ntypes if b[t].x is not None}
    ei = {et: b[et].edge_index for et in etypes if b[et].edge_index is not None}
    bs = b['paper'].batch_size
    loss = F.cross_entropy(model(x, ei)[:bs], b['paper'].y[:bs])
    opt.zero_grad(); loss.backward(); opt.step()
    return loss

  ms, loss = timed(step)
  emit(ms, {'loss': float(loss.detach()), 'path': 'reference hetero NeighborLoader (graph_mode CUDA, split_ratio 1.0) '
            '+ plain-PyTorch R-SAGE fp32', 'dtype': 'fp32'})


def run_ours():
  import graphlearn_for_pytorch_b200 as glt
  from graphlearn_for_pytorch_b200.models import RGNN, HeteroGatEngine, HeteroSageEngine
  from graphlearn_for_pytorch_b200.parallel import PartitionedFeature, partition_hetero_graph
  from graphlearn_for_pytorch_b200.sampler import NeighborSampler, NodeSamplerInput
  device_gen = args.device_gen or world > 1 or args.papers >= 2_000_000
  if device_gen:
    edges, feat_shard, labels, sizes = igbh_graph_device()
  else:
    edges, feats, labels, sizes = igbh_graph()
    feat_shard = lambda nt, lo, hi: feats[nt][lo:hi].to(dev).to(torch.bfloat16)   # noqa: E731
  if args.feat_format == 'mxfp8':
    if args.path != 'engine':
      raise SystemExit('--feat-format mxfp8 is read by the engines (--path engine)')
    bf16_shard = feat_shard
    feat_shard = lambda nt, lo, hi: glt.data.quantize_mxfp8_chunked(bf16_shard(nt, lo, hi))   # noqa: E731
  edge_dir = 'in'
  topos = {}
  for et in list(edges):
    topos[et] = glt.data.Topology(edges.pop(et).to(dev), layout='CSC', num_nodes=sizes[et[2]])
  torch.cuda.empty_cache()
  if world > 1:
    graphs, bounds, keep = partition_hetero_graph(topos, sizes, rank, world, dev, edge_dir)
    fstore = {nt: PartitionedFeature(feat_shard(nt, bounds[nt][rank], bounds[nt][rank + 1]), bounds[nt], dev)
              for nt in sizes}
    tables = {nt: f.table for nt, f in fstore.items()}
  else:
    graphs = {et: glt.data.Graph(t, 'CUDA', local) for et, t in topos.items()}
    fstore, tables = {}, {}
    for nt in sizes:
      shard = feat_shard(nt, 0, sizes[nt])
      ut = glt.data.UnifiedTensor(local, shard.dtype)
      ut.append_shared_tensor(shard)
      fstore[nt], tables[nt] = ut, ut._table()
  del topos
  torch.cuda.empty_cache()
  y = labels['paper'].to(dev)
  pool = torch.randperm(args.papers, generator=torch.Generator().manual_seed(3))[rank::world].to(dev)

  def seeds_of(i):
    return pool[(i * args.batch) % (pool.numel() - args.batch):][:args.batch]

  if args.path == 'engine':
    kw = dict(fanouts=fan, batch_size=args.batch, hidden=args.hidden, num_classes=args.classes, edge_dir=edge_dir,
              lr=1e-3, seed=1, device=dev, use_cuda_graph=True, cap_limit=args.cap_limit, feature_format=args.feat_format)
    if args.model == 'rgat':
      eng = HeteroGatEngine(graphs, tables, y, args.feat_dim, sizes, 'paper', heads=args.heads, **kw)
      path = ('HeteroGatEngine: native grouped hetero sampling arena + per-relation wgmma projections + attention '
              'kernels, one CUDA graph')
    else:
      eng = HeteroSageEngine(graphs, tables, y, args.feat_dim, sizes, 'paper', **kw)
      path = 'HeteroSageEngine: native grouped hetero sampling arena + per-type wgmma GEMMs, one CUDA graph'
    eng.warmup_and_capture(n_eager=1)
    ms, loss = timed(lambda i: eng.train_step(seeds_of(i)))
    nodes, edges_n = eng.batch_sizes()
    emit(ms, {'loss': float(loss.item()), 'dtype': 'bf16', 'kernels_per_step': eng.kernels_per_step,
              'nodes_per_batch': {k: sum(v) for k, v in nodes.items()},
              'edges_per_batch': {'/'.join(k): sum(v) for k, v in edges_n.items()},
              'dropped_neighbours': eng.overflow_count(), 'path': path})
    eng.close()
    return
  sampler = NeighborSampler(graphs, fan, device=dev, edge_dir=edge_dir, seed=1)
  out0 = sampler.sample_from_nodes(NodeSamplerInput(torch.arange(args.batch, device=dev), 'paper'))
  model = RGNN(list(out0.row.keys()), args.feat_dim, args.hidden, args.classes, num_layers=len(fan), node_type='paper',
               model=args.model, heads=args.heads).to(dev).to(torch.bfloat16)
  if world > 1:
    model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local])
  opt = torch.optim.Adam(model.parameters(), lr=1e-3)

  def step(i):
    out = sampler.sample_from_nodes(NodeSamplerInput(seeds_of(i), 'paper'))
    x = {nt: fstore[nt][ids] for nt, ids in out.node.items()}
    ei = {et: torch.stack([out.row[et], out.col[et]]) for et in out.row}
    logits = model(x, ei, out.num_sampled_nodes, out.num_sampled_edges)[:out.batch['paper'].numel()].float()
    loss = F.cross_entropy(logits, y[out.batch['paper']])
    opt.zero_grad(); loss.backward(); opt.step()
    return loss

  ms, loss = timed(step)
  extra = {}
  if args.model == 'rgat':
    extra['model_note'] = ('the eager RGNN\'s last conv outputs the classes and it has no head Linear, unlike the '
                           'R-GAT engine (examples/igbh/rgnn.py): this arm compares cost, not identical math')
  emit(ms, dict({'loss': float(loss.detach()), 'dtype': 'bf16',
                 'path': 'hetero NeighborSampler (native arena, one sync per batch) + eager RGNN (bf16)'}, **extra))


if args.impl == 'reference':
  try:
    run_reference()
  except Exception as e:  # noqa: BLE001
    if rank == 0:
      print(json.dumps({'impl': 'reference', 'unavailable': f'{type(e).__name__}: {str(e)[:300]}'}))
else:
  run_ours()
if world > 1:
  dist.barrier()
  dist.destroy_process_group()
