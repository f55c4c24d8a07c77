"""Single-node multi-GPU R-GNN training on the on-disk IGBH dataset (the MLPerf-GNN workload).

Counterpart of the reference's examples/igbh/train_rgnn_multi_gpu.py:80-142,358: the dataset is built once in the
parent, shared with one spawned trainer per GPU through IPC handles, every rank trains on its split of the seeds,
evaluates inside the epoch (`--validation_frac_within_epoch`), stops at `--validation_acc`, logs MLPerf events and
writes resumable checkpoints (`--ckpt_steps`, `--ckpt_path`).  Two trainer back-ends:

  --trainer loader   hetero `NeighborLoader` (native grouped sampling arena on the GPU) + eager `models.RGNN`
                     (rgat / rsage / rgcn) + DistributedDataParallel -- the reference's structure
  --trainer engine   `models.HeteroGatEngine` (--model rgat, `--num_heads` heads) or `models.HeteroSageEngine`
                     (--model rsage): the whole step (sampling, aggregation, wgmma GEMMs, backward, Adam with the
                     gradient all-reduce fused in over NVLink peer memory) is one CUDA graph per rank; relations and
                     features are range-partitioned over the GPUs (no replica per rank).  rgcn has no engine.

  python examples/igbh/train_rgnn_multi_gpu.py --path /data/igbh --dataset_size tiny --model rgat --trainer engine

Without a GPU the loader back-end runs on gloo + CPU so the script stays testable anywhere.
"""
import argparse
import os
import os.path as osp
import socket
import sys
import time

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

sys.path.insert(0, osp.dirname(osp.dirname(osp.abspath(__file__))))
sys.path.insert(0, osp.dirname(osp.abspath(__file__)))
from common import glt  # noqa: E402
from dataset import IGBHeteroDataset  # noqa: E402
from graphlearn_for_pytorch_b200.models import RGNN  # noqa: E402
from mlperf_logging_utils import get_mlperf_logger  # noqa: E402


def evaluate(model, loader, device, max_batches=-1):
  model.eval()
  correct = total = 0
  with torch.no_grad():
    for i, b in enumerate(loader):
      if 0 <= max_batches <= i:
        break
      bs = b['paper'].batch_size
      x = {k: v.float() for k, v in b.x_dict.items()}
      out = model(x, b.edge_index_dict, b.num_sampled_nodes, b.num_sampled_edges)[:bs]
      correct += int((out.argmax(1) == b['paper'].y[:bs].to(device)).sum()); total += bs
  model.train()
  t = torch.tensor([correct, total], dtype=torch.float64, device=device)
  if dist.is_initialized():
    dist.all_reduce(t)
  return float(t[0] / t[1].clamp(min=1))


def run_loader(rank, world, ds, igbh_meta, a, port):
  cuda = torch.cuda.is_available()
  os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
  dist.init_process_group('nccl' if cuda else 'gloo', rank=rank, world_size=world)
  if cuda:
    torch.cuda.set_device(rank)
  device = torch.device('cuda', rank) if cuda else torch.device('cpu')
  glt.utils.seed_everything(a.random_seed)
  log = get_mlperf_logger()
  train_idx, val_idx, num_classes = igbh_meta
  fan = [int(v) for v in a.fan_out.split(',')]
  mine = train_idx.split((train_idx.numel() + world - 1) // world)[rank]
  vmine = val_idx.split((val_idx.numel() + world - 1) // world)[rank]
  loader = glt.loader.NeighborLoader(ds, fan, ('paper', mine), batch_size=a.train_batch_size, shuffle=True,
                                     device=device, seed=a.random_seed)
  val_loader = glt.loader.NeighborLoader(ds, fan, ('paper', vmine), batch_size=a.val_batch_size, device=device,
                                         seed=a.random_seed)
  first = next(iter(loader))
  in_dim = next(iter(first.x_dict.values())).shape[1]
  model = RGNN(list(first.edge_index_dict.keys()), in_dim, a.hidden_channels, num_classes, num_layers=len(fan),
               node_type='paper', model=a.model, heads=a.num_heads).to(device)
  start_epoch, step0 = 0, 0
  if a.ckpt_path and osp.exists(a.ckpt_path):
    ck = torch.load(a.ckpt_path, map_location=device, weights_only=False)
    model.load_state_dict(ck['model_state_dict'])
    start_epoch, step0 = ck.get('epoch', 0), ck.get('step', 0)
  model = torch.nn.parallel.DistributedDataParallel(model, device_ids=[rank] if cuda else None,
                                                    find_unused_parameters=True)
  opt = torch.optim.Adam(model.parameters(), lr=a.learning_rate)
  if a.ckpt_path and osp.exists(a.ckpt_path) and 'optimizer_state_dict' in ck:
    opt.load_state_dict(ck['optimizer_state_dict'])
  eval_every = max(1, int(len(loader) * a.validation_frac_within_epoch))
  if rank == 0:
    log.start('RUN')
  done = False
  for epoch in range(start_epoch, a.epochs):
    t0 = time.time()
    for i, b in enumerate(loader):
      if 0 <= a.max_steps <= i:
        break
      bs = b['paper'].batch_size
      x = {k: v.float() for k, v in b.x_dict.items()}
      out = model(x, b.edge_index_dict, b.num_sampled_nodes, b.num_sampled_edges)[:bs]
      loss = F.cross_entropy(out, b['paper'].y[:bs].to(device))
      opt.zero_grad(); loss.backward(); opt.step()
      step = step0 + epoch * len(loader) + i + 1
      if a.ckpt_steps > 0 and step % a.ckpt_steps == 0 and rank == 0:
        os.makedirs(a.ckpt_dir, exist_ok=True)
        torch.save({'model_state_dict': model.module.state_dict(), 'optimizer_state_dict': opt.state_dict(),
                    'epoch': epoch, 'step': step, 'loader': loader.state_dict()},
                   osp.join(a.ckpt_dir, f'model_step_{step}.ckpt'))
      if (i + 1) % eval_every == 0:
        acc = evaluate(model.module, val_loader, device, max_batches=a.val_batches)
        if rank == 0:
          log.event('EVAL_ACCURACY', acc, {'epoch_num': epoch + (i + 1) / len(loader)})
        if acc >= a.validation_acc:
          done = True
          break
    acc = evaluate(model.module, val_loader, device, max_batches=a.val_batches)
    if rank == 0:
      log.event('EVAL_ACCURACY', acc, {'epoch_num': epoch + 1})
      print(f'epoch {epoch}: loss {float(loss.detach()):.4f} val-acc {acc:.4f} ({time.time() - t0:.1f}s)', flush=True)
    if done or acc >= a.validation_acc:
      break
  if rank == 0:
    log.end('RUN', status='success' if acc >= a.validation_acc else 'aborted')
  dist.barrier()
  dist.destroy_process_group()


def run_engine(rank, world, igbh, a, port):
  """Device-resident back-end: relations and features range-partitioned over the GPUs, one CUDA graph per step."""
  from graphlearn_for_pytorch_b200.models import HeteroGatEngine, HeteroSageEngine
  from graphlearn_for_pytorch_b200.parallel import PartitionedFeature, partition_hetero_graph
  os.environ['MASTER_ADDR'], os.environ['MASTER_PORT'] = '127.0.0.1', str(port)
  torch.cuda.set_device(rank)
  device = torch.device('cuda', rank)
  if world > 1:
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=device)
  edge_dict, feat_dict, label, num_nodes, train_idx, val_idx, num_classes = igbh
  log = get_mlperf_logger()
  topos = {et: glt.data.Topology(ei.to(device), layout='CSC', num_nodes=num_nodes[et[2]]) for et, ei in edge_dict.items()}
  keep = []
  # --feat-format mxfp8: every type whose width is a multiple of 32 is stored as MXFP8 rows (about half the bytes)
  fmt = {nt: 'mxfp8' if a.feat_format == 'mxfp8' and f.shape[1] % 32 == 0 else 'bf16' for nt, f in feat_dict.items()}

  def shard(nt, rows):
    rows = rows.to(device).to(torch.bfloat16)
    return glt.data.quantize_mxfp8_chunked(rows) if fmt[nt] == 'mxfp8' else rows
  if world > 1:
    graphs, bounds, keep = partition_hetero_graph(topos, num_nodes, rank, world, device, 'in')
    stores = {nt: PartitionedFeature(shard(nt, feat_dict[nt][bounds[nt][rank]:bounds[nt][rank + 1]]),
                                     bounds[nt], device) for nt in num_nodes}
    tables = {nt: s.table for nt, s in stores.items()}
  else:
    graphs = {et: glt.data.Graph(t, 'CUDA', rank) for et, t in topos.items()}
    stores, tables = {}, {}
    for nt in num_nodes:
      rows = shard(nt, feat_dict[nt])
      ut = glt.data.UnifiedTensor(rank, rows.dtype)
      ut.append_shared_tensor(rows)
      stores[nt], tables[nt] = ut, ut._table()
  in_dim = {nt: (f.shape[1] + 7) // 8 * 8 for nt, f in feat_dict.items()}
  fan = [int(v) for v in a.fan_out.split(',')]
  common = dict(fanouts=fan, batch_size=a.train_batch_size, hidden=a.hidden_channels, num_classes=num_classes,
                edge_dir='in', lr=a.learning_rate, seed=a.random_seed, device=device, feature_format=fmt)
  if a.model == 'rgat':
    eng = HeteroGatEngine(graphs, tables, label.to(device), in_dim, num_nodes, 'paper', heads=a.num_heads, **common)
  else:
    eng = HeteroSageEngine(graphs, tables, label.to(device), in_dim, num_nodes, 'paper', **common)
  eng.warmup_and_capture(n_eager=1)
  mine = train_idx.split((train_idx.numel() + world - 1) // world)[rank]
  steps = mine.numel() // a.train_batch_size
  if world > 1:                               # every rank replays the same number of steps (one NVLink barrier each)
    t = torch.tensor([steps], device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    steps = int(t.item())
  if rank == 0:
    log.start('RUN')
  pinned = mine.pin_memory()
  for epoch in range(a.epochs):
    t0 = time.time()
    perm = torch.randperm(mine.numel(), generator=torch.Generator().manual_seed(a.random_seed + epoch))
    for i in range(steps if a.max_steps < 0 else min(steps, a.max_steps)):
      loss = eng.train_step(pinned[perm[i * a.train_batch_size:(i + 1) * a.train_batch_size]])
    torch.cuda.synchronize()
    if rank == 0:
      print(f'epoch {epoch}: loss {float(loss.item()):.4f} ({time.time() - t0:.2f}s, '
            f'{steps * a.train_batch_size * world / (time.time() - t0):.0f} seeds/s, dropped={eng.overflow_count()})',
            flush=True)
      # exact layer-wise full-neighbourhood inference (not collective: peer shards are read in place)
      pred = eng.inference().argmax(-1).cpu()
      acc = float((pred[val_idx] == label[val_idx]).float().mean())
      log.event('EVAL_ACCURACY', acc, {'epoch_num': epoch + 1})
      print(f'epoch {epoch}: val-acc {acc:.4f} (full-neighbourhood)', flush=True)
    if world > 1:
      dist.barrier()
  if rank == 0:
    log.end('RUN')
  eng.close()
  if world > 1:
    dist.barrier()
    dist.destroy_process_group()


def free_port():
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    return s.getsockname()[1]


if __name__ == '__main__':
  ap = argparse.ArgumentParser()
  ap.add_argument('--path', required=True)
  ap.add_argument('--dataset_size', default='tiny')
  ap.add_argument('--num_classes', type=int, default=19)
  ap.add_argument('--layout', default='COO', choices=['COO', 'CSC'])
  ap.add_argument('--use_fp16', action='store_true')
  ap.add_argument('--model', default='rgat', choices=['rgat', 'rsage', 'rgcn'])
  ap.add_argument('--trainer', default='loader', choices=['loader', 'engine'])
  ap.add_argument('--feat-format', default='bf16', choices=['bf16', 'mxfp8'],
                  help='--trainer engine: store the feature tables as MXFP8 rows (e4m3 + one scale per 32 elements)')
  ap.add_argument('--fan_out', default='15,10,5')
  ap.add_argument('--train_batch_size', type=int, default=1024)
  ap.add_argument('--val_batch_size', type=int, default=1024)
  ap.add_argument('--hidden_channels', type=int, default=512)
  ap.add_argument('--learning_rate', type=float, default=0.001)
  ap.add_argument('--epochs', type=int, default=2)
  ap.add_argument('--num_heads', type=int, default=4)
  ap.add_argument('--random_seed', type=int, default=42)
  ap.add_argument('--validation_frac_within_epoch', type=float, default=0.05)
  ap.add_argument('--validation_acc', type=float, default=0.72)
  ap.add_argument('--val_batches', type=int, default=-1)
  ap.add_argument('--max_steps', type=int, default=-1)
  ap.add_argument('--ckpt_steps', type=int, default=-1)
  ap.add_argument('--ckpt_dir', default='./ckpt')
  ap.add_argument('--ckpt_path', default=None)
  ap.add_argument('--world_size', type=int, default=0, help='0 = every visible GPU (2 CPU processes without a GPU)')
  a = ap.parse_args()
  cuda = torch.cuda.is_available()
  world = a.world_size or (torch.cuda.device_count() if cuda else 2)
  log = get_mlperf_logger()
  log.start('INIT')
  igbh = IGBHeteroDataset(a.path, a.dataset_size, layout=a.layout, use_fp16=a.use_fp16)
  assert igbh.train_idx is not None, 'run split_seeds.py first'
  port = free_port()
  if a.trainer == 'engine' and a.model == 'rgcn':
    ap.error('--trainer engine trains --model rgat (HeteroGatEngine) or rsage (HeteroSageEngine); '
             'rgcn runs with --trainer loader')
  if a.trainer == 'engine':
    assert cuda, 'the engine back-end needs a GPU'
    assert a.layout == 'COO', 'the engine builds its own CSC shards from the COO edge lists'
    payload = (igbh.edge_dict, {k: v.float() for k, v in igbh.feat_dict.items()}, igbh.label, igbh.num_nodes,
               igbh.train_idx, igbh.val_idx, igbh.num_classes)
    log.end('INIT')
    mp.spawn(run_engine, args=(world, payload, a, port), nprocs=world, join=True)
  else:
    ds = glt.data.Dataset(edge_dir='in')
    ds.init_graph(igbh.edge_dict, layout=a.layout, graph_mode='CUDA' if cuda else 'CPU', num_nodes=igbh.num_nodes)
    ds.init_node_features(igbh.feat_dict, with_gpu=cuda, split_ratio=1.0 if cuda else 0.0,
                          device_group_list=[glt.data.DeviceGroup(0, list(range(world)))] if cuda else None,
                          dtype=torch.float16 if a.use_fp16 else torch.float32)
    ds.init_node_labels({'paper': igbh.label})
    ds.share_ipc()
    igbh.train_idx.share_memory_(); igbh.val_idx.share_memory_()
    log.end('INIT')
    mp.spawn(run_loader, args=(world, ds, (igbh.train_idx, igbh.val_idx, igbh.num_classes), a, port), nprocs=world,
             join=True)
