"""Multi-GPU GraphSAGE on one NVSwitch box: graph + features range-partitioned over the GPUs,
sampling and layer-1 gather read peer HBM in-kernel, gradients all-reduced over NVLink inside the Adam kernel.

Counterpart of the reference's examples/multi_gpu/train_sage_ogbn_papers100m.py (which shares one
Dataset over spawned processes by IPC and shards a 15%-hot feature cache over NVLink groups).

  torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/multi_gpu/train_sage_p2p.py
"""
import argparse
import os
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from common import add_dataset_args, glt, load_homo  # noqa: E402
from graphlearn_for_pytorch_b200.models import GraphSageEngine  # noqa: E402
from graphlearn_for_pytorch_b200.parallel import (PartitionedFeature, PartitionedGraph, range_bounds,  # noqa: E402
                                                   shard_topology)

p = argparse.ArgumentParser()
add_dataset_args(p, nodes=500_000, edges=10_000_000)   # --root <dir> --dataset ogbn-papers100M reads the OGB files
p.add_argument('--steps', type=int, default=200)
args = p.parse_args()

rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
local = int(os.environ.get('LOCAL_RANK', 0))
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
if world > 1:
  dist.init_process_group('nccl', device_id=dev)
ei, x, y, split, args.nodes = load_homo(args, feat_dim=128, num_classes=16)
n_cls = int(y.max()) + 1
in_dim = (x.shape[1] + 63) // 64 * 64                 # the fused layer-1 kernel takes 64-column multiples
if in_dim != x.shape[1]:
  x = torch.nn.functional.pad(x, (0, in_dim - x.shape[1]))
y = y.clamp(min=0)                                    # papers100M: unlabelled nodes (never seeds) carry -1
topo = glt.data.Topology(ei.to(dev), layout='CSR', num_nodes=args.nodes)
bounds = range_bounds(args.nodes, world)
if world > 1:
  pg = PartitionedGraph(shard_topology(topo, bounds, rank, dev), bounds, dev)
  pf = PartitionedFeature(x[bounds[rank]:bounds[rank + 1]].to(dev).to(torch.bfloat16), bounds, dev)
  graph, table = pg.graph, pf.table
else:
  graph = glt.data.Graph(topo, 'CUDA', local)
  ut = glt.data.UnifiedTensor(local, torch.bfloat16); ut.append_shared_tensor(x.to(dev).to(torch.bfloat16))
  table = ut._table()
pool = split['train'][rank::world]
eng = GraphSageEngine(graph, table, y.to(dev), in_dim=in_dim, num_nodes=args.nodes, fanouts=[15, 10, 5],
                      batch_size=1024, hidden=256, num_classes=n_cls, device=dev, calibration_seeds=pool, pipeline=True)
eng.warmup_and_capture()
t0 = time.time()
for i in range(args.steps):
  idx = torch.randint(0, pool.numel(), (1024,))
  loss = eng.train_step(pool[idx].pin_memory())
  if rank == 0 and loss is not None and i % 50 == 0:
    print(f'step {i}: loss {float(loss.item()):.4f}')
eng.flush()
torch.cuda.synchronize()
if rank == 0:
  print(f'{args.steps * 1024 * world / (time.time() - t0):.0f} seeds/s on {world} GPU(s)')
test = split['test'][rank::world].to(dev)
stat = torch.zeros(2, device=dev)
for i in range(0, test.numel() - 1024 + 1, 1024):
  _, c, n = eng.evaluate_batch(test[i:i + 1024])
  stat += torch.tensor([c, n], device=dev, dtype=stat.dtype)
if world > 1:
  dist.all_reduce(stat)
if rank == 0:
  print(f'test acc {float(stat[0] / stat[1].clamp(min=1)):.4f} ({int(stat[1])} nodes)')
eng.close()
if world > 1:
  dist.barrier()
  dist.destroy_process_group()
