"""SEAL training throughput: SealEngine (one captured CUDA-graph step per batch) against the per-link eager path
(examples/seal_link_pred.py's extract: NeighborSampler.subgraph + drnl_node_labeling per link, then models.seal.DGCNN
under autograd and torch.optim.Adam), on a Cora-shape graph (2 hops, as the reference runs Cora) and an
ogbl-collab-shape graph (1 hop: collab's 2-hop subgraphs exceed the per-link node capacity).

  python benchmarks/bench_seal.py [--steps 50] [--eager-steps 2] [--out result.json]

Prints one JSON object (and writes it to --out): links/s of both arms per graph, the engine's launches per step and
truncated links, and the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import graphlearn_for_pytorch_b200 as glt                                      # noqa: E402
from graphlearn_for_pytorch_b200.models import DGCNN, SealEngine, drnl_node_labeling    # noqa: E402
from graphlearn_for_pytorch_b200.sampler import NeighborSampler, NodeSamplerInput     # noqa: E402
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges              # noqa: E402

B = 256
SHAPES = {'cora': dict(nodes=2_708, edges=5_278, hops=2), 'collab': dict(nodes=235_868, edges=1_285_465, hops=1)}


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                         text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(',')]
    return name, power
  except Exception:                                   # noqa: BLE001
    return torch.cuda.get_device_name(0), 'unknown'


def batches(ei, n, count, gen):
  out = []
  for _ in range(count):
    pos = ei[:, torch.randint(0, ei.shape[1], (B // 2,), generator=gen)]
    neg = torch.randint(0, n, (2, B // 2), generator=gen)
    out.append((torch.cat([pos, neg], 1), torch.cat([torch.ones(B // 2), torch.zeros(B // 2)])))
  return out


def bench_engine(g, ei, n, hops, steps, warmup, gen):
  cal = torch.cat([b[0] for b in batches(ei, n, 4, gen)], 1)
  eng = SealEngine(g, n, num_hops=hops, max_nodes=1024, hidden=32, num_layers=3, sort_k=0.6, batch_size=B, lr=1e-4,
                   calibration_links=cal)
  eng.warmup_and_capture()
  work = [(l.cuda(), y.cuda()) for l, y in batches(ei, n, steps + warmup, gen)]
  for l, y in work[:warmup]:
    eng.train_step(l, y)
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for l, y in work[warmup:]:
    eng.train_step(l, y)
  torch.cuda.synchronize()
  dt = time.perf_counter() - t0
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    eng._step()
    torch.cuda.synchronize()
  launches = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
  return dict(links_per_s=steps * B / dt, ms_per_step=1e3 * dt / steps, launches_per_step=launches,
              truncated_links=eng.truncated(), links_trained=(steps + warmup) * B, k=eng.k, max_z=eng.max_z,
              max_edges=eng.max_edges)


def bench_eager(g, ei, n, hops, steps, gen):
  dev = torch.device('cuda', 0)
  sampler = NeighborSampler(g, [-1] * hops, device=dev)
  model = DGCNN(num_labels=200, hidden=32, num_layers=3, k=30).to(dev)
  opt = torch.optim.Adam(model.parameters(), lr=1e-4)

  def step(links, y):
    zs, eis, bt, off = [], [], [], 0
    for i, (s, d) in enumerate(links.t().tolist()):
      out = sampler.subgraph(NodeSamplerInput(torch.tensor([s, d])))
      sub = torch.stack([out.row, out.col])
      m = out.metadata
      keep = ~(((sub[0] == m[0]) & (sub[1] == m[1])) | ((sub[0] == m[1]) & (sub[1] == m[0])))
      sub = sub[:, keep]
      k = out.node.numel()
      zs.append(drnl_node_labeling(sub, int(m[0]), int(m[1]), k, max_z=199))
      eis.append(sub + off)
      bt.append(torch.full((k,), i, device=dev))
      off += k
    logit = model(torch.cat(zs).to(dev), torch.cat(eis, 1).to(dev), torch.cat(bt), links.shape[1])
    loss = F.binary_cross_entropy_with_logits(logit, y.to(dev))
    opt.zero_grad()
    loss.backward()
    opt.step()

  work = batches(ei, n, steps + 1, gen)
  step(*work[0])
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for l, y in work[1:]:
    step(l, y)
  torch.cuda.synchronize()
  dt = time.perf_counter() - t0
  return dict(links_per_s=steps * B / dt, ms_per_step=1e3 * dt / steps)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--eager-steps', type=int, default=2)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_seal.py measures on a GPU; none is available')
  name, power = card()
  res = dict(bench='seal', batch_size=B, gpu=name, power_limit=power, graphs={})
  for tag, s in SHAPES.items():
    gen = torch.Generator().manual_seed(0)
    ei = rmat_edges(s['nodes'], s['edges'], seed=0)
    ei = ei[:, ei[0] != ei[1]]
    ei = torch.cat([ei, ei.flip(0)], 1)
    g = glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=s['nodes']), 'CUDA')
    g.lazy_init()
    res['graphs'][tag] = dict(nodes=s['nodes'], directed_edges=int(ei.shape[1]), num_hops=s['hops'],
                              engine=bench_engine(g, ei, s['nodes'], s['hops'], args.steps, args.warmup, gen),
                              eager=bench_eager(g, ei, s['nodes'], s['hops'], args.eager_steps, gen))
    r = res['graphs'][tag]
    r['speedup'] = r['engine']['links_per_s'] / r['eager']['links_per_s']
  line = json.dumps(res)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
