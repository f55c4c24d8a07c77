"""metapath2vec on an OGB-MAG-sized heterogeneous graph: `MetaPath2VecEngine` against an eager PyTorch arm of the
same math, in one call.

The workload is the one the reference's ogbn-mag HGT example takes its featureless-type vectors from (PyG
MetaPath2Vec with embedding_dim 128, walk_length 64, context_size 7, walks_per_node 5, num_negative_samples 5,
batch_size 128, SparseAdam lr 0.01) over the metapath author -> paper -> field_of_study -> paper -> author ->
institution -> author, on `synthetic_mag` at ogbn-mag's node counts (736,389 papers, 1,134,649 authors, 8,740
institutions, 59,965 fields).

  python benchmarks/bench_metapath2vec.py --arm both

Arms (one JSON line each):
  engine  MetaPath2VecEngine: walks, negatives, fused SGNS loss / gradient and sparse Adam as one CUDA graph
  eager   metapath walks in pure torch ops on the device CSRs, nn.Embedding(sparse=True) over the concatenated
          tables, the same loss and negatives (centre kept, context drawn per position type), torch.optim.SparseAdam

ms_per_step is device-timed (CUDA events around --steps steps after --warmup), the median over --rounds rounds;
pos_pairs_per_s counts (valid window, context) pairs, summed on the device over the timed steps.  The card name and
power limit are read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))
sys.path.insert(0, os.path.join(ROOT, 'examples', 'hetero'))
sys.path.insert(0, os.path.join(ROOT, 'benchmarks'))

from bench_hgt import MAG, card  # noqa: E402
from common import glt, synthetic_mag  # noqa: E402
from train_hgt_mag import MAG_METAPATH, M2V_ARGS  # noqa: E402

EPS = 1e-15


class EagerMetaPath2Vec:
  """The engine's step in eager torch ops (same walks distribution, loss, negatives and optimizer)."""

  def __init__(self, edges, sizes, metapath, dev, embedding_dim, walk_length, context_size, walks_per_node,
               num_negative_samples, lr, **_):
    self.mp, self.R, self.dev = metapath, len(metapath), dev
    self.L, self.C, self.W, self.K = walk_length, context_size, walks_per_node, num_negative_samples
    types = list(dict.fromkeys([metapath[0][0]] + [e[2] for e in metapath]))
    off, o = {}, 0
    for t in types:
      off[t] = o
      o += sizes[t]
    self.csr = []
    for e in metapath:
      topo = glt.data.Topology(edges[e], layout='CSR', num_nodes=max(sizes[e[0]], sizes[e[2]]))
      self.csr.append((topo.indptr.to(dev), topo.indices.to(dev)))
    slot_types = [metapath[0][0]] + [e[2] for e in metapath]
    slot = [0] + [(p - 1) % self.R + 1 for p in range(1, self.L + 1)]
    self.pos_off = torch.tensor([off[slot_types[s]] for s in slot], device=dev).unfold(0, self.C, 1)   # [J, C]
    self.pos_n = torch.tensor([sizes[slot_types[s]] for s in slot], device=dev).unfold(0, self.C, 1)
    self.emb = torch.nn.Embedding(o, embedding_dim, sparse=True).to(dev)
    self.opt = torch.optim.SparseAdam(self.emb.parameters(), lr=lr)

  def walks(self, starts):
    cur = starts.repeat_interleave(self.W)
    out = [cur]
    for s in range(1, self.L + 1):
      indptr, indices = self.csr[(s - 1) % self.R]
      ok = cur >= 0
      c = cur.clamp(min=0).clamp(max=indptr.numel() - 2)
      beg = indptr[c]
      deg = indptr[c + 1] - beg
      pick = (torch.rand(cur.numel(), device=self.dev) * deg).long().clamp(max=(deg - 1).clamp(min=0))
      nxt = indices[(beg + pick).clamp(max=max(indices.numel() - 1, 0))].long()
      cur = torch.where(ok & (deg > 0), nxt, torch.full_like(cur, -1))
      out.append(cur)
    return torch.stack(out, 1)

  def step(self, starts):
    wins = self.walks(starts).unfold(1, self.C, 1)                    # [n_walks, J, C]
    valid = (wins >= 0).all(-1)
    rows = (wins + self.pos_off)[valid]                                # [nv, C]
    nv = rows.shape[0]
    n = self.pos_n.expand(valid.shape[0], -1, -1)[valid][:, None, 1:]  # [nv, 1, C - 1]
    noff = self.pos_off.expand(valid.shape[0], -1, -1)[valid][:, None, 1:]
    neg = (torch.rand(nv, self.K, self.C - 1, device=self.dev) * n).long() + noff
    h = self.emb(rows[:, 0])
    s = (h[:, None, :] * self.emb(rows[:, 1:])).sum(-1)
    sn = (h[:, None, None, :] * self.emb(neg)).sum(-1)
    loss = -torch.log(torch.sigmoid(s) + EPS).mean() - torch.log(torch.sigmoid(-sn) + EPS).mean()
    self.opt.zero_grad()
    loss.backward()
    self.opt.step()
    return loss.detach(), valid.sum()


def timed(step, args):
  for i in range(args.warmup):
    step(i)
  torch.cuda.synchronize()
  ms, pairs = [], []
  for _ in range(args.rounds):
    acc = torch.zeros((), dtype=torch.int64, device='cuda')
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(args.steps):
      acc += step(i)
    b.record()
    torch.cuda.synchronize()
    ms.append(a.elapsed_time(b) / args.steps)
    pairs.append(int(acc) / args.steps)
  return statistics.median(ms), statistics.mean(pairs)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--arm', choices=['engine', 'eager', 'both'], default='both')
  p.add_argument('--steps', type=int, default=50)
  p.add_argument('--warmup', type=int, default=5)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--scale', type=float, default=1.0, help='fraction of the ogbn-mag node counts')
  args = p.parse_args()
  if not torch.cuda.is_available():
    sys.exit('bench_metapath2vec measures on a CUDA GPU; none is visible')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  edges, _, _, sizes = synthetic_mag(**{k: max(1, int(v * args.scale)) for k, v in MAG.items()}, feat_dim=8)
  hp = dict(M2V_ARGS)
  C, B = hp['context_size'], hp['batch_size']
  gen = torch.Generator().manual_seed(0)
  n_auth = sizes['author']
  batches = [torch.randint(0, n_auth, (B,), generator=gen).to(dev) for _ in range(64)]
  info = card()
  for arm in (['engine', 'eager'] if args.arm == 'both' else [args.arm]):
    if arm == 'engine':
      from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine
      graphs = {e: glt.data.Graph(glt.data.Topology(edges[e], layout='CSR',
                                                    num_nodes=max(sizes[e[0]], sizes[e[2]])), 'CUDA', 0)
                for e in MAG_METAPATH}
      eng = MetaPath2VecEngine(graphs, sizes, MAG_METAPATH, device=dev, **hp)
      eng.warmup_and_capture()

      def step(i):
        eng.train_step(batches[i % len(batches)])
        return eng.n_valid[0]
    else:
      eager = EagerMetaPath2Vec(edges, sizes, MAG_METAPATH, dev, **hp)

      def step(i):
        return eager.step(batches[i % len(batches)])[1]
    ms, windows = timed(step, args)
    print(json.dumps({'bench': 'metapath2vec', 'arm': arm, 'ms_per_step': round(ms, 4),
                      'pos_pairs_per_s': round(windows * (C - 1) / (ms / 1e3)),
                      'valid_windows_per_step': round(windows, 1), 'steps': args.steps, 'rounds': args.rounds,
                      'scale': args.scale, 'gpu': info['name'], 'power_limit': info['power_limit'], **hp}), flush=True)
    if arm == 'engine':
      del eng, graphs
    else:
      del eager
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
