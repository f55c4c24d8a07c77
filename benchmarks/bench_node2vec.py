"""node2vec on an ogbn-products-shape graph: `MetaPath2VecEngine` with node2vec's p / q walks against an eager
PyTorch arm of the same math, in one call.

The workload is PyG's node2vec recipe (embedding_dim 128, walk_length 40, context_size 20, walks_per_node 10,
num_negative_samples 1, batch_size 256, SparseAdam lr 0.01) on the undirected RMAT graph that bench.py trains
GraphSAGE on (2,449,029 nodes, 123.7 M directed edges at --scale 1), built the same way (rmat_csr_shard +
Graph.from_shards, column-sorted rows).

  python benchmarks/bench_node2vec.py --arm both

Arms (one JSON line each):
  engine  MetaPath2VecEngine at (p, q) = (1, 1), (0.25, 4) and (4, 0.25): (1, 1) is the uniform DeepWalk walk, so
          the other two show what the second-order rule costs on the same graph
  eager   at (0.25, 4) and (4, 0.25): biased walks in torch ops (propose for every walk still drawing, test edge
          membership with torch.searchsorted over the sorted keys row * N + col, repeat until every walk has accepted),
          then bench_metapath2vec's eager loss and torch.optim.SparseAdam

ms_per_step is device-timed (CUDA events around --steps steps after --warmup), the median over --rounds rounds;
pos_pairs_per_s counts (valid window, context) pairs.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))
sys.path.insert(0, os.path.join(ROOT, 'examples', 'hetero'))
sys.path.insert(0, os.path.join(ROOT, 'benchmarks'))

from bench_hgt import card  # noqa: E402
from bench_metapath2vec import EagerMetaPath2Vec, timed  # noqa: E402
import graphlearn_for_pytorch_b200 as glt  # noqa: E402
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_csr_shard  # noqa: E402

PRODUCTS = dict(nodes=2_449_029, edges=123_718_280)
HP = dict(embedding_dim=128, walk_length=40, context_size=20, walks_per_node=10, num_negative_samples=1,
          batch_size=256, lr=0.01)
REL = ('n', 'to', 'n')
PQ = [(1.0, 1.0), (0.25, 4.0), (4.0, 0.25)]
MAX_PROPOSALS = 4096


class EagerNode2Vec(EagerMetaPath2Vec):
  """EagerMetaPath2Vec with node2vec's biased walks (the engine's transition rule, rejection sampled in torch ops)."""

  def __init__(self, edges, sizes, dev, p, q, **hp):
    super().__init__(edges, sizes, [REL], dev, **hp)
    indptr, indices = self.csr[0]
    self.n = sizes['n']
    rows = torch.repeat_interleave(torch.arange(indptr.numel() - 1, device=dev), indptr[1:] - indptr[:-1])
    self.keys = rows * self.n + indices.long()                      # sorted: CSR rows with sorted columns
    hi = max(1.0, 1 / p, 1 / q)
    self.w_ret, self.w_in, self.w_out = 1 / p / hi, 1 / hi, 1 / q / hi

  def walks(self, starts):
    indptr, indices = self.csr[0]
    cur = starts.repeat_interleave(self.W)
    prev = torch.full_like(cur, -1)
    out = [cur]
    for s in range(1, self.L + 1):
      c = cur.clamp(min=0, max=indptr.numel() - 2)
      beg = indptr[c]
      deg = indptr[c + 1] - beg
      nxt = torch.full_like(cur, -1)
      todo = torch.nonzero((cur >= 0) & (deg > 0)).flatten()
      for k in range(MAX_PROPOSALS):
        if todo.numel() == 0:
          break
        d = deg[todo]
        x = indices[beg[todo] + (torch.rand(todo.numel(), device=self.dev) * d).long().clamp(max=d - 1)].long()
        if s == 1 or k == MAX_PROPOSALS - 1:
          acc = torch.ones_like(x, dtype=torch.bool)
        else:
          t = prev[todo]
          key = t * self.n + x
          pos = torch.searchsorted(self.keys, key).clamp(max=self.keys.numel() - 1)
          w = torch.where(x == t, self.w_ret, torch.where(self.keys[pos] == key, self.w_in, self.w_out))
          acc = torch.rand(x.numel(), device=self.dev) < w
        nxt[todo[acc]] = x[acc]
        todo = todo[~acc]
      nxt = torch.where(nxt < self.n, nxt, torch.full_like(nxt, -1))
      prev, cur = cur, nxt
      out.append(cur)
    return torch.stack(out, 1)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--arm', choices=['engine', 'eager', 'both'], default='both')
  p.add_argument('--steps', type=int, default=50)
  p.add_argument('--eager-steps', type=int, default=5)
  p.add_argument('--warmup', type=int, default=5)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--scale', type=float, default=1.0, help='fraction of the ogbn-products node and edge counts')
  args = p.parse_args()
  if not torch.cuda.is_available():
    sys.exit('bench_node2vec measures on a CUDA GPU; none is visible')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  N, E = (max(2, int(v * args.scale)) for v in (PRODUCTS['nodes'], PRODUCTS['edges']))
  shard = rmat_csr_shard(N, E // 2, 0, N, seed=0, device=dev, undirected=True)
  graph = glt.data.Graph.from_shards([shard], dev.index)
  C, B = HP['context_size'], HP['batch_size']
  gen = torch.Generator().manual_seed(0)
  batches = [torch.randint(0, N, (B,), generator=gen).to(dev) for _ in range(64)]
  info = card()

  def report(arm, pq, ms, windows, steps):
    print(json.dumps({'bench': 'node2vec', 'arm': arm, 'p': pq[0], 'q': pq[1], 'ms_per_step': round(ms, 4),
                      'pos_pairs_per_s': round(windows * (C - 1) / (ms / 1e3)),
                      'valid_windows_per_step': round(windows, 1), 'steps': steps, 'rounds': args.rounds,
                      'scale': args.scale, 'nodes': N, 'directed_edges': int(shard['indptr'][-1]),
                      'gpu': info['name'], 'power_limit': info['power_limit'], **HP}), flush=True)

  if args.arm in ('engine', 'both'):
    from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine
    for pq in PQ:
      eng = MetaPath2VecEngine({REL: graph}, {'n': N}, [REL], device=dev, p=pq[0], q=pq[1], **HP)
      eng.warmup_and_capture()

      def step(i):
        eng.train_step(batches[i % len(batches)])
        return eng.n_valid[0]
      ms, windows = timed(step, args)
      report('engine', pq, ms, windows, args.steps)
      del eng
      torch.cuda.empty_cache()
  if args.arm in ('eager', 'both'):
    ei = torch.stack([torch.repeat_interleave(torch.arange(N, device=dev), shard['indptr'][1:] - shard['indptr'][:-1]),
                      shard['indices'].long()])
    eargs = argparse.Namespace(**{**vars(args), 'steps': args.eager_steps})
    for pq in PQ[1:]:
      eager = EagerNode2Vec({REL: ei}, {'n': N}, dev, pq[0], pq[1], **HP)

      def step(i):
        return eager.step(batches[i % len(batches)])[1]
      ms, windows = timed(step, eargs)
      report('eager', pq, ms, windows, args.eager_steps)
      del eager
      torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
