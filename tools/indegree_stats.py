"""In-batch in-degree distribution of the sampled sub-graph at bench shape (how skewed is the backward gather?)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench

args = bench.parse_args(['--no-pipeline'])
dev = torch.device('cuda', 0)
eng, pool = bench.build_ours(args, 0, 1, dev)
ar = eng.arena
for it in range(3):
  eng.seeds_dev.copy_(pool[it * 1024:(it + 1) * 1024].to(dev))
  eng._sample()
  torch.cuda.synchronize()
  c = ar.counters.cpu().tolist()
  cnt = ar.tr_cnt.cpu()
  for h in range(cnt.shape[0]):
    v = cnt[h, :c[h + 2]].float()
    q = torch.quantile(v, torch.tensor([0.5, 0.9, 0.99, 0.999]))
    print(f'batch {it} hops<= {h}: sources {v.numel()} edges {int(v.sum())} mean {v.mean():.2f} '
          f'p50/p90/p99/p99.9 {[int(x) for x in q]} max {int(v.max())} rows>32 {(v > 32).sum().item()} '
          f'edges in rows>32 {int(v[v > 32].sum())}')
