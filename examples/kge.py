"""Knowledge-graph embeddings with KgeEngine (TransE, DistMult, ComplEx, RotatE) and filtered link-prediction metrics.

  python examples/kge.py --model rotate --root data/FB15k-237
  python examples/kge.py --model transe                 # synthetic_kg, no download

--root DIR holds train.txt / valid.txt / test.txt with one tab-separated (head, relation, tail) triple of names per
line, the layout of the FB15k-237 and WN18RR releases.  Prints the loss per epoch, then the filtered mean rank, MRR and
Hits@1/3/10 on valid and test, averaged over head and tail prediction.
"""
import argparse
import os
import sys
import time
from typing import Dict, List, Tuple

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def parse_args(argv=None) -> argparse.Namespace:
  p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  p.add_argument('--model', choices=['transe', 'distmult', 'complex', 'rotate'], default='transe')
  p.add_argument('--root', default=None, help='directory with train.txt / valid.txt / test.txt (default: synthetic)')
  p.add_argument('--hidden-channels', type=int, default=128)
  p.add_argument('--margin', type=float, default=None)
  p.add_argument('--p-norm', type=float, default=1.0)
  p.add_argument('--num-negatives', type=int, default=16)
  p.add_argument('--batch-size', type=int, default=1024)
  p.add_argument('--lr', type=float, default=0.01)
  p.add_argument('--epochs', type=int, default=20)
  p.add_argument('--seed', type=int, default=0)
  p.add_argument('--num-nodes', type=int, default=2000, help='synthetic entities')
  p.add_argument('--num-relations', type=int, default=8, help='synthetic relations')
  p.add_argument('--num-triples', type=int, default=50000, help='synthetic triples drawn')
  return p.parse_args(argv)


def read_kg(root: str) -> Tuple[Dict[str, torch.Tensor], Dict[str, int], Dict[str, int]]:
  """({'train' | 'valid' | 'test': int64 [3, m]}, entity ids, relation ids) of a directory of tab-separated triples.
  Ids are assigned in order of first appearance over train, valid, test."""
  ents: Dict[str, int] = {}
  rels: Dict[str, int] = {}
  splits = {}
  for split in ('train', 'valid', 'test'):
    rows: List[Tuple[int, int, int]] = []
    with open(os.path.join(root, f'{split}.txt'), encoding='utf-8') as f:
      for ln, line in enumerate(f, 1):
        line = line.rstrip('\n')
        if not line.strip():
          continue
        parts = line.split('\t')
        if len(parts) != 3:
          raise ValueError(f'{split}.txt:{ln}: expected head<TAB>relation<TAB>tail, got {line!r}')
        h, r, t = parts
        rows.append((ents.setdefault(h, len(ents)), rels.setdefault(r, len(rels)), ents.setdefault(t, len(ents))))
    splits[split] = torch.tensor(rows, dtype=torch.int64).reshape(-1, 3).t().contiguous()
  return splits, ents, rels


def main(argv=None):
  args = parse_args(argv)
  from graphlearn_for_pytorch_b200.models import KgeEngine, kge_filter
  from graphlearn_for_pytorch_b200.utils.synthetic import synthetic_kg
  if not torch.cuda.is_available():
    raise SystemExit('KgeEngine needs a CUDA device')
  dev = torch.device('cuda', 0)
  if args.root:
    splits, ents, rels = read_kg(args.root)
    N, R = len(ents), len(rels)
  else:
    N, R = args.num_nodes, args.num_relations
    tr, va, te = synthetic_kg(N, R, args.num_triples, seed=args.seed)
    splits = {'train': tr, 'valid': va, 'test': te}
  print(f'{N} entities, {R} relations, ' + ', '.join(f'{k} {v.size(1)}' for k, v in splits.items()))
  eng = KgeEngine(N, R, model=args.model, hidden_channels=args.hidden_channels, margin=args.margin,
                  p_norm=args.p_norm, num_negatives=args.num_negatives, batch_size=args.batch_size, lr=args.lr,
                  seed=args.seed, device=dev)
  eng.warmup_and_capture()
  flt = kge_filter(torch.cat(list(splits.values()), 1).to(dev), N, R)
  train = splits['train'].to(dev)
  g = torch.Generator(device=dev).manual_seed(args.seed)
  B = args.batch_size
  for epoch in range(1, args.epochs + 1):
    t0 = time.perf_counter()
    perm = torch.randperm(train.size(1), device=dev, generator=g)
    total = torch.zeros((), device=dev)
    steps = 0
    for b in range(0, train.size(1), B):
      total += eng.train_step(train[:, perm[b:b + B]].contiguous())
      steps += 1
    print(f'epoch {epoch:3d}  loss {float(total) / max(steps, 1):.4f}  {time.perf_counter() - t0:.2f} s')
  for split in ('valid', 'test'):
    h, r, t = splits[split].to(dev)
    mr, mrr, h1 = eng.test(h, r, t, k=1, filter=flt)
    h3 = eng.test(h, r, t, k=3, filter=flt)[2]
    h10 = eng.test(h, r, t, k=10, filter=flt)[2]
    print(f'{split}: filtered MR {mr:.1f}  MRR {mrr:.4f}  Hits@1 {h1:.4f}  Hits@3 {h3:.4f}  Hits@10 {h10:.4f}')


if __name__ == '__main__':
  main()
