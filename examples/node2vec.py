"""node2vec node embeddings on a homogeneous graph (the counterpart of PyG's examples/node2vec.py), trained by
`MetaPath2VecEngine` over the one relation ('n', 'to', 'n') with node2vec's p / q walks.

  python examples/node2vec.py --root <dir> --dataset ogbn-arxiv --p 1 --q 1     # an OGB download, made undirected
  python examples/node2vec.py --p 0.25 --q 4                                     # synthetic RMAT graph

One epoch visits every node once as a start (batches of --batch-size); then a logistic-regression probe is fitted on
the train split's embeddings and scored on the valid and test splits.  The synthetic graph's labels come from random
features, not from the graph, so there the probe scores near chance: run it on a real dataset to judge the embeddings.
"""
import argparse
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from common import add_dataset_args, glt, load_homo  # noqa: E402
from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine  # noqa: E402

REL = ('n', 'to', 'n')


def probe(z, y, split, epochs=200):
  """Multinomial logistic regression on z[train] (full-batch Adam) -> (valid accuracy, test accuracy)."""
  z = (z - z[split['train']].mean(0)) / (z[split['train']].std(0) + 1e-6)
  clf = torch.nn.Linear(z.shape[1], int(y.max()) + 1).to(z.device)
  opt = torch.optim.Adam(clf.parameters(), lr=0.01, weight_decay=1e-4)
  tr = split['train']
  for _ in range(epochs):
    opt.zero_grad()
    torch.nn.functional.cross_entropy(clf(z[tr]), y[tr]).backward()
    opt.step()
  with torch.no_grad():
    return tuple(float((clf(z[split[s]]).argmax(1) == y[split[s]]).float().mean()) for s in ('valid', 'test'))


def main(argv=None):
  p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  add_dataset_args(p)
  p.add_argument('--p', type=float, default=1.0, help='return parameter')
  p.add_argument('--q', type=float, default=1.0, help='in-out parameter')
  p.add_argument('--embedding-dim', type=int, default=128)
  p.add_argument('--walk-length', type=int, default=20)
  p.add_argument('--context-size', type=int, default=10)
  p.add_argument('--walks-per-node', type=int, default=10)
  p.add_argument('--num-negative-samples', type=int, default=1)
  p.add_argument('--batch-size', type=int, default=128)
  p.add_argument('--lr', type=float, default=0.01)
  p.add_argument('--epochs', type=int, default=1)
  p.add_argument('--seed', type=int, default=0)
  args = p.parse_args(argv)
  if not torch.cuda.is_available():
    sys.exit('node2vec.py trains on a CUDA GPU; none is visible')
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  ei, _, y, split, n = load_homo(args, undirected=True)
  graph = glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=n), 'CUDA', 0)
  eng = MetaPath2VecEngine({REL: graph}, {'n': n}, [REL], embedding_dim=args.embedding_dim,
                           walk_length=args.walk_length, context_size=args.context_size,
                           walks_per_node=args.walks_per_node, num_negative_samples=args.num_negative_samples,
                           batch_size=args.batch_size, lr=args.lr, seed=args.seed, device=dev, p=args.p, q=args.q)
  eng.warmup_and_capture()
  gen = torch.Generator(device=dev).manual_seed(args.seed)
  for epoch in range(args.epochs):
    t0 = time.time()
    perm = torch.randperm(n, device=dev, generator=gen)
    total = torch.zeros((), device=dev)
    steps = 0
    for i in range(0, n, args.batch_size):
      total += eng.train_step(perm[i:i + args.batch_size])
      steps += 1
    loss = float(total) / steps
    print(f'epoch {epoch}: loss {loss:.4f} ({steps} steps, {time.time() - t0:.2f} s)')
  splits = {k: v.to(dev) for k, v in split.items()}
  valid_acc, test_acc = probe(eng.embedding('n'), y.to(dev), splits)
  print(f'p={args.p} q={args.q}: valid accuracy {valid_acc:.4f}, test accuracy {test_acc:.4f}')
  return {'loss': loss, 'valid_acc': valid_acc, 'test_acc': test_acc}


if __name__ == '__main__':
  main()
