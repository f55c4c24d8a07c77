"""Multi-label node classification with GraphSAGE: T independent binary labels per node, scored by mean ROC-AUC.

  --mode engine   GraphSageMultiLabelEngine: the captured, pipelined GraphSAGE step with the fused sigmoid-BCE loss
                  kernel (needs an H100); validation / test ROC-AUC from exact full-neighbourhood `inference()`
  --mode trainer  GraphSageMultiLabelTrainer: sampler + eager GraphSAGE + autograd BCE, on the CPU

Without --root the graph is synthetic and each of --tasks tasks thresholds a random projection of the neighbour-mean
features.  With --root <dir> --dataset ogbn-proteins the real dataset is read from its OGB directory (species split,
112 tasks).  It has no node features, so a node's features are the mean of its incident edges' features, as in OGB's
own example, zero-padded to 64 columns.
"""
import argparse
import time

import torch

from common import add_dataset_args, glt
from graphlearn_for_pytorch_b200.models import (GraphSageMultiLabelEngine, GraphSageMultiLabelTrainer, multilabel_auc,
                                               multilabel_f1)
from graphlearn_for_pytorch_b200.utils.synthetic import multilabel_targets, rmat_edges

p = argparse.ArgumentParser()
p.add_argument('--mode', default='engine', choices=['engine', 'trainer'])
add_dataset_args(p, nodes=20_000, edges=400_000)
p.add_argument('--tasks', type=int, default=112, help='tasks of the synthetic dataset')
p.add_argument('--epochs', type=int, default=2)
p.add_argument('--batch', type=int, default=1024)
p.add_argument('--hidden', type=int, default=256)
p.add_argument('--fanouts', default='15,10,5')
p.add_argument('--dropout', type=float, default=0.0)
p.add_argument('--lr', type=float, default=3e-3)
args = p.parse_args()
fanouts = [int(f) for f in args.fanouts.split(',')]

if args.root:
  scheme = 'species' if args.dataset == 'ogbn-proteins' else None
  d = glt.utils.load_ogb_node_dataset(args.root, args.dataset, split_scheme=scheme)
  n = d['num_nodes']
  ei = torch.cat([d['edge_index'], d['edge_index'].flip(0)], 1)
  x = d['x']
  if x is None:                  # mean of the incident edges' features (each undirected edge counted at both ends)
    ea = torch.cat([d['edge_attr'], d['edge_attr']]).float()
    deg = torch.bincount(ei[1], minlength=n).clamp(min=1).float()
    x = torch.zeros(n, ea.shape[1]).index_add_(0, ei[1], ea) / deg.unsqueeze(1)
  y = d['y']
  split = d['split']
else:
  n = args.nodes
  ei = rmat_edges(n, args.edges // 2, seed=0)
  ei = torch.cat([ei, ei.flip(0)], 1)
  x = torch.randn(n, 64, generator=torch.Generator().manual_seed(1))
  y = multilabel_targets(ei, x, args.tasks, seed=2)
  perm = torch.randperm(n, generator=torch.Generator().manual_seed(0))
  n_tr, n_ev = n // 2, n // 10
  split = {'train': perm[:n_tr], 'valid': perm[n_tr:n_tr + n_ev], 'test': perm[n_tr + n_ev:n_tr + 2 * n_ev]}
in_dim = (x.shape[1] + 63) // 64 * 64
x = torch.nn.functional.pad(x.float(), (0, in_dim - x.shape[1]))
train_idx = split['train']
print(f'{n} nodes, {ei.shape[1]} edges, {y.shape[1]} tasks, positive rate {float(y.float().mean()):.3f}, '
      f'{train_idx.numel()} training nodes')

if args.mode == 'engine':
  if not torch.cuda.is_available():
    raise SystemExit('--mode engine needs a CUDA device; --mode trainer runs on the CPU')
  dev = torch.device('cuda', 0)
  topo = glt.data.Topology(ei.to(dev), layout='CSR', num_nodes=n)
  graph = glt.data.Graph(topo, 'CUDA', 0)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(x.to(dev, torch.bfloat16))
  model = GraphSageMultiLabelEngine(graph, ut._table(), y, in_dim=in_dim, num_nodes=n, fanouts=fanouts,
                                    batch_size=args.batch, hidden=args.hidden, lr=args.lr, device=dev,
                                    calibration_seeds=train_idx, pipeline=True, dropout=args.dropout)
  model.warmup_and_capture()
  seeds_src = train_idx.pin_memory()
else:
  dev = torch.device('cpu')
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CPU', directed=False, num_nodes=n)
  ds.init_node_features(x, with_gpu=False)
  model = GraphSageMultiLabelTrainer(ds.graph, ds.node_features, y, in_dim=in_dim, fanouts=fanouts,
                                     hidden=args.hidden, lr=args.lr, device=dev)
  seeds_src = train_idx

for epoch in range(args.epochs):
  t0 = time.time()
  perm = torch.randperm(train_idx.numel())
  losses = []
  for i in range(0, perm.numel() - args.batch + 1, args.batch):
    loss = model.train_step(seeds_src[perm[i:i + args.batch]])
    if loss is not None:
      losses.append(loss.detach().clone())     # the engine returns the same device scalar every step
  model.flush()
  mean_loss = float(torch.stack([l.reshape(()) for l in losses]).mean()) if losses else float('nan')
  print(f'epoch {epoch}: loss {mean_loss:.4f} time {time.time() - t0:.2f}s')

logits = model.inference().float().cpu()
ys = y.cpu()
for k in ('valid', 'test'):
  idx = split[k]
  print(f'{k} ROC-AUC {multilabel_auc(logits[idx], ys[idx]):.4f}  micro-F1 {multilabel_f1(logits[idx], ys[idx]):.4f}')
