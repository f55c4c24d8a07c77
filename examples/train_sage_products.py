"""GraphSAGE on an ogbn-products-shaped graph, single GPU (or CPU).

Counterpart of the reference's examples/train_sage_ogbn_products.py and
train_sage_prod_with_trim.py.  Two paths:
  --mode loader   PyG-style: NeighborLoader -> eager GraphSAGE with per-layer trimming
  --mode engine   fused CUDA-graph engine (wgmma layer 1, hand-written backward); train / valid / test accuracy
                  from exact layer-wise full-neighbourhood inference (`inference()`), the protocol of the reference
                  example and of published ogbn-products accuracies
  --cs            (engine mode, also its CPU fallback) Correct & Smooth after inference: PyG's ogbn-products recipe
                  (`CorrectAndSmooth`, 50 + 50 layers, alphas 1.0 / 0.8, no autoscale, scale 20; sym-normalised
                  correction, row-normalised smoothing) on the softmax of the full-neighbourhood logits, with the
                  train split as the mask; accuracies before and after
"""
import argparse
import time

import torch
import torch.nn.functional as F

from common import add_dataset_args, glt, load_homo
from graphlearn_for_pytorch_b200.models import GraphSAGE, GraphSageEngine

p = argparse.ArgumentParser()
p.add_argument('--mode', default='loader', choices=['loader', 'engine'])
add_dataset_args(p)        # --root <dir with ogbn_products/> --dataset ogbn-products, or synthetic --nodes / --edges
p.add_argument('--epochs', type=int, default=2)
p.add_argument('--batch', type=int, default=1024)
p.add_argument('--dropout', type=float, default=0.5, help='hidden-layer dropout (engine mode and loader-mode model)')
p.add_argument('--split-ratio', type=float, default=0.2, help='fraction of (hot) feature rows kept in HBM')
p.add_argument('--cs', action='store_true', help='engine mode: Correct & Smooth the inference() predictions')
args = p.parse_args()

cuda = torch.cuda.is_available()
device = torch.device('cuda', 0) if cuda else torch.device('cpu')
ei, x, y, split, num_nodes = load_homo(args)
args.nodes = num_nodes
n_cls = int(y.max()) + 1
train_idx = split['train']


def correct_and_smooth(logits, graph):
  """PyG's ogbn-products C&S recipe on softmax(logits) over `graph`, the train split as the mask."""
  from graphlearn_for_pytorch_b200.models import CorrectAndSmooth
  t0 = time.time()
  y_soft = logits.float().softmax(-1)
  mask, y_train = train_idx.to(y_soft.device), y[train_idx].to(y_soft.device)
  cs = CorrectAndSmooth(50, 1.0, 50, 0.8, autoscale=False, scale=20.0)
  out = cs.correct(y_soft, y_train, mask, graph, norm='sym')
  out = cs.smooth(out, y_train, mask, graph, norm='row')
  if cuda:
    torch.cuda.synchronize()
  pred, yd = out.argmax(1), y.to(out.device)
  print('  '.join(f'{k} acc {float((pred[split[k].to(out.device)] == yd[split[k].to(out.device)]).float().mean()):.4f}'
                  for k in ('train', 'valid', 'test')) + f'  (after C&S, {time.time() - t0:.2f}s)')

if args.mode == 'loader':
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CUDA' if cuda else 'CPU', directed=False)
  ds.init_node_features(x, sort_func=glt.data.sort_by_in_degree, split_ratio=args.split_ratio, with_gpu=cuda)
  ds.init_node_labels(y)
  loader = glt.loader.NeighborLoader(ds, [15, 10, 5], train_idx, batch_size=args.batch, shuffle=True,
                                     drop_last=True, device=device)
  model = GraphSAGE(x.shape[1], 256, n_cls, num_layers=3, dropout=args.dropout).to(device)
  opt = torch.optim.Adam(model.parameters(), lr=3e-3)

  @torch.no_grad()
  def accuracy(idx):
    # sampled 15/10/5 neighbourhoods over the evaluation split: a quick estimate that changes from call to call.
    # The reference example scores with exact full-neighbourhood inference (SAGE.inference); --mode engine does that.
    model.eval()
    hit = tot_n = 0
    for b in glt.loader.NeighborLoader(ds, [15, 10, 5], idx, batch_size=args.batch, shuffle=False, device=device):
      out = model(b.x, b.edge_index, b.num_sampled_nodes, b.num_sampled_edges)[:b.batch_size]
      hit += int((out.argmax(1) == b.y[:b.batch_size].to(device)).sum()); tot_n += b.batch_size
    model.train()
    return hit / max(tot_n, 1)

  for epoch in range(args.epochs):
    t0, tot, correct, seen = time.time(), 0.0, 0, 0
    for b in loader:
      out = model(b.x, b.edge_index, b.num_sampled_nodes, b.num_sampled_edges)[:b.batch_size]
      tgt = b.y[:b.batch_size].to(device)
      loss = F.cross_entropy(out, tgt)
      opt.zero_grad(); loss.backward(); opt.step()
      tot += float(loss.detach()); correct += int((out.argmax(1) == tgt).sum()); seen += b.batch_size
    print(f'epoch {epoch}: loss {tot / len(loader):.4f} acc {correct / seen:.4f} time {time.time() - t0:.2f}s')
  print(f"valid acc {accuracy(split['valid']):.4f}  test acc {accuracy(split['test']):.4f}")
elif not cuda:
  # no GPU: the same step-level loop on the device-agnostic trainer (sampler + eager GraphSAGE + torch Adam)
  from graphlearn_for_pytorch_b200.models import GraphSageTrainer
  print('no CUDA device: --mode engine falls back to GraphSageTrainer (same train_step/evaluate_batch API)')
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CPU', directed=False)
  ds.init_node_features(x, with_gpu=False)
  tr = GraphSageTrainer(ds.graph, ds.node_features, y, in_dim=x.shape[1], fanouts=[15, 10, 5], hidden=256,
                        num_classes=n_cls, device=device)
  for epoch in range(args.epochs):
    t0 = time.time()
    perm = torch.randperm(train_idx.numel())
    losses = [float(tr.train_step(train_idx[perm[i:i + args.batch]]))
              for i in range(0, perm.numel() - args.batch + 1, args.batch)]
    print(f'epoch {epoch}: loss {sum(losses) / max(len(losses), 1):.4f} time {time.time() - t0:.2f}s')
  logits = tr.inference()
  pred = logits.argmax(1)
  print('  '.join(f'{k} acc {float((pred[split[k]] == y[split[k]]).float().mean()):.4f}'
                  for k in ('train', 'valid', 'test')))
  if args.cs:
    correct_and_smooth(logits, ds.graph)
else:
  in_dim = (x.shape[1] + 63) // 64 * 64
  feats = torch.zeros(args.nodes, in_dim, dtype=torch.bfloat16, device=device)
  feats[:, :x.shape[1]] = x.to(device).to(torch.bfloat16)
  topo = glt.data.Topology(ei.to(device), layout='CSR', num_nodes=args.nodes)
  graph = glt.data.Graph(topo, 'CUDA', 0)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16); ut.append_shared_tensor(feats)
  eng = GraphSageEngine(graph, ut._table(), y.to(device), in_dim=in_dim, num_nodes=args.nodes, fanouts=[15, 10, 5],
                        batch_size=args.batch, hidden=256, num_classes=n_cls, device=device,
                        calibration_seeds=train_idx, pipeline=True, dropout=args.dropout)
  eng.warmup_and_capture()
  pinned = train_idx.pin_memory()
  for epoch in range(args.epochs):
    t0 = time.time()
    perm = torch.randperm(train_idx.numel())
    losses = []
    for i in range(0, perm.numel() - args.batch + 1, args.batch):
      loss = eng.train_step(pinned[perm[i:i + args.batch]])
      if loss is not None and (i // args.batch) % 20 == 0:
        losses.append(float(loss.item()))
    eng.flush()
    torch.cuda.synchronize()
    l, c, n = eng.evaluate_batch(train_idx[:args.batch].to(device))
    print(f'epoch {epoch}: loss {sum(losses) / max(len(losses), 1):.4f} eval-acc {c / n:.4f} '
          f'time {time.time() - t0:.2f}s ({perm.numel() / (time.time() - t0):.0f} seeds/s)')
  t0 = time.time()
  logits = eng.inference()
  pred = logits.argmax(1)
  torch.cuda.synchronize()
  y_dev = y.to(device)
  accs = {k: float((pred[split[k].to(device)] == y_dev[split[k].to(device)]).float().mean())
          for k in ('train', 'valid', 'test')}
  print('  '.join(f'{k} acc {a:.4f}' for k, a in accs.items()) + f'  (full-neighbourhood inference, '
        f'{time.time() - t0:.2f}s)')
  if args.cs:
    correct_and_smooth(logits, graph)
