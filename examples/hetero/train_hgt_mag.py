"""HGT on an OGB-MAG-shaped heterogeneous graph through the hetero `NeighborLoader`.

Counterpart of the reference's examples/hetero/train_hgt_mag.py (PyG HGTConv, hidden 64, 2 heads, 2 layers,
fanout [10, 10], batch 1024, ZERO_COPY topology + 20 % of the features on the GPU): the model is this repo's
dependency-free `models.HGT`, the graph is synthetic with the MAG schema (no network access; swap
`synthetic_mag` for the real tensors).  On a GPU the loader samples through the native grouped hetero arena
(one launch per hop over all seven relations).

`--mode engine` trains `models.HeteroHgtEngine` instead: the whole step (sampling, the HGT layers on the project's
sm_90a kernels, loss, backward and Adam) as one CUDA graph on one GPU, with the reference's hyper-parameters.  The
engine's model has a per-type input `Linear` + ReLU in front of its HGT layers, as the reference's model does; the
loader mode trains `models.HGT`, which has no input Linear, so the two modes do not train the same architecture.

`--featureless metapath2vec` (needs a GPU) gives every node type except paper the embeddings `models.MetaPath2VecEngine`
trains over the metapath author -> paper -> field_of_study -> paper -> author -> institution -> author, with PyG's
MetaPath2Vec hyper-parameters (the reference's `OGB_MAG(preprocess='metapath2vec')` vectors come from that recipe).
It runs for --m2v-steps steps of 128 start authors (default: one pass over the authors).  On synthetic data it
replaces the random features of those types; the default, `--featureless mean`, keeps the neighbour means of
`load_mag_from_disk`.
"""
import argparse
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from common import glt, synthetic_mag  # noqa: E402
from graphlearn_for_pytorch_b200.models import HGT  # noqa: E402


MAG_METAPATH = [('author', 'writes', 'paper'), ('paper', 'has_topic', 'field_of_study'),
                ('field_of_study', 'rev_has_topic', 'paper'), ('paper', 'rev_writes', 'author'),
                ('author', 'affiliated_with', 'institution'), ('institution', 'rev_affiliated_with', 'author')]
M2V_ARGS = dict(embedding_dim=128, walk_length=64, context_size=7, walks_per_node=5, num_negative_samples=5,
                batch_size=128, lr=0.01)


def metapath2vec_features(edges, sizes, feats, steps=0, seed=0):
  """feats with every type except paper replaced by metapath2vec embeddings of the paper features' width, trained by
  MetaPath2VecEngine on cuda:0 for `steps` steps (0: one pass over the authors)."""
  from graphlearn_for_pytorch_b200.models import MetaPath2VecEngine
  dev = torch.device('cuda', 0)
  graphs = {e: glt.data.Graph(glt.data.Topology(edges[e], layout='CSR', num_nodes=max(sizes[e[0]], sizes[e[2]])),
                              'CUDA', 0) for e in MAG_METAPATH}
  hp = dict(M2V_ARGS, embedding_dim=feats['paper'].shape[1])
  eng = MetaPath2VecEngine(graphs, sizes, MAG_METAPATH, seed=seed, device=dev, **hp)
  eng.warmup_and_capture()
  B = hp['batch_size']
  steps = steps or -(-sizes['author'] // B)
  t0, done, losses = time.time(), 0, []
  while done < steps:
    perm = torch.randperm(sizes['author'], device=dev)
    for i in range(0, perm.numel(), B):
      losses.append(eng.train_step(perm[i:i + B]).clone())
      done += 1
      if done == steps:
        break
  print(f'metapath2vec: {steps} steps, loss {float(losses[0]):.4f} -> {float(torch.stack(losses[-10:]).mean()):.4f}, '
        f'{time.time() - t0:.1f}s')
  out = dict(feats)
  for t in eng.node_types:
    if t != 'paper':
      out[t] = eng.embedding(t).cpu()
  return out


def load_mag_from_disk(root, name='ogbn-mag'):
  """ogbn-mag from its OGB directory: reverse relations are added (what T.ToUndirected(merge=True) does in the
  reference script) and node types that ship without features get the mean of their featured neighbours' rows,
  propagated until every type has some (author <- papers written, institution <- authors, field <- papers); the
  reference substitutes pre-trained metapath2vec vectors there (examples/hetero/train_hgt_mag.py:33-36), which
  `--featureless metapath2vec` trains with MetaPath2VecEngine."""
  d = glt.utils.load_ogb_hetero_dataset(root, name)
  edges = dict(d['edge_index'])
  for (s, r, t), ei in list(edges.items()):
    if s == t:
      edges[(s, r, t)] = torch.cat([ei, ei.flip(0)], 1)
    elif (t, f'rev_{r}', s) not in edges:
      edges[(t, f'rev_{r}', s)] = ei.flip(0)
  sizes, feats = dict(d['num_nodes']), dict(d['x'])
  while len(feats) < len(sizes):
    progressed = False
    for (s, r, t), ei in edges.items():
      if s in feats and t not in feats:
        acc = torch.zeros(sizes[t], feats[s].shape[1]).index_add_(0, ei[1], feats[s][ei[0]])
        deg = torch.zeros(sizes[t]).index_add_(0, ei[1], torch.ones(ei.shape[1]))
        feats[t] = acc / deg.clamp(min=1).unsqueeze(1)
        progressed = True
    if not progressed:
      raise ValueError(f'node types without features and without a featured neighbour type: '
                       f'{sorted(set(sizes) - set(feats))}')
  labels = {t: v.to(torch.int64) for t, v in d['y'].items()}
  return edges, feats, labels, sizes, d['split']


def load_data(args):
  """(edges, feats, labels, sizes, split or None) from --root or synthetic, with the --featureless choice applied."""
  split = None
  if getattr(args, 'root', None):
    edges, feats, labels, sizes, split = load_mag_from_disk(args.root, args.dataset)
  else:
    edges, feats, labels, sizes = synthetic_mag(args.papers)
  if getattr(args, 'featureless', 'mean') == 'metapath2vec':
    feats = metapath2vec_features(edges, sizes, feats, args.m2v_steps)
  return edges, feats, labels, sizes, split


def build_dataset(args, cuda, device_index=0):
  edges, feats, labels, sizes, split = load_data(args)
  ds = glt.data.Dataset()
  ds.init_graph(edges, graph_mode=('ZERO_COPY' if args.zero_copy else 'CUDA') if cuda else 'CPU', num_nodes=sizes,
                device=device_index)
  ds.init_node_features(feats, split_ratio=args.split_ratio if cuda else 0.0, with_gpu=cuda, device=device_index)
  ds.init_node_labels(labels)
  if split and 'train' in split and 'paper' in split['train']:
    return ds, sizes, labels, split['train']['paper'], split.get('valid', split['train'])['paper']
  n = sizes['paper']
  perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
  return ds, sizes, labels, perm[: n // 2], perm[n // 2: n // 2 + n // 10]


def make_model(ds, sizes, labels, loader, args, device):
  first = next(iter(loader))
  in_dim = ds.node_features['paper'].shape[1]
  return HGT(list(sizes.keys()), list(first.edge_index_dict.keys()), in_dim, args.hidden, int(labels['paper'].max()) + 1,
             num_layers=2, heads=args.heads, node_type='paper').to(device)


def train_epoch(model, loader, opt, device):
  model.train()
  tot = seen = 0
  for b in loader:
    bs = b['paper'].batch_size
    out = model(b.x_dict, b.edge_index_dict)[:bs]
    loss = F.cross_entropy(out, b['paper'].y[:bs].to(device))
    opt.zero_grad(); loss.backward(); opt.step()
    tot += float(loss.detach()) * bs; seen += bs
  return tot / max(seen, 1)


@torch.no_grad()
def evaluate(model, loader, device):
  model.eval()
  correct = seen = 0
  for b in loader:
    bs = b['paper'].batch_size
    pred = model(b.x_dict, b.edge_index_dict)[:bs].argmax(-1)
    correct += int((pred == b['paper'].y[:bs].to(device)).sum()); seen += bs
  return correct / max(seen, 1)


def parse():
  p = argparse.ArgumentParser()
  p.add_argument('--root', default=None, help='directory that contains ogbn_mag/ (OGB raw layout); default: synthetic')
  p.add_argument('--dataset', default='ogbn-mag')
  p.add_argument('--papers', type=int, default=30_000)
  p.add_argument('--epochs', type=int, default=3)
  p.add_argument('--batch', type=int, default=1024)
  p.add_argument('--hidden', type=int, default=64)
  p.add_argument('--heads', type=int, default=2)
  p.add_argument('--split-ratio', type=float, default=0.2)
  p.add_argument('--zero-copy', action='store_true', help='keep the topology in pinned host memory (reference default)')
  p.add_argument('--mode', choices=['loader', 'engine'], default='loader',
                 help='loader: hetero NeighborLoader + models.HGT under autograd; engine: HeteroHgtEngine (one GPU)')
  p.add_argument('--feat-format', choices=['bf16', 'mxfp8'], default='bf16',
                 help='--mode engine: store the feature tables as MXFP8 rows (e4m3 + one scale per 32 elements)')
  p.add_argument('--eval', choices=['sampled', 'full'], default='sampled',
                 help='--mode engine: validation accuracy from sampled batches (evaluate_batch), or validation and test '
                      'accuracy of exact layer-wise full-neighbourhood inference (HeteroHgtEngine.inference)')
  p.add_argument('--featureless', choices=['mean', 'metapath2vec'], default='mean',
                 help='features of the types other than paper: neighbour means (--root) or the synthetic ones, or '
                      'metapath2vec embeddings trained by MetaPath2VecEngine (needs a GPU)')
  p.add_argument('--m2v-steps', type=int, default=0,
                 help='--featureless metapath2vec: training steps of 128 start authors (0: one pass over the authors)')
  return p.parse_args()


def run_engine(args):
  """Train HeteroHgtEngine with the reference's hyper-parameters (fanout [10, 10], Adam lr 0.01)."""
  from graphlearn_for_pytorch_b200.models import HeteroHgtEngine
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  edges, feats, labels, sizes, split = load_data(args)
  if split and 'train' in split and 'paper' in split['train']:
    train_idx, val_idx = split['train']['paper'], split.get('valid', split['train'])['paper']
    test_idx = split.get('test', split.get('valid', split['train']))['paper']
  else:
    n = sizes['paper']
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(1))
    train_idx, val_idx = perm[: n // 2], perm[n // 2: n // 2 + n // 10]
    test_idx = perm[n // 2 + n // 10: n // 2 + n // 5]
  graphs, tables, keep = {}, {}, []
  for et, ei in edges.items():
    topo = glt.data.Topology(ei.to(dev), layout='CSC', num_nodes=sizes[et[2]])
    graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
  in_dim, fmt = {}, {}
  for t, x in feats.items():
    rows = x.to(dev).to(torch.bfloat16)
    fmt[t] = 'mxfp8' if args.feat_format == 'mxfp8' and x.shape[1] % 32 == 0 else 'bf16'
    if fmt[t] == 'mxfp8':
      rows = glt.data.quantize_mxfp8_chunked(rows)
    ut = glt.data.UnifiedTensor(0, rows.dtype)
    ut.append_shared_tensor(rows)
    keep.append(ut)
    tables[t] = ut._table()
    in_dim[t] = x.shape[1]
  y = labels['paper']
  eng = HeteroHgtEngine(graphs, tables, y.to(dev), in_dim, sizes, 'paper', fanouts=[10, 10], batch_size=args.batch,
                        hidden=args.hidden, heads=args.heads, num_classes=int(y.max()) + 1, edge_dir='in', lr=0.01,
                        device=dev, feature_format=fmt)
  eng.warmup_and_capture()
  print(f'HeteroHgtEngine: {eng.kernels_per_step} kernels per step, one CUDA graph')
  for epoch in range(1, args.epochs + 1):
    t0 = time.time()
    perm = train_idx[torch.randperm(train_idx.numel())].to(dev)
    losses = [eng.train_step(perm[i:i + args.batch]).clone() for i in range(0, perm.numel(), args.batch)]
    loss = float(torch.stack(losses).mean())
    if args.eval == 'full':
      pred = eng.inference().argmax(-1).cpu()
      val, test = (float((pred[idx] == y[idx]).float().mean()) for idx in (val_idx, test_idx))
      print(f'Epoch: {epoch:02d}, Loss: {loss:.4f}, Val: {val:.4f}, Test: {test:.4f} (full-neighbourhood), '
            f'Time: {time.time() - t0:.2f}s')
      continue
    correct = seen = 0
    for i in range(0, val_idx.numel(), args.batch):
      _, c, n = eng.evaluate_batch(val_idx[i:i + args.batch].to(dev))
      correct += c; seen += n
    print(f'Epoch: {epoch:02d}, Loss: {loss:.4f}, Val: {correct / max(seen, 1):.4f}, Time: {time.time() - t0:.2f}s')
  eng.close()


if __name__ == '__main__':
  args = parse()
  if args.featureless == 'metapath2vec' and not torch.cuda.is_available():
    sys.exit('--featureless metapath2vec trains MetaPath2VecEngine, which needs a CUDA GPU; use --featureless mean '
             'without one')
  if args.mode == 'engine':
    if not torch.cuda.is_available():
      sys.exit('--mode engine trains HeteroHgtEngine, which needs a CUDA GPU; use the default --mode loader without one')
    run_engine(args)
    sys.exit(0)
  cuda = torch.cuda.is_available()
  device = torch.device('cuda', 0) if cuda else torch.device('cpu')
  ds, sizes, labels, train_idx, val_idx = build_dataset(args, cuda)
  train_loader = glt.loader.NeighborLoader(ds, [10, 10], ('paper', train_idx), batch_size=args.batch, shuffle=True,
                                           device=device)
  val_loader = glt.loader.NeighborLoader(ds, [10, 10], ('paper', val_idx), batch_size=args.batch, device=device)
  model = make_model(ds, sizes, labels, train_loader, args, device)
  opt = torch.optim.Adam(model.parameters(), lr=0.01)
  for epoch in range(1, args.epochs + 1):
    t0 = time.time()
    loss = train_epoch(model, train_loader, opt, device)
    acc = evaluate(model, val_loader, device)
    print(f'Epoch: {epoch:02d}, Loss: {loss:.4f}, Val: {acc:.4f}, Time: {time.time() - t0:.2f}s')
