"""Unsupervised GraphSAGE with link sampling + binary negatives
(counterpart of the reference's examples/graph_sage_unsup_ppi.py).

  python examples/graph_sage_unsup.py                  # LinkNeighborLoader + eager GraphSAGE + torch Adam
  python examples/graph_sage_unsup.py --mode engine    # GraphSageLinkEngine (GraphSageLinkTrainer without a GPU),
                                                       # then the held-out link AUC of the inference() embeddings
  python examples/graph_sage_unsup.py --mode engine --rank-k 20
                                                       # also recall@20 of the held-out edges over every node
                                                       # (training edges excluded), Hits@20 and MRR
"""
import argparse

import torch
import torch.nn.functional as F

from common import glt, synthetic_homo
from graphlearn_for_pytorch_b200.models import GraphSAGE
from graphlearn_for_pytorch_b200.sampler import NegativeSampling

p = argparse.ArgumentParser()
p.add_argument('--mode', default='loader', choices=['loader', 'engine'])
p.add_argument('--epochs', type=int, default=2)
p.add_argument('--steps-per-epoch', type=int, default=40, help='engine mode: training steps per epoch')
p.add_argument('--rank-k', type=int, default=0,
               help='engine mode: also rank every node for each held-out edge endpoint and print recall@K, Hits@K, MRR')
args = p.parse_args()

cuda = torch.cuda.is_available()
device = torch.device('cuda', 0) if cuda else torch.device('cpu')
ei, x, _ = synthetic_homo(20_000, 200_000, feat_dim=50, num_classes=4)


def run_loader():
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CUDA' if cuda else 'CPU')
  ds.init_node_features(x, with_gpu=cuda, split_ratio=1.0 if cuda else 0.0)
  loader = glt.loader.LinkNeighborLoader(ds, [10, 10], edge_label_index=ei[:, :20_000], batch_size=512,
                                         shuffle=True, neg_sampling=NegativeSampling('binary', 1), device=device)
  model = GraphSAGE(50, 64, 64, num_layers=2).to(device)
  opt = torch.optim.Adam(model.parameters(), lr=5e-3)
  for epoch in range(args.epochs):
    tot = 0.0
    for b in loader:
      h = model(b.x, b.edge_index)
      src, dst = b.edge_label_index[1], b.edge_label_index[0]
      logit = (h[src] * h[dst]).sum(-1)
      loss = F.binary_cross_entropy_with_logits(logit, b.edge_label.float().to(device))
      opt.zero_grad(); loss.backward(); opt.step()
      tot += float(loss.detach())
    print(f'epoch {epoch}: loss {tot / len(loader):.4f}')


def run_engine():
  from graphlearn_for_pytorch_b200.models import GraphSageLinkEngine, GraphSageLinkTrainer, link_auc
  N, bs = x.shape[0], 512
  g = torch.Generator().manual_seed(0)
  # hold out 5 % of the (undirected) edges: they are removed from the graph the model samples from
  und = ei[:, ei[0] < ei[1]]
  und = und[:, torch.randperm(und.shape[1], generator=g)]
  n_held = und.shape[1] // 20
  held, train = und[:, :n_held], und[:, n_held:]
  topo = glt.data.Topology(torch.cat([train, train.flip(0)], 1), layout='CSR', num_nodes=N)
  in_dim = (x.shape[1] + 7) // 8 * 8                       # the engine wants feature rows of a multiple of 8
  feats = F.pad(x, (0, in_dim - x.shape[1]))
  graph = glt.data.Graph(topo, 'CUDA' if cuda else 'CPU', 0 if cuda else None)
  if cuda:
    ut = glt.data.UnifiedTensor(0, torch.bfloat16)
    ut.append_shared_tensor(feats.to(device, torch.bfloat16))
    model = GraphSageLinkEngine(graph, ut._table(), in_dim, N, fanouts=[10, 10], batch_size=bs, hidden=64,
                                out_channels=64, lr=5e-3, device=device)
    model.warmup_and_capture(n_eager=1)
  else:
    model = GraphSageLinkTrainer(graph, feats, in_dim, fanouts=[10, 10], hidden=64,
                                 out_channels=64, lr=5e-3)
  for epoch in range(args.epochs):
    perm = train[:, torch.randperm(train.shape[1], generator=g)[:args.steps_per_epoch * bs]]
    losses = [float(model.train_step(perm[:, i:i + bs])) for i in range(0, perm.shape[1], bs)]
    print(f'epoch {epoch}: loss {sum(losses) / len(losses):.4f}')
  neg = torch.randint(0, N, (2, n_held), generator=g)     # as many uniform random pairs as held-out edges
  emb_dev = model.inference()
  emb = emb_dev.cpu()
  print(f'held-out link AUC {link_auc(emb, held, neg):.4f} ({n_held} edges vs {n_held} random pairs)')
  if args.rank_k > 0:
    rank_report(emb_dev, graph, held, neg, N)


def rank_report(emb, graph, held, neg, N):
  """recall@K of the held-out edges over every node (training edges excluded), and Hits@K / MRR of the held-out edges
  against the random pairs."""
  from graphlearn_for_pytorch_b200.models import link_hits_at_k, link_mrr, link_recall_at_k, link_scores, link_topk
  K = args.rank_k
  truth = glt.data.Topology(torch.cat([held, held.flip(0)], 1), layout='CSR', num_nodes=N)
  queries = torch.unique(held).to(emb.device)
  ids, _ = link_topk(emb, queries, K, exclude=graph)
  recall, hit = link_recall_at_k(ids, (truth.indptr, truth.indices), queries)
  pos, negs = link_scores(emb, held), link_scores(emb, neg)
  print(f'held-out recall@{K} {recall:.4f} (hit rate {hit:.4f}, {queries.numel()} query nodes, training edges '
        f'excluded); Hits@{K} {link_hits_at_k(pos, negs, K):.4f}, '
        f'MRR {link_mrr(pos, negs.unsqueeze(0).expand(pos.numel(), -1)):.4f} against the random pairs')


run_loader() if args.mode == 'loader' else run_engine()
