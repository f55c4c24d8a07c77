"""SEAL link prediction: enclosing-subgraph sampling + DRNL + DGCNN
(counterpart of the reference's examples/seal_link_pred.py).

  python examples/seal_link_pred.py                  # per-link extract + DRNL on the host, eager DGCNN
  python examples/seal_link_pred.py --mode engine    # SealEngine: the reference's DGCNN in one captured CUDA-graph step
                                                     # per batch, then the val / test AUC of held-out links
"""
import argparse
import math

import torch
import torch.nn.functional as F

from common import glt, synthetic_homo
from graphlearn_for_pytorch_b200.models import DGCNN, drnl_node_labeling
from graphlearn_for_pytorch_b200.sampler import NeighborSampler, NodeSamplerInput, RandomNegativeSampler

ap = argparse.ArgumentParser()
ap.add_argument('--links', type=int, default=2000, help='positive (and negative) links')
ap.add_argument('--epochs', type=int, default=2)
ap.add_argument('--mode', default='eager', choices=['eager', 'engine'])
args = ap.parse_args()
L = args.links
cuda = torch.cuda.is_available()
device = torch.device('cuda', 0) if cuda else torch.device('cpu')
ei, _, _ = synthetic_homo(3_000, 24_000, feat_dim=4, num_classes=2)


def auc(pos, neg):
  """ROC AUC of positive against negative scores (rank statistic)."""
  r = torch.cat([pos, neg]).double().argsort().argsort().double() + 1
  return float((r[:pos.numel()].sum() - pos.numel() * (pos.numel() + 1) / 2) / (pos.numel() * neg.numel()))


def run_engine():
  """Hold out 5% / 10% of the undirected edges as val / test links (the reference's RandomLinkSplit), train SealEngine
  on the rest, and score val on the training graph and test on the training + val graph, as the reference does."""
  from graphlearn_for_pytorch_b200.models import SealEngine
  if not cuda:
    raise SystemExit('--mode engine needs a GPU')
  n = 3000
  und = torch.unique(ei[:, ei[0] < ei[1]], dim=1)
  und = und[:, torch.randperm(und.shape[1], generator=torch.Generator().manual_seed(0))]
  n_val, n_test = int(0.05 * und.shape[1]), int(0.1 * und.shape[1])
  val, test, train = und[:, :n_val], und[:, n_val:n_val + n_test], und[:, n_val + n_test:]
  both = lambda e: torch.cat([e, e.flip(0)], 1)
  graph_of = lambda e: glt.data.Graph(glt.data.Topology(both(e), layout='CSR', num_nodes=n), 'CUDA')
  train_g, test_g = graph_of(train), graph_of(torch.cat([train, val], 1))
  gen = torch.Generator().manual_seed(1)
  neg = lambda k: torch.randint(0, n, (2, k), generator=gen)
  pos = train[:, :L]
  links = torch.cat([pos, neg(pos.shape[1])], 1)
  labels = torch.cat([torch.ones(pos.shape[1]), torch.zeros(pos.shape[1])])
  eng = SealEngine(train_g, n, num_hops=2, max_nodes=512, hidden=32, num_layers=3, sort_k=0.6, batch_size=256,
                   lr=1e-3, calibration_links=links)
  eng.warmup_and_capture()
  val_neg, test_neg = neg(val.shape[1]), neg(test.shape[1])
  for epoch in range(args.epochs):
    perm = torch.randperm(links.shape[1], generator=gen)
    tot, steps = 0.0, math.ceil(perm.numel() / 256)
    for i in range(0, perm.numel(), 256):
      idx = perm[i:i + 256]
      tot += float(eng.train_step(links[:, idx].to(device), labels[idx].to(device)))
    val_auc = auc(eng.predict(val.to(device)).cpu(), eng.predict(val_neg.to(device)).cpu())
    test_auc = auc(eng.predict(test.to(device), graph=test_g).cpu(), eng.predict(test_neg.to(device), graph=test_g).cpu())
    print(f'epoch {epoch}: loss {tot / steps:.4f} val AUC {val_auc:.4f} test AUC {test_auc:.4f} '
          f'(k {eng.k}, max_z {eng.max_z}, truncated links {eng.truncated()})')


if args.mode == 'engine':
  run_engine()
  raise SystemExit(0)
topo = glt.data.Topology(ei, layout='CSR', num_nodes=3000)
graph = glt.data.Graph(topo, 'CUDA' if cuda else 'CPU')
sampler = NeighborSampler(graph, [-1], device=device)          # 1-hop enclosing subgraphs
neg = RandomNegativeSampler(graph, 'CUDA' if cuda else 'CPU').sample(L, padding=True).cpu()
pos = ei[:, torch.randperm(ei.shape[1])[:L]]
links = torch.cat([pos, neg], 1)
labels = torch.cat([torch.ones(L), torch.zeros(L)])
model = DGCNN(num_labels=200, hidden=32, num_layers=3, k=30).to(device)
opt = torch.optim.Adam(model.parameters(), lr=1e-3)


def extract(batch_links):
  zs, eis, batch, off = [], [], [], 0
  for g, (s, d) in enumerate(batch_links.t().tolist()):
    out = sampler.subgraph(NodeSamplerInput(torch.tensor([s, d])))
    sub_ei = torch.stack([out.row, out.col])
    m = out.metadata
    keep = ~(((sub_ei[0] == m[0]) & (sub_ei[1] == m[1])) | ((sub_ei[0] == m[1]) & (sub_ei[1] == m[0])))
    sub_ei = sub_ei[:, keep]                                    # hide the target link
    n = out.node.numel()
    zs.append(drnl_node_labeling(sub_ei, int(m[0]), int(m[1]), n, max_z=199))
    eis.append(sub_ei + off)
    batch.append(torch.full((n,), g, device=device))
    off += n
  return torch.cat(zs), torch.cat(eis, 1), torch.cat(batch)


for epoch in range(args.epochs):
  perm = torch.randperm(links.shape[1])
  tot, correct = 0.0, 0
  for i in range(0, perm.numel(), 32):
    idx = perm[i:i + 32]
    z, sub_ei, batch = extract(links[:, idx])
    logit = model(z.to(device), sub_ei.to(device), batch, idx.numel())
    y = labels[idx].to(device)
    loss = F.binary_cross_entropy_with_logits(logit, y)
    opt.zero_grad(); loss.backward(); opt.step()
    tot += float(loss.detach()) * idx.numel(); correct += int(((logit > 0).float() == y).sum())
  print(f'epoch {epoch}: loss {tot / perm.numel():.4f} acc {correct / perm.numel():.4f}')
