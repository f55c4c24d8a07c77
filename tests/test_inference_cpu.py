"""GraphSageTrainer.inference(): exact layer-wise full-neighbourhood inference on the host."""
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageTrainer
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges


def _trainer(ei, n, d, c, fanouts, hidden=32, train_steps=10):
  torch.manual_seed(1)
  x = torch.randn(n, d)
  y = torch.randint(0, c, (n,))
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CPU', directed=False, num_nodes=n)
  ds.init_node_features(x, with_gpu=False)
  tr = GraphSageTrainer(ds.graph, ds.node_features, y, in_dim=d, fanouts=fanouts, hidden=hidden, num_classes=c,
                        lr=1e-2, seed=3)
  for _ in range(train_steps):
    tr.train_step(torch.randperm(n)[:128])
  return tr, ds, x, y


def _index_add_reference(tr, indptr, indices, x):
  """Independent recomputation: mean over every CSR row by index_add, then [mean | self] . [W_l | W_r]^T + b."""
  n = indptr.numel() - 1
  deg = (indptr[1:] - indptr[:-1]).float()
  dst = torch.repeat_interleave(torch.arange(n), indptr[1:] - indptr[:-1])
  h = x.double()
  convs = tr.model.convs
  for i, conv in enumerate(convs):
    s = torch.zeros(n, h.shape[1], dtype=torch.float64).index_add_(0, dst, h[indices.long()])
    mean = s / deg.clamp(min=1).double().unsqueeze(1)
    W = torch.cat([conv.lin_l.weight, conv.lin_r.weight], 1).double()
    h = torch.cat([mean, h], 1) @ W.t() + conv.lin_l.bias.double()
    if i < len(convs) - 1:
      h = h.clamp(min=0)
  return h


def test_trainer_inference_matches_index_add_over_the_csr():
  n, d, c = 1500, 16, 5
  ei = rmat_edges(n, 9000, seed=2)
  ei = torch.cat([ei, ei.flip(0), torch.tensor([[3, 3], [7, 7]])], 1)     # a repeated edge counts twice
  tr, ds, x, _ = _trainer(ei, n, d, c, [5, 5])
  topo = ds.graph.topo
  got = tr.inference(chunk_rows=257)
  assert got.shape == (n, c) and got.dtype == torch.float32
  ref = _index_add_reference(tr, topo.indptr, topo.indices, x)
  torch.testing.assert_close(got.double(), ref, rtol=1e-4, atol=1e-4)
  assert torch.equal(got, tr.inference())                       # chunking does not change the result


def test_trainer_inference_agrees_with_evaluate_batch_when_fanout_covers_every_row():
  # a bounded-degree graph: every node has at most 6 neighbours, so fanouts [6, 6] sample every neighbourhood whole
  n, d, c = 800, 16, 4
  g = torch.Generator().manual_seed(5)
  src = torch.arange(n).repeat_interleave(3)
  dst = torch.randint(0, n, (3 * n,), generator=g)
  ei = torch.stack([src, dst])
  ei = torch.unique(torch.cat([ei, ei.flip(0)], 1), dim=1)
  keep = ei[0] != ei[1]
  ei = ei[:, keep]
  deg = torch.bincount(ei[0], minlength=n)
  ok = (deg[ei[0]] <= 6) & (deg[ei[1]] <= 6)
  ei = ei[:, ok]
  tr, ds, x, y = _trainer(ei, n, d, c, [6, 6])
  topo = ds.graph.topo
  assert int((topo.indptr[1:] - topo.indptr[:-1]).max()) <= 6
  logits = tr.inference()
  seeds = torch.randperm(n)[:200]
  _, correct, m = tr.evaluate_batch(seeds)
  assert m == 200
  assert correct == int((logits[seeds].argmax(1) == y[seeds]).sum())
