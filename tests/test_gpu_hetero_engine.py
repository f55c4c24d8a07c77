"""HeteroSageEngine (device-resident R-SAGE step) against a plain fp32 PyTorch recomputation on the SAME sampled
batch: forward loss, weight and bias gradients of every (layer, type), and training progress under CUDA-graph
replay.  The numerics are checked at 64-wide features / hidden 64 / 19 classes, at IGBH-like per-type feature widths
(up to 1024) with a hidden width that does not divide 2048, and with the 2983-class IGBH label set."""
import os
import sys

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))


def _build(papers=4000, feat_dim=64, hidden=64, fan=(4, 3, 2), bs=256, use_graph=False, classes=19):
  """feat_dim: one width for every node type, or {type: width}."""
  from common import synthetic_igbh
  from graphlearn_for_pytorch_b200.models import HeteroSageEngine
  edges, feats, labels, sizes = synthetic_igbh(papers, papers // 2, 50, 30, feat_dim=64, num_classes=classes, seed=2)
  if isinstance(feat_dim, dict):
    g = torch.Generator().manual_seed(3)
    feats = {t: torch.randn(sizes[t], feat_dim[t], generator=g) for t in sizes}
  elif feat_dim != 64:
    feats = {t: torch.randn(sizes[t], feat_dim, generator=torch.Generator().manual_seed(3)) for t in sizes}
  graphs, tables, keep = {}, {}, []
  for et, ei in edges.items():
    topo = glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=sizes[et[2]])
    graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
  fb = {}
  for nt, x in feats.items():
    fb[nt] = x.to(DEV).to(torch.bfloat16)
    ut = glt.data.UnifiedTensor(0, torch.bfloat16)
    ut.append_shared_tensor(fb[nt])
    tables[nt] = ut._table()
    keep.append(ut)
  eng = HeteroSageEngine(graphs, tables, labels['paper'].to(DEV), feat_dim, sizes, 'paper', fanouts=list(fan),
                         batch_size=bs, hidden=hidden, num_classes=classes, edge_dir='in', lr=5e-3, seed=1,
                         device=DEV, use_cuda_graph=use_graph)
  eng._keep = keep
  return eng, fb, labels['paper'].to(DEV), sizes


def _reference(eng, fb, labels):
  """fp32 recomputation from the arena's COO, rounding to bf16 where the engine stores bf16."""
  nodes, rows, cols, _, nn, ne = eng.arena.to_coo()
  L, nt, kt = eng.L, eng.nt, eng.kt
  bf = lambda x: x.to(torch.bfloat16).float()
  P = {k: eng.param(k).float().requires_grad_(True) for k in eng.param_index}
  x = {t: fb[eng.ntypes[t]][nodes[t]].float() for t in range(len(eng.ntypes))}
  for l in range(1, L + 1):
    nh = L - l + 1
    out = {}
    for t in eng.targets[l]:
      T = sum(nn[t][:nh])
      blocks = []
      for r in eng.in_rel[l][t]:
        E = sum(ne[r][:nh])
        src, dst = rows[r][:E], cols[r][:E]
        d = x[nt[r]].shape[1]
        agg = torch.zeros(T, d, device=DEV).index_add_(0, dst, x[nt[r]][src])
        deg = torch.zeros(T, device=DEV).index_add_(0, dst, torch.ones(E, device=DEV))
        blocks.append(bf(agg / deg.clamp(min=1).unsqueeze(1)))
      blocks.append(x[t][:T])
      A = torch.cat(blocks, 1)
      z = A @ P[('W', l, t)].t() + P[('b', l, t)]
      out[t] = bf(torch.relu(z)) if l < L else z
    x = out
  st = eng.tid[eng.seed_type]
  n0 = nn[st][0]
  logits = x[st][:n0, :eng.C]
  y = labels[nodes[st][:n0]]
  loss = torch.nn.functional.cross_entropy(logits, y)
  loss.backward()
  return float(loss), {k: p.grad for k, p in P.items()}, (nn, ne)


def _gradient_errors(feat_dim=64, hidden=64, classes=19, batch_seed=0):
  """Runs one engine step on a seeded batch and returns {name: max |engine - fp32 reference| / max |reference|} for the
  loss and every weight and bias gradient."""
  eng, fb, labels, sizes = _build(feat_dim=feat_dim, hidden=hidden, classes=classes)
  seeds = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(batch_seed))[:eng.bs]
  eng._seeds.copy_(seeds.to(DEV))
  eng._sample()
  eng._forward()
  eng._backward()
  torch.cuda.synchronize()
  assert eng.overflow_count() == 0
  ref_loss, ref_grads, (nn, ne) = _reference(eng, fb, labels)
  assert sum(sum(v) for v in ne) > 1000                     # the batch really has relations of every kind
  errs = {'loss': abs(float(eng.loss.item()) - ref_loss) / max(1.0, abs(ref_loss))}
  for k, r in ref_grads.items():
    if r is not None:
      errs[f'{k[0]}{k[1:]}'] = float((eng.param(k, True) - r).abs().max()) / max(float(r.abs().max()), 1e-6)
  return errs


def _assert_gradients_match(errs):
  assert errs.pop('loss') < 3e-2, errs
  bad = {k: e for k, e in errs.items() if not e < 6e-2}
  assert not bad, bad


def test_hetero_engine_forward_backward_match_fp32():
  _assert_gradients_match(_gradient_errors())


@pytest.mark.parametrize('feat_dim,hidden,classes', [
    ({'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128}, 192, 19),   # hidden width not dividing 2048
    (64, 64, 2983),                                                          # IGBH's 2983-class label set
], ids=['igbh_widths-192-19', '64-64-2983'])
def test_hetero_engine_gradients_match_fp32_at_wide_layers(feat_dim, hidden, classes):
  _assert_gradients_match(_gradient_errors(feat_dim, hidden, classes))


@pytest.mark.parametrize('feat_dim,hidden', [
    ({'paper': 64, 'author': 64, 'institute': 64, 'fos': 40}, 64),   # fos operand 64 + 40 = 104 columns
    (2048, 64),
    (64, 96),
    (64, 2048),
])
def test_hetero_engine_rejects_unsupported_widths(feat_dim, hidden):
  with pytest.raises(ValueError, match='in_dim|hidden|multiple of 64'):
    _build(papers=1000, feat_dim=feat_dim, hidden=hidden)


def test_hetero_engine_trains_under_cuda_graph():
  eng, fb, labels, sizes = _build(use_graph=True)
  eng.warmup_and_capture(n_eager=1)
  assert eng._graph is not None
  g = torch.Generator().manual_seed(0)
  losses = []
  for i in range(60):
    seeds = torch.randperm(sizes['paper'], generator=g)[:eng.bs].to(DEV)
    losses.append(float(eng.train_step(seeds).item()))
  assert all(l == l for l in losses)
  assert sum(losses[-10:]) / 10 < sum(losses[:10]) / 10 - 0.05, (losses[:5], losses[-5:])
  l, c, n = eng.evaluate_batch(torch.arange(eng.bs, device=DEV))
  assert n == eng.bs and 0 <= c <= n
  nodes, edges = eng.batch_sizes()
  assert nodes['paper'][0] == eng.bs and sum(sum(v) for v in edges.values()) > 0
