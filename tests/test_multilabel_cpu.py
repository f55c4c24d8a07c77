"""Multi-label node classification without a GPU: the label bit matrix, the ROC-AUC / F1 helpers against brute force,
`GraphSageMultiLabelTrainer` against a hand-written autograd step, and the example script in trainer mode."""
import copy
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageMultiLabelTrainer, multilabel_auc, multilabel_f1, pack_label_bits
from graphlearn_for_pytorch_b200.models.sage_multilabel import check_multilabel
from graphlearn_for_pytorch_b200.utils.synthetic import multilabel_targets, rmat_edges

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unpack_label_bits(bits, T):
  b = bits.to(torch.int64)
  return ((b.unsqueeze(-1) >> torch.arange(32)) & 1).view(b.shape[0], -1)[:, :T]


@pytest.mark.parametrize('T', [1, 31, 32, 33, 112, 121])
@pytest.mark.parametrize('dtype', [torch.bool, torch.int64, torch.float32])
def test_pack_label_bits_round_trips(T, dtype):
  y = torch.rand(57, T, generator=torch.Generator().manual_seed(T)) < 0.4
  y[0] = True                                 # bit 31 of a full word: the sign bit of an int32 view
  y[1] = False
  bits = pack_label_bits(y.to(dtype))
  assert bits.dtype == torch.uint32 and bits.shape == (57, (T + 31) // 32) and bits.is_contiguous()
  full = unpack_label_bits(bits, 32 * bits.shape[1])
  assert torch.equal(full[:, :T], y.to(torch.int64))
  assert not bool(full[:, T:].any())                # padding bits are zero


@pytest.mark.parametrize('bad', [torch.tensor([[0, 2]]), torch.tensor([[0.5, 1.0]]), torch.tensor([[-1, 0]]),
                                 torch.tensor([[float('nan'), 1.0]])])
def test_non_binary_labels_raise(bad):
  with pytest.raises(ValueError, match='0 and 1'):
    pack_label_bits(bad)


@pytest.mark.parametrize('bad', [torch.zeros(5), torch.zeros(5, 0), torch.zeros(2, 3, 4)])
def test_misshaped_labels_raise(bad):
  with pytest.raises(ValueError, match='num_nodes, T'):
    pack_label_bits(bad)
  with pytest.raises(ValueError):
    check_multilabel(torch.zeros(5, 3), num_nodes=6)


def _brute_auc(s, y):
  """Mean over tasks with both classes of P(score_pos > score_neg) + P(tie) / 2, by counting every pair in float64."""
  aucs = []
  for t in range(y.shape[1]):
    p, n = s[y[:, t], t].double(), s[~y[:, t], t].double()
    if p.numel() == 0 or n.numel() == 0:
      continue
    d = p.unsqueeze(1) - n.unsqueeze(0)
    aucs.append(float(((d > 0).double() + 0.5 * (d == 0).double()).mean()))
  return sum(aucs) / len(aucs)


def test_metrics_match_brute_force():
  g = torch.Generator().manual_seed(0)
  n, T = 300, 9
  s = torch.randint(-4, 5, (n, T), generator=g).float() / 2          # many ties, exact zeros
  y = torch.rand(n, T, generator=g) < 0.3
  y[:, 2] = True                                                     # single-class tasks are skipped
  y[:, 5] = False
  assert abs(multilabel_auc(s, y) - _brute_auc(s, y)) < 1e-12
  # a perfect ranking and a reversed one
  assert multilabel_auc(y.float(), y) == 1.0 and multilabel_auc(-y.float(), y) == 0.0
  assert math.isnan(multilabel_auc(torch.zeros(4, 1), torch.ones(4, 1, dtype=torch.bool)))   # no task has both classes
  tp = fp = fn = 0
  for i in range(n):
    for t in range(T):
      pred = float(s[i, t]) > 0
      tp += pred and bool(y[i, t])
      fp += pred and not bool(y[i, t])
      fn += (not pred) and bool(y[i, t])
  assert abs(multilabel_f1(s, y) - 2 * tp / (2 * tp + fp + fn)) < 1e-12


def _dataset(n=600, d=32, T=20):
  ei = rmat_edges(n, 3000, seed=1)
  ei = torch.cat([ei, ei.flip(0)], 1)
  x = torch.randn(n, d, generator=torch.Generator().manual_seed(2))
  y = multilabel_targets(ei, x, T, seed=3)
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CPU', directed=False, num_nodes=n)
  ds.init_node_features(x, with_gpu=False)
  return ds, x, y


def test_trainer_step_is_an_autograd_bce_step():
  ds, x, y = _dataset()
  tr = GraphSageMultiLabelTrainer(ds.graph, ds.node_features, y, in_dim=32, fanouts=[4, 3], hidden=32, lr=1e-2,
                                  weight_decay=1e-4, seed=4)
  seeds = torch.arange(0, 600, 7)
  batch = tr._batch(seeds)
  tr._batch = lambda s: batch                       # the same sampled batch for the trainer and the hand-written step
  ref = copy.deepcopy(tr.model)
  opt = torch.optim.Adam(ref.parameters(), lr=1e-2, weight_decay=1e-4)
  xb, ei, nn_, ne_, yb, n = batch
  assert torch.equal(yb, y[seeds].float())
  ref_loss = F.binary_cross_entropy_with_logits(ref(xb, ei, nn_, ne_)[:n], y[seeds].float())
  opt.zero_grad()
  ref_loss.backward()
  opt.step()
  loss = tr.train_step(seeds)
  assert torch.equal(loss, ref_loss.detach())
  for (name, a), b in zip(tr.model.named_parameters(), ref.parameters()):
    assert torch.equal(a, b), name
  l, tp, fp, fn, cnt = tr.evaluate_batch(seeds)
  logits = tr.model(xb, ei, nn_, ne_)[:n].detach()
  pred, yt = logits > 0, y[seeds]
  assert cnt == seeds.numel() and (tp, fp, fn) == (int((pred & yt).sum()), int((pred & ~yt).sum()),
                                                    int((~pred & yt).sum()))
  assert abs(l - float(F.binary_cross_entropy_with_logits(logits, yt.float()))) < 1e-6


def test_trainer_rejects_bad_labels():
  ds, x, y = _dataset()
  with pytest.raises(ValueError):
    GraphSageMultiLabelTrainer(ds.graph, ds.node_features, y.float() * 2, in_dim=32, fanouts=[4, 3], hidden=32)


def test_example_trainer_mode_prints_auc():
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  out = subprocess.run([sys.executable, 'examples/train_sage_multilabel.py', '--mode', 'trainer', '--nodes', '3000',
                        '--edges', '30000', '--epochs', '2', '--batch', '256', '--hidden', '64', '--fanouts', '5,5',
                        '--tasks', '40'], cwd=ROOT, capture_output=True, text=True, timeout=300, env=env)
  assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
  assert 'test ROC-AUC' in out.stdout
  auc = float(out.stdout.split('test ROC-AUC')[1].split()[0])
  assert 0.0 <= auc <= 1.0
