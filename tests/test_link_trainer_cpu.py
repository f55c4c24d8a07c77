"""GraphSageLinkTrainer (the CPU counterpart of GraphSageLinkEngine) and the link-prediction example."""
import copy
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageLinkTrainer, link_auc
from link_task import pair_batches, sbm_link_task

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _trainer(task, **kw):
  g = glt.data.Graph(task['topo'], 'CPU')
  return GraphSageLinkTrainer(g, task['x'], 64, fanouts=[10, 5], hidden=64, out_channels=64, **kw)


def test_link_auc_rank_statistic():
  emb = torch.tensor([[1.0], [2.0], [0.0], [-1.0]])
  assert link_auc(emb, torch.tensor([[0, 1], [1, 1]]), torch.tensor([[2, 3], [0, 0]])) == 1.0
  assert link_auc(emb, torch.tensor([[2, 3], [0, 0]]), torch.tensor([[0, 1], [1, 1]])) == 0.0
  assert link_auc(emb, torch.tensor([[2], [0]]), torch.tensor([[2], [1]])) == 0.5      # tie


def test_loss_is_bce_over_the_sampled_edge_labels():
  task = sbm_link_task(num_nodes=1024)
  tr = _trainer(task, neg_ratio=2, seed=3)
  seen = []
  sample = tr.sampler.sample_from_edges

  def spy(inputs, **kw):
    out = sample(inputs, **kw)
    seen.append(out)
    return out
  tr.sampler.sample_from_edges = spy
  before = copy.deepcopy(tr.model)
  pairs = task['train_pairs'][:, :100]
  loss = float(tr.train_step(pairs))
  out = seen[0]
  eli, y = out.metadata['edge_label_index'], out.metadata['edge_label'].float()
  assert eli.shape == (2, 300) and int(y.sum()) == 100 and bool((y[:100] == 1).all())
  # the positives are the given pairs, in order
  assert torch.equal(out.node[eli[:, :100]], pairs)
  h = before(task['x'][out.node], torch.stack([out.row, out.col]), out.num_sampled_nodes, out.num_sampled_edges)
  s = (h[eli[0]] * h[eli[1]]).sum(-1).double().detach()
  ref = -(y * F.logsigmoid(s) + (1 - y) * F.logsigmoid(-s)).mean()
  assert abs(loss - float(ref)) < 1e-5 * max(1.0, float(ref))
  assert all(not torch.equal(p0, p1) for p0, p1 in zip(before.parameters(), tr.model.parameters()))


def test_learns_the_block_graph():
  task = sbm_link_task()
  tr = _trainer(task, seed=0)
  auc0 = link_auc(tr.inference(), task['held'], task['neg'])
  for b in pair_batches(task['train_pairs'], 256, 300):
    tr.train_step(b)
  auc = link_auc(tr.inference(), task['held'], task['neg'])
  assert auc0 < 0.75 and auc >= 0.85, (auc0, auc)
  loss, correct, n = tr.evaluate_batch(task['train_pairs'][:, :256])
  assert n == 512 and correct / n > 0.65 and loss < 0.6


def test_state_dict_round_trip():
  task = sbm_link_task(num_nodes=1024)
  a = _trainer(task, seed=1)
  for b in pair_batches(task['train_pairs'], 128, 5):
    a.train_step(b)
  b_ = _trainer(task, seed=2)
  b_.load_state_dict(a.state_dict())
  assert b_.step_idx == 5 and b_.sampler.state_dict() == a.sampler.state_dict()
  assert torch.equal(a.inference(), b_.inference())
  sa, sb = a.opt.state_dict()['state'], b_.opt.state_dict()['state']
  assert all(torch.equal(sa[k]['exp_avg_sq'], sb[k]['exp_avg_sq']) for k in sa)


def test_example_engine_mode_runs_on_the_cpu_fallback():
  env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
  out = subprocess.run([sys.executable, 'examples/graph_sage_unsup.py', '--mode', 'engine', '--epochs', '1',
                        '--steps-per-epoch', '10'], cwd=ROOT, capture_output=True, text=True, timeout=600, env=env)
  assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
  assert 'epoch 0: loss' in out.stdout and 'held-out link AUC' in out.stdout
