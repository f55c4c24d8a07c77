"""KgeEngine without a GPU: constructor argument errors, kge_filter keys, synthetic_kg, and the example's argument
parsing and triple reader."""
import importlib.util
import os

import pytest
import torch

from graphlearn_for_pytorch_b200.models import KgeEngine, kge_filter
from graphlearn_for_pytorch_b200.utils.synthetic import synthetic_kg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('kw', [
  dict(model='transR'),
  dict(hidden_channels=12), dict(hidden_channels=0), dict(hidden_channels=520),
  dict(p_norm=3.0), dict(p_norm=0.5),
  dict(num_negatives=0), dict(batch_size=0), dict(lr=0.0), dict(lr=-1.0),
  dict(num_nodes=0), dict(num_nodes=2 ** 31), dict(num_relations=0), dict(num_relations=2 ** 31),
  dict(margin=float('nan')),
])
def test_constructor_errors(kw):
  args = dict(num_nodes=10, num_relations=3)
  args.update(kw)
  with pytest.raises(ValueError):
    KgeEngine(**args)


def test_filter_keys():
  N, R = 7, 3
  trip = torch.tensor([[1, 4, 1, 6, 1], [2, 0, 2, 1, 0], [5, 3, 5, 0, 2]])   # (1, 2, 5) twice
  tail, head = kge_filter(trip, N, R)
  h, r, t = trip
  assert torch.equal(tail, torch.sort((h * R + r) * N + t).values)
  assert torch.equal(head, torch.sort((t * R + r) * N + h).values)
  assert tail.numel() == head.numel() == 5                         # duplicates kept
  assert torch.all(tail[1:] >= tail[:-1]) and torch.all(head[1:] >= head[:-1])
  # the tails known for (1, 2, ?) are one contiguous range
  base = (1 * R + 2) * N
  sel = tail[(tail >= base) & (tail < base + N)] - base
  assert sel.tolist() == [5, 5]
  base = (3 * R + 0) * N
  assert (head[(head >= base) & (head < base + N)] - base).tolist() == [4]


def test_filter_errors():
  with pytest.raises(ValueError):
    kge_filter(torch.zeros(3, 1, dtype=torch.int64), 2 ** 31, 2 ** 2)       # N^2 R >= 2^63
  with pytest.raises(ValueError):
    kge_filter(torch.zeros(2, 1, dtype=torch.int64), 5, 2)
  with pytest.raises(ValueError):
    kge_filter(torch.zeros(3, 1, dtype=torch.int32), 5, 2)
  with pytest.raises(ValueError):
    kge_filter(torch.tensor([[0], [2], [0]]), 5, 2)                          # relation out of range
  assert kge_filter(torch.zeros(3, 0, dtype=torch.int64), 5, 2)[0].numel() == 0


def test_synthetic_kg_structure():
  N, R = 400, 5
  a = synthetic_kg(N, R, 5000, seed=3)
  b = synthetic_kg(N, R, 5000, seed=3)
  c = synthetic_kg(N, R, 5000, seed=4)
  assert all(torch.equal(x, y) for x, y in zip(a, b))
  assert not torch.equal(a[0], c[0])
  allt = torch.cat(a, 1)
  assert allt.dtype == torch.int64 and allt.size(0) == 3
  assert torch.unique(allt, dim=1).size(1) == allt.size(1)               # distinct
  h, r, t = allt
  assert ((r >= 0) & (r < R)).all() and ((h >= 0) & (h < N)).all() and ((t >= 0) & (t < N)).all()
  assert torch.equal(t // 8, h // 8 + r + 1)                               # cluster c -> c + r + 1
  m = allt.size(1)
  assert a[0].size(1) == int(0.8 * m) and a[1].size(1) == int(0.9 * m) - int(0.8 * m)
  with pytest.raises(ValueError):
    synthetic_kg(40, 5, 100)                                              # 5 clusters cannot hold 5 relations


def _example():
  spec = importlib.util.spec_from_file_location('kge_example', os.path.join(ROOT, 'examples', 'kge.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def test_example_args_and_reader(tmp_path):
  ex = _example()
  a = ex.parse_args(['--model', 'complex', '--root', str(tmp_path), '--epochs', '3'])
  assert (a.model, a.root, a.epochs, a.margin) == ('complex', str(tmp_path), 3, None)
  assert ex.parse_args([]).model == 'transe'
  with pytest.raises(SystemExit):
    ex.parse_args(['--model', 'transh'])
  (tmp_path / 'train.txt').write_text('/m/a\t/r/x\t/m/b\n/m/b\t/r/y\t/m/c\n\n')
  (tmp_path / 'valid.txt').write_text('/m/c\t/r/x\t/m/a\n')
  (tmp_path / 'test.txt').write_text('/m/d\t/r/y\t/m/a\n')
  splits, ents, rels = ex.read_kg(str(tmp_path))
  assert ents == {'/m/a': 0, '/m/b': 1, '/m/c': 2, '/m/d': 3} and rels == {'/r/x': 0, '/r/y': 1}
  assert splits['train'].tolist() == [[0, 1], [0, 1], [1, 2]]
  assert splits['valid'].tolist() == [[2], [0], [0]]
  assert splits['test'].tolist() == [[3], [1], [0]]
  (tmp_path / 'test.txt').write_text('/m/d /r/y /m/a\n')
  with pytest.raises(ValueError):
    ex.read_kg(str(tmp_path))
