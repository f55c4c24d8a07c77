"""`kernels_per_step` of the training engines: the kernel, memset and memcpy nodes of the captured step, counted by
`graph_node_counts` on the graph itself rather than tallied by the Python step code."""
import collections
import re

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageEngine
from helpers import rmat_csr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _sage(graph, pipeline, N=6000, E=120000, Fdim=128, C=47):
  """A small GraphSageEngine with the unfused layer 1 (pre-aggregated on the sampling stream when pipelined)."""
  _, topo = rmat_csr(N, E, seed=3)
  g = glt.data.Graph(topo, 'CUDA', 0)
  gen = torch.Generator(device=DEV).manual_seed(0)
  feats = torch.randn(N, Fdim, device=DEV, generator=gen).to(torch.bfloat16)
  labels = torch.randint(0, C, (N,), device=DEV, generator=gen)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=Fdim, num_nodes=N, fanouts=[5, 4, 3], batch_size=256,
                        hidden=128, num_classes=C, device=DEV, use_fused=False, use_cuda_graph=graph, pipeline=pipeline)
  eng._keep = (ut, feats, topo)
  return eng


def test_graph_node_counts_of_a_known_graph(native):
  ctr = torch.tensor([0, 10, 0, 0], dtype=torch.int32, device=DEV)
  logits = torch.zeros(16, 64, dtype=torch.bfloat16, device=DEV)
  dlogits, y = logits.clone(), torch.zeros(16, dtype=torch.int64, device=DEV)
  loss, correct, colsum = (torch.zeros(1, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV),
                           torch.zeros(64, device=DEV))
  a = torch.zeros(1024, device=DEV)
  b = torch.empty_like(a)
  g = torch.cuda.CUDAGraph(keep_graph=True)
  with torch.cuda.graph(g):
    # not prezeroed: memsets of the bias gradient, the loss and #correct, then the loss kernel
    native.softmax_nll(logits, 47, y, None, None, ctr, loss, dlogits, correct, colsum, False)
    b.copy_(a)                                  # one device-to-device memcpy
    a.add_(1.0)                                 # one elementwise kernel
  assert tuple(native.graph_node_counts(g.raw_cuda_graph())) == (2, 3, 1)
  with pytest.raises(RuntimeError):
    native.graph_node_counts(0)


@pytest.mark.parametrize('pipeline', [False, True])
def test_graph_and_eager_engines_count_the_same(native, pipeline):
  counts = []
  for graph in (True, False):
    eng = _sage(graph, pipeline)
    eng.warmup_and_capture()
    assert bool(eng._graphs) == graph
    counts.append(eng.kernels_per_step)
  assert counts[0] == counts[1] > 0, counts


def test_hetero_graph_and_eager_engines_count_the_same(native):
  from test_gpu_hetero_engine import _build
  counts = []
  for graph in (True, False):
    eng = _build(use_graph=graph)[0]
    eng.warmup_and_capture()
    assert (eng._graph is not None) == graph
    counts.append(eng.kernels_per_step)
  assert counts[0] == counts[1] > 0, counts


def test_pipelined_parities_count_the_same(native):
  eng = _sage(True, True)
  eng.warmup_and_capture()
  counts = [sum(native.graph_node_counts(g.raw_cuda_graph())) for g in eng._graphs]
  assert counts == [eng.kernels_per_step] * 2, (counts, eng.kernels_per_step)


@pytest.mark.parametrize('pipeline', [False, True])
def test_count_matches_the_dot_dump(native, tmp_path, pipeline):
  eng = _sage(True, pipeline)
  eng.warmup_and_capture()
  path = tmp_path / 'step.dot'
  eng._graphs[0].debug_dump(str(path))
  types = collections.Counter(re.findall(r'label="\{?\s*([A-Z_]+)\b', path.read_text()))
  assert types['KERNEL'] + types['MEMSET'] + types['MEMCPY'] == eng.kernels_per_step > 0, (types, eng.kernels_per_step)
