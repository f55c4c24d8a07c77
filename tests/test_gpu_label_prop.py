"""The label-propagation kernel (csrc/cuda/label_prop.cu) and LabelPropagation / CorrectAndSmooth on device graphs,
against the float64 transcriptions of PyG's semantics in test_label_prop_cpu.py, at every lane shape of the kernel, on
both sides of the hub threshold and on every graph layout the inference kernels read."""
import math

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import CorrectAndSmooth, GraphSageEngine, LabelPropagation
from graphlearn_for_pytorch_b200.models.label_prop import propagate
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges

from test_label_prop_cpu import ref_correct, ref_lp, ref_propagate, ref_smooth

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
N, N_RMAT = 3000, 2880                 # rows N_RMAT..2899 and the last rows have no entries
# every lane shape of the ladder (C / 4 vectors, LPR 1 .. 32, VPL 1, 2, 4), with and without padding
CLASSES = [1, 3, 4, 5, 8, 16, 17, 40, 47, 112, 128, 129, 172, 256, 349, 512]


def _csr():
  """(indptr, indices int64) over N rows: RMAT rows, rows of degree 256 (2900) and 257 (2901), a degree-5000 hub with
  repeats (2902), four hubs of degree 300 in one CTA at every lane shape (2904..2907), self-loops, a duplicate edge,
  and column ids outside [0, N) (row 5: N + 7 and -1)."""
  g = torch.Generator().manual_seed(11)
  ei = rmat_edges(N_RMAT, 30000, seed=7)
  extra = [(2900, torch.randint(0, N, (256,), generator=g)), (2901, torch.randint(0, N, (257,), generator=g)),
           (2902, torch.randint(0, N_RMAT, (5000,), generator=g))]
  extra += [(r, torch.randint(0, N, (300,), generator=g)) for r in range(2904, 2908)]
  extra += [(7, torch.tensor([7, 7, 3, 3])), (5, torch.tensor([N + 7, -1, 2]))]
  rows = torch.cat([ei[0]] + [torch.full((c.numel(),), r) for r, c in extra])
  cols = torch.cat([ei[1]] + [c for _, c in extra])
  order = torch.argsort(rows, stable=True)
  rows, cols = rows[order], cols[order]
  indptr = torch.zeros(N + 1, dtype=torch.int64)
  indptr[1:] = torch.cumsum(torch.bincount(rows, minlength=N), 0)
  return indptr, cols


def _coo(indptr, indices):
  return torch.repeat_interleave(torch.arange(N), indptr[1:] - indptr[:-1]).to(DEV), indices.to(DEV, torch.int64)


def _graph(layout):
  """A device Graph over the CSR of _csr() (int32 / int64 columns, two shards on one device, pinned host)."""
  indptr, indices = _csr()
  if layout == 'int32':
    shards = [{'indptr': indptr.to(DEV), 'indices': indices.to(DEV, torch.int32), 'row_begin': 0, 'row_end': N}]
  elif layout == 'int64':
    shards = [{'indptr': indptr.to(DEV), 'indices': indices.to(DEV), 'row_begin': 0, 'row_end': N}]
  elif layout == 'two_shards':
    h = 2903                     # the degree-5000 hub ends shard 0, the hub CTA starts shard 1
    shards = [{'indptr': indptr[:h + 1].to(DEV), 'indices': indices[:indptr[h]].to(DEV), 'row_begin': 0, 'row_end': h},
              {'indptr': (indptr[h:] - indptr[h]).to(DEV), 'indices': indices[indptr[h]:].to(DEV),
               'row_begin': h, 'row_end': N}]
  else:                          # zero_copy: the CSR read in place from pinned host memory
    shards = [{'indptr': indptr.pin_memory(), 'indices': indices.to(torch.int32).pin_memory(), 'row_begin': 0,
               'row_end': N}]
  graph = glt.data.Graph.from_shards(shards, 0)
  graph._keep_shards = shards
  return graph, _coo(indptr, indices)


@pytest.fixture(scope='module')
def graphs():
  return {k: _graph(k) for k in ('int32', 'int64', 'two_shards', 'zero_copy')}


def _check(got, ref):
  err = float((got.double() - ref).abs().max())
  assert err <= 1e-4 * max(1.0, float(ref.abs().max())), err


def test_graph_covers_the_hub_boundary():
  indptr, indices = _csr()
  deg = indptr[1:] - indptr[:-1]
  assert int(deg[2900]) == 256 and int(deg[2901]) == 257 and int(deg[2902]) == 5000
  assert all(int(deg[r]) > 256 for r in range(2904, 2908)) and int((deg == 0).sum()) >= 50
  assert int(((indices < 0) | (indices >= N)).sum()) == 2


@pytest.mark.parametrize('norm', ['sym', 'row'])
@pytest.mark.parametrize('C', CLASSES)
def test_kernel_against_float64(native, graphs, C, norm):
  graph, (rows, cols) = graphs['int32']
  cp = (C + 3) // 4 * 4
  gen = torch.Generator(device=DEV).manual_seed(C)
  base = torch.zeros(N, cp, device=DEV)
  base[:, :C] = torch.rand(N, C, device=DEV, generator=gen) * 2 - 1
  fixed = torch.rand(N, device=DEV, generator=gen) < 0.3
  for layers in (1, 50):
    for alpha in (0.0, 0.8, 1.0):
      for post in ('clamp', 'fixed'):
        lo, hi = (-0.5, 0.75) if post == 'clamp' else (-math.inf, math.inf)
        fx = fixed if post == 'fixed' else None
        got = native.label_prop(graph.graph_handler, base, C, layers, alpha, norm, lo, hi, fx)
        ref = ref_propagate(N, rows, cols, base[:, :C], layers, alpha, norm,
                            clamp=(lo, hi) if post == 'clamp' else None, fixed=fx)
        _check(got[:, :C], ref)
        assert got.shape == (N, cp) and not got[:, C:].any(), 'padding columns must stay 0'
        if layers == 50 and alpha == 0.8:
          assert torch.equal(got, native.label_prop(graph.graph_handler, base, C, layers, alpha, norm, lo, hi, fx))


@pytest.mark.parametrize('layout', ['int64', 'two_shards', 'zero_copy'])
@pytest.mark.parametrize('C', [5, 47, 349])
def test_every_graph_layout_gives_the_int32_result(native, graphs, layout, C):
  """Same CSR, same rows: the same reduction order, so the same bits."""
  g32, (rows, cols) = graphs['int32']
  graph, _ = graphs[layout]
  gen = torch.Generator(device=DEV).manual_seed(1)
  base = torch.zeros(N, (C + 3) // 4 * 4, device=DEV)
  base[:, :C] = torch.rand(N, C, device=DEV, generator=gen)
  for norm in ('sym', 'row'):
    ref = native.label_prop(g32.graph_handler, base, C, 50, 0.8, norm, 0.0, 1.0)
    got = native.label_prop(graph.graph_handler, base, C, 50, 0.8, norm, 0.0, 1.0)
    _check(got[:, :C], ref_propagate(N, rows, cols, base[:, :C], 50, 0.8, norm, clamp=(0., 1.)))
    assert torch.equal(got, ref)


def test_directed_orientation(native):
  """Row i receives from the columns of row i: the kernel follows the CSR, not its transpose."""
  ei = torch.tensor([[0, 0, 1, 2, 2, 3], [1, 2, 2, 0, 3, 3]])
  for e in (ei, ei.flip(0)):
    topo = glt.data.Topology(e, layout='CSR', num_nodes=5)
    graph = glt.data.Graph(topo, 'CUDA', 0)
    rows = torch.repeat_interleave(torch.arange(5), topo.indptr[1:] - topo.indptr[:-1]).to(DEV)
    y = torch.tensor([0, 1, 2, 0, 1])
    _check(LabelPropagation(3, 0.8)(y, graph), ref_lp(5, rows, topo.indices.to(DEV), y.to(DEV), 3, 0.8, 'sym'))
  a = LabelPropagation(3, 0.8)(y, glt.data.Graph(glt.data.Topology(ei, layout='CSR', num_nodes=5), 'CUDA', 0))
  b = LabelPropagation(3, 0.8)(y, glt.data.Graph(glt.data.Topology(ei.flip(0), layout='CSR', num_nodes=5), 'CUDA', 0))
  assert (a - b).abs().max() > 1e-2


def _topo_pair():
  """The same RMAT topology as a 'CUDA', a 'ZERO_COPY' and a 'CPU' Graph."""
  ei = rmat_edges(2000, 16000, seed=3)
  ei = torch.cat([ei, ei.flip(0)], 1)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=2048)
  rows = torch.repeat_interleave(torch.arange(2048), topo.indptr[1:] - topo.indptr[:-1]).to(DEV)
  return (glt.data.Graph(topo, 'CUDA', 0), glt.data.Graph(topo, 'ZERO_COPY', 0), glt.data.Graph(topo, 'CPU'),
          rows, topo.indices.to(DEV, torch.int64))


@pytest.mark.parametrize('norm', ['sym', 'row'])
def test_label_propagation_gpu_and_cpu_paths(native, norm):
  gpu, zc, cpu, rows, cols = _topo_pair()
  gen = torch.Generator().manual_seed(0)
  y = torch.randint(0, 47, (2048,), generator=gen)
  mask = torch.rand(2048, generator=gen) < 0.4
  lp = LabelPropagation(50, 0.9, norm)
  ref = ref_lp(2048, rows, cols, y.to(DEV), 50, 0.9, norm, mask.to(DEV))
  got = lp(y, gpu, mask)
  assert got.device == DEV and got.dtype == torch.float32
  _check(got, ref)
  _check(lp(y, zc, mask.nonzero().view(-1)), ref)
  on_cpu = lp(y, cpu, mask)
  assert on_cpu.device.type == 'cpu'
  _check(got.cpu(), on_cpu.double())


@pytest.mark.parametrize('autoscale', [True, False])
def test_correct_and_smooth_against_float64_and_cpu(native, autoscale):
  gpu, zc, cpu, rows, cols = _topo_pair()
  n, C = 2048, 47
  gen = torch.Generator().manual_seed(1)
  y_soft = torch.randn(n, C, generator=gen).softmax(-1)
  mask = torch.rand(n, generator=gen) < 0.2
  y_true = torch.randint(0, C, (int(mask.sum()),), generator=gen)
  cs = CorrectAndSmooth(50, 0.9, 50, 0.8, autoscale=autoscale, scale=20.0)
  d = lambda t: t.to(DEV)
  for norm in ('sym', 'row'):
    ref_c = ref_correct(n, rows, cols, d(y_soft), d(y_true), d(mask), 50, 0.9, autoscale, 20.0, norm)
    corr = cs.correct(y_soft, y_true, mask, gpu, norm=norm)
    _check(corr, ref_c)
    _check(corr.cpu(), cs.correct(y_soft, y_true, mask, cpu, norm=norm).double())
    sm = cs.smooth(corr, y_true, mask, gpu, norm=norm)
    _check(sm, ref_smooth(n, rows, cols, corr, d(y_true), d(mask), 50, 0.8, norm))
    _check(sm.cpu(), cs.smooth(corr.cpu(), y_true, mask, cpu, norm=norm).double())


def test_products_recipe_sym_then_row(native):
  gpu, _, cpu, rows, cols = _topo_pair()
  n, C = 2048, 47
  gen = torch.Generator().manual_seed(2)
  y_soft = torch.randn(n, C, generator=gen).softmax(-1)
  idx = torch.randperm(n, generator=gen)[:300]
  y_true = torch.randint(0, C, (300,), generator=gen)
  cs = CorrectAndSmooth(50, 1.0, 50, 0.8, autoscale=False, scale=20.0)
  got = cs.smooth(cs.correct(y_soft, y_true, idx, gpu, norm='sym'), y_true, idx, gpu, norm='row')
  ref = ref_correct(n, rows, cols, y_soft.to(DEV), y_true.to(DEV), idx.to(DEV), 50, 1.0, False, 20.0, 'sym')
  _check(got, ref_smooth(n, rows, cols, ref.float(), y_true.to(DEV), idx.to(DEV), 50, 0.8, 'row'))
  on_cpu = cs.smooth(cs.correct(y_soft, y_true, idx, cpu, norm='sym'), y_true, idx, cpu, norm='row')
  _check(got.cpu(), on_cpu.double())


def test_engine_state_is_untouched(native):
  """C&S on a trained GraphSageEngine's inference() output changes no engine state, and the next step's loss is the
  loss of the same step without it."""
  ei = rmat_edges(3000, 30000, seed=4)
  topo = glt.data.Topology(torch.cat([ei, ei.flip(0)], 1), layout='CSR', num_nodes=3000)
  graph = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(0)
  feats = torch.randn(3000, 128, device=DEV).to(torch.bfloat16)
  labels = torch.randint(0, 47, (3000,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageEngine(graph, ut._table(), labels, in_dim=128, num_nodes=3000, fanouts=[5, 4, 3], batch_size=256,
                        hidden=256, num_classes=47, device=DEV, use_cuda_graph=False, seed=5,
                        deterministic_sampling=True)
  gen = torch.Generator(device='cpu').manual_seed(9)
  for _ in range(3):
    eng.train_step(torch.randperm(3000, generator=gen)[:256].to(DEV))
  eng.flush()
  torch.cuda.synchronize()
  snap = eng.state_dict()
  extra = {'p16': eng.p16.clone(), 'step_dev': eng.step_dev.clone()}
  y_soft = eng.inference().float().softmax(-1)
  train = torch.arange(0, 3000, 3, device=DEV)
  LabelPropagation(10, 0.9)(labels, graph, train)
  cs = CorrectAndSmooth(10, 1.0, 10, 0.8, autoscale=False, scale=20.0)
  cs.smooth(cs.correct(y_soft, labels[train], train, graph), labels[train], train, graph, norm='row')
  CorrectAndSmooth(10, 1.0, 10, 0.8).correct(y_soft, labels[train], train, graph)
  torch.cuda.synchronize()
  after = eng.state_dict()
  for k in ('p32', 'm', 'v'):
    assert torch.equal(after[k], snap[k]), k
  assert after['step'] == snap['step'] and after['sample_step'] == snap['sample_step']
  assert after['step_idx'] == snap['step_idx']
  assert torch.equal(eng.p16, extra['p16']) and torch.equal(eng.step_dev, extra['step_dev'])
  seeds = torch.randperm(3000, generator=gen)[:256].to(DEV)
  loss_after = float(eng.train_step(seeds))
  eng.flush()
  eng.load_state_dict(snap)
  loss_without = float(eng.train_step(seeds))
  assert abs(loss_after - loss_without) <= 1e-6 * max(1.0, abs(loss_without)), (loss_after, loss_without)


def test_argument_errors(native, graphs):
  graph, _ = graphs['int32']
  gh = graph.graph_handler
  ok = torch.zeros(N, 48, device=DEV)
  native.label_prop(gh, ok, 47, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):                           # C = 513
    native.label_prop(gh, torch.zeros(N, 516, device=DEV), 513, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):
    propagate(graph, torch.zeros(N, 513, device=DEV), 1, 0.5)
  with pytest.raises(RuntimeError):                           # dtype
    native.label_prop(gh, ok.double(), 47, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):                           # pitch is not C rounded up to 4
    native.label_prop(gh, torch.zeros(N, 47, device=DEV), 47, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):                           # contiguity
    native.label_prop(gh, torch.zeros(48, N, device=DEV).t(), 47, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):                           # row count
    native.label_prop(gh, torch.zeros(N - 1, 48, device=DEV), 47, 1, 0.5, 'sym', 0.0, 1.0)
  with pytest.raises(ValueError):
    propagate(graph, torch.zeros(N + 1, 4, device=DEV), 1, 0.5)
  with pytest.raises(RuntimeError):                           # mask length
    native.label_prop(gh, ok, 47, 1, 0.5, 'sym', 0.0, 1.0, torch.ones(N + 1, dtype=torch.bool, device=DEV))
  with pytest.raises(ValueError):
    LabelPropagation(2, 0.5)(torch.zeros(N, 3), graph, torch.ones(N - 1, dtype=torch.bool))
  with pytest.raises(RuntimeError):                           # norm, alpha, num_layers
    native.label_prop(gh, ok, 47, 1, 0.5, 'col', 0.0, 1.0)
  with pytest.raises(ValueError):
    LabelPropagation(2, 0.5, norm='col')
  with pytest.raises(RuntimeError):
    native.label_prop(gh, ok, 47, 1, math.inf, 'sym', 0.0, 1.0)
  with pytest.raises(RuntimeError):
    native.label_prop(gh, ok, 47, -1, 0.5, 'sym', 0.0, 1.0)
  native.label_prop(gh, ok, 47, 1, 0.5, 'sym', 0.0, 1.0)      # the process is still healthy
  torch.cuda.synchronize()
