"""GraphSageEngine.inference(): exact layer-wise full-neighbourhood inference (csrc/cuda/sage_infer.cu + TcGemm)
against fp32 PyTorch recomputations over the CSR."""
import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageEngine
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
N, N_RMAT, HUB = 6000, 5940, 11          # nodes N_RMAT..N-1 have no edges at all


def _hub_graph_edges():
  """RMAT over the first N_RMAT nodes, plus a hub row of degree 5200 (with repeated neighbours)."""
  ei = rmat_edges(N_RMAT, 60000, seed=3)
  g = torch.Generator().manual_seed(4)
  hub = torch.stack([torch.full((5200,), HUB, dtype=torch.int64), torch.randint(0, N_RMAT, (5200,), generator=g)])
  return torch.cat([ei, hub], 1)


def _graph(mode='CUDA', int64_cols=False):
  topo = glt.data.Topology(_hub_graph_edges(), layout='CSR', num_nodes=N)
  if int64_cols:
    shard = {'indptr': topo.indptr.to(DEV), 'indices': topo.indices.to(DEV, torch.int64), 'row_begin': 0, 'row_end': N}
    g = glt.data.Graph.from_shards([shard], 0)
    g._keep_shard = shard
  else:
    g = glt.data.Graph(topo, mode, 0)
  return g, topo


def _features(Fdim=128):
  torch.manual_seed(0)
  return torch.randn(N, Fdim, device=DEV).to(torch.bfloat16)


def _engine(g, table, labels, train_steps=0, **kw):
  args = dict(in_dim=128, num_nodes=N, fanouts=[5, 4, 3], batch_size=256, hidden=256, num_classes=47, device=DEV,
              use_cuda_graph=False, seed=5, lr=5e-3)
  args.update(kw)
  eng = GraphSageEngine(g, table, labels, **args)
  gen = torch.Generator(device='cpu').manual_seed(9)
  for _ in range(train_steps):
    eng.train_step(torch.randperm(N, generator=gen)[:args['batch_size']].to(DEV))
  eng.flush()
  return eng


def _seg_mean(x, indptr, indices):
  n = indptr.numel() - 1
  deg = indptr[1:] - indptr[:-1]
  dst = torch.repeat_interleave(torch.arange(n, device=x.device), deg)
  s = torch.zeros(n, x.shape[1], device=x.device).index_add_(0, dst, x[indices.long()])
  return s / deg.clamp(min=1).unsqueeze(1).float()


def _reference(eng, topo, x):
  """fp32 recomputation with the engine's rounding points: bf16 A operand (aggregate-first layers), bf16 P
  (project-first layers), bf16 activations."""
  indptr, indices = topo.indptr.to(DEV), topo.indices.to(DEV)
  H = x.float()
  for l in range(1, eng.L + 1):
    W, b = eng.W(l).float(), eng.b(l).float()
    d, n = eng.dims_in[l - 1], eng.dims_out[l - 1]
    if l >= 2 and n < d:
      P = (H @ torch.cat([W[:, :d], W[:, d:]], 0).t()).to(torch.bfloat16).float()
      Z = _seg_mean(P[:, :n], indptr, indices) + P[:, n:] + b
    else:
      A = torch.cat([_seg_mean(H, indptr, indices), H], 1).to(torch.bfloat16).float()
      Z = A @ W.t() + b
    if l < eng.L:
      Z = F.relu(Z)
    H = Z.to(torch.bfloat16).float()
  return H[:, :eng.C]


def _check_close(got, ref):
  assert got.shape == ref.shape and got.dtype == torch.bfloat16
  torch.testing.assert_close(got.float(), ref, rtol=2e-2, atol=2e-2)
  agree = (got.float().argmax(1) == ref.argmax(1)).float().mean().item()
  assert agree >= 0.99, agree


@pytest.fixture(scope='module')
def trained():
  g, topo = _graph()
  feats = _features()
  labels = torch.randint(0, 47, (N,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = _engine(g, ut._table(), labels, train_steps=5, use_fused=False)
  eng._keep = (ut, feats, topo, g)
  return eng, topo, feats


def test_inference_matches_fp32_reference_on_hub_and_isolated_nodes(native, trained):
  eng, topo, feats = trained
  deg = topo.indptr[1:] - topo.indptr[:-1]
  assert int(deg[HUB]) >= 5000 and int((deg == 0).sum()) >= 50
  assert not eng._project_first(2) and eng._project_first(3)        # both orders are exercised
  got = eng.inference()
  _check_close(got, _reference(eng, topo, feats))


def test_inference_is_deterministic_and_independent_of_chunking(native, trained):
  eng, _, _ = trained
  a = eng.inference()
  assert torch.equal(a, eng.inference())
  assert torch.equal(a, eng.inference(chunk_rows=997))


def test_inference_is_the_full_fanout_limit_of_evaluate_batch(native):
  # every node has at most 6 neighbours, so fanouts [6, 6] sample each neighbourhood whole
  gen = torch.Generator().manual_seed(5)
  n = 4000
  src = torch.arange(n).repeat_interleave(3)
  ei = torch.stack([src, torch.randint(0, n, (3 * n,), generator=gen)])
  ei = torch.unique(torch.cat([ei, ei.flip(0)], 1), dim=1)
  ei = ei[:, ei[0] != ei[1]]
  deg = torch.bincount(ei[0], minlength=n)
  ei = ei[:, (deg[ei[0]] <= 6) & (deg[ei[1]] <= 6)]
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=n)
  assert int((topo.indptr[1:] - topo.indptr[:-1]).max()) <= 6
  g = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(1)
  feats = torch.randn(n, 128, device=DEV).to(torch.bfloat16)
  labels = torch.randint(0, 47, (n,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  # hidden 64 = padded class width: both layers aggregate first, like the training forward
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=128, num_nodes=n, fanouts=[6, 6], batch_size=512, hidden=64,
                        num_classes=47, device=DEV, use_cuda_graph=False, use_fused=False, seed=2)
  full = eng.inference()
  seeds = torch.randperm(n, device=DEV)[:512]
  _, _, m = eng.evaluate_batch(seeds)
  assert m == 512
  sampled = eng.Z[eng.L][:512, :eng.C]
  torch.testing.assert_close(sampled.float(), full[seeds].float(), rtol=1e-2, atol=1e-2)


def test_inference_with_mxfp8_features_matches_dequantised_reference(native):
  from graphlearn_for_pytorch_b200.data import dequantize_mxfp8, quantize_mxfp8
  g, topo = _graph()
  torch.manual_seed(0)
  x = torch.randn(N, 128, device=DEV)
  q = quantize_mxfp8(x)
  labels = torch.randint(0, 47, (N,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.uint8)
  ut.append_shared_tensor(q)
  eng = _engine(g, ut._table(), labels, train_steps=3, feature_format='mxfp8')
  _check_close(eng.inference(), _reference(eng, topo, dequantize_mxfp8(q, 128)))


def test_inference_is_identical_across_memory_tiers_and_column_id_widths(native):
  feats = _features()
  labels = torch.randint(0, 47, (N,), device=DEV)
  g_hbm, _ = _graph('CUDA')
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  ref = _engine(g_hbm, ut._table(), labels).inference()
  g_zc, _ = _graph('ZERO_COPY')
  g_i64, _ = _graph(int64_cols=True)
  split = glt.data.UnifiedTensor(0, torch.bfloat16)
  split.append_shared_tensor(feats[:N // 3])
  split.append_cpu_tensor(feats[N // 3:].cpu())
  for g, table in ((g_zc, split._table()), (g_i64, ut._table()), (g_zc, ut._table())):
    assert torch.equal(_engine(g, table, labels).inference(), ref)


def test_inference_leaves_a_pipelined_captured_engine_untouched(native):
  g, _ = _graph()
  feats = _features()
  labels = torch.randint(0, 47, (N,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=128, num_nodes=N, fanouts=[5, 4, 3], batch_size=256,
                        hidden=256, num_classes=47, device=DEV, use_cuda_graph=True, pipeline=True, seed=5)
  eng.warmup_and_capture(n_eager=1)
  gen = torch.Generator(device='cpu').manual_seed(3)
  for _ in range(4):
    eng.train_step(torch.randperm(N, generator=gen)[:256].to(DEV))
  torch.cuda.synchronize()
  snap = {'p32': eng.p32.clone(), 'p16': eng.p16.clone(), 'm': eng.m.clone(), 'v': eng.v.clone(),
          'step_dev': eng.step_dev.clone(), 'g32': [g_.clone() for g_ in eng._g]}
  steps = [a.step.clone() for a in eng._arenas]
  graphs = list(eng._graphs)
  eng.inference()
  torch.cuda.synchronize()
  for k in ('p32', 'p16', 'm', 'v', 'step_dev'):
    assert torch.equal(getattr(eng, k), snap[k]), k
  assert all(torch.equal(a, b) for a, b in zip(eng._g, snap['g32']))
  assert all(torch.equal(a.step, s) for a, s in zip(eng._arenas, steps))
  assert eng._graphs == graphs
  loss = eng.train_step(torch.randperm(N, generator=gen)[:256].to(DEV))
  assert torch.isfinite(loss).all()


@pytest.mark.parametrize('d', [64, 128, 256, 512])
@pytest.mark.parametrize('combine', [False, True])
def test_full_aggregate_kernel_modes_against_torch(native, d, combine):
  g, topo = _graph()
  indptr, indices = topo.indptr.to(DEV), topo.indices.to(DEV)
  torch.manual_seed(d)
  width = 2 * d if combine else d + 64
  src = torch.randn(N, width, device=DEV).to(torch.bfloat16)
  src_col, self_col = (0, d) if combine else (64, 64)
  bias = torch.randn(d, device=DEV).to(torch.bfloat16)
  r0, r1 = 5, N - 3                           # the hub (row 11) and the isolated tail are inside
  out = torch.full((r1 - r0, d if combine else 2 * d), float('nan'), device=DEV, dtype=torch.bfloat16)
  native.sage_full_aggregate(g.graph_handler, None, src, src_col, self_col, d, r0, r1, combine,
                             bias if combine else None, combine, out)
  mean = _seg_mean(src[:, src_col:src_col + d].float(), indptr, indices)[r0:r1]
  self_ = src[r0:r1, self_col:self_col + d]
  if combine:
    ref = F.relu(mean + self_.float() + bias.float())
    torch.testing.assert_close(out.float(), ref, rtol=1e-2, atol=1e-2)
  else:
    torch.testing.assert_close(out[:, :d].float(), mean, rtol=1e-2, atol=1e-2)
    assert torch.equal(out[:, d:], self_)
    assert (out[N_RMAT - r0:, :d] == 0).all()          # degree 0 -> mean 0
  again = torch.empty_like(out)
  native.sage_full_aggregate(g.graph_handler, None, src, src_col, self_col, d, r0, r1, combine,
                             bias if combine else None, combine, again)
  assert torch.equal(out, again)
