"""Layer-1 pre-aggregation on the sampling stream (GraphSageEngine(preaggregate_layer1=...)) and the ticketed tile
claiming of the wgmma GEMM kernel (csrc/cuda/tc_gemm.cu).

Pre-aggregation moves the same deterministic aggregation kernel, on the same inputs, from the head of the training
chain to the end of the sampling of the batch, so the forward is bitwise unchanged; what differs between two engines
is only the arrival order of fp32 atomics (the loss sum, bias-gradient column sums, split-K weight gradients) and of
the transposed adjacency that the gather backward sums over."""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageEngine
from helpers import bound_ratio, gemm_bound, rmat_csr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _task(N=8000, E=100000, C=8):
  """A learnable task: labels are a linear function of the features."""
  ei, topo = rmat_csr(N, E, seed=3)
  g = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(0)
  feats = torch.randn(N, 128, device=DEV).to(torch.bfloat16)
  labels = (feats.float() @ torch.randn(128, C, device=DEV)).argmax(1)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  return g, ut, feats, labels, (topo,)


def _engine(task, preagg, fan=(4, 3), bs=512, C=8, **kw):
  g, ut, feats, labels, keep = task
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=128, num_nodes=feats.shape[0], fanouts=list(fan),
                        batch_size=bs, hidden=256, num_classes=C, device=DEV, seed=5, pipeline=True,
                        use_fused=False, deterministic_sampling=True, preaggregate_layer1=preagg, **kw)
  eng._keep = (ut, feats, keep)
  return eng


def test_preaggregate_applies_to_pipelined_unfused_layer1_only(native):
  task = _task()
  assert _engine(task, None).preaggregate
  assert not _engine(task, False).preaggregate
  g, ut, feats, labels, _ = task
  common = dict(in_dim=128, num_nodes=8000, fanouts=[4, 3], batch_size=512, hidden=256, num_classes=8, device=DEV)
  assert not GraphSageEngine(g, ut._table(), labels, use_fused=False, pipeline=False, **common).preaggregate
  assert not GraphSageEngine(g, ut._table(), labels, use_fused=True, pipeline=True, **common).preaggregate


def test_sample_writes_the_layer1_aggregate_of_its_arena(native):
  """_sample(which) on a side stream leaves in A1[which] exactly what the aggregation kernel computes on the main
  stream over the same arena."""
  eng = _engine(_task(), None, fan=(5, 4, 3), bs=256)
  assert eng.preaggregate and eng._A1[0].data_ptr() != eng._A1[1].data_ptr()
  for which in (0, 1):
    eng._seeds[which].copy_(torch.randperm(8000, device=DEV)[:256])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
      eng._sample(which)
    torch.cuda.current_stream().wait_stream(side)
    ar = eng._arenas[which]
    ref = torch.full_like(eng._A1[which], 7.0)
    native.sage_aggregate(eng.feat, ar.nodes, None, 128, ar.counters, eng.L, list(ar.ell[:eng.L]),
                          eng.fanouts[:eng.L], ar.deg, ref)
    torch.cuda.synchronize()
    T = int(ar.counters[eng.L].item())
    assert T > 256
    assert torch.equal(eng._A(1, which)[:T], ref[:T])


def test_first_step_and_gradients_match_without_preaggregation(native):
  task = _task()
  engs = [_engine(task, on, use_cuda_graph=False) for on in (True, False)]
  assert engs[0].preaggregate and not engs[1].preaggregate
  torch.manual_seed(1)
  batches = [torch.randperm(8000, device=DEV)[:512] for _ in range(2)]
  for e in engs:
    assert e.train_step(batches[0]) is None           # priming call: samples batch 0
    e.train_step(batches[1])                          # trains batch 0 || samples batch 1
  torch.cuda.synchronize()
  on, off = engs
  T = int(on._arenas[0].counters[on.L].item())
  assert int(off._arenas[0].counters[off.L].item()) == T
  assert torch.equal(on._A(1, 0)[:T], off._A(1, 0)[:T])
  n_seeds = int(on._arenas[0].counters[1].item())
  # the forward is bitwise identical; the loss is a sum of per-row fp32 atomics (order varies run to run)
  assert torch.equal(on.Z[on.L][:n_seeds], off.Z[off.L][:n_seeds])
  assert torch.equal(on.dPre[on.L][:n_seeds], off.dPre[off.L][:n_seeds])
  l_on, l_off = float(on.loss.item()), float(off.loss.item())
  assert abs(l_on - l_off) <= 1e-5 * abs(l_off), (l_on, l_off)
  # gradients: split-K red.add and bias column sums in fp32 atomic order.  Below the last layer, dPre also follows the
  # gather backward's summation order, which is the arrival order of the transposed adjacency's fill: a few of its bf16
  # elements can round differently in two runs, and what they contribute to dW = dPre^T A and db = colsum(dPre) is
  # measured and allowed on top of the atomic-order bound.
  for l in range(1, on.L + 1):
    T_l = int(on._arenas[0].counters[on.L - l + 1].item())
    ddp = (on.dPre[l][:T_l].float() - off.dPre[l][:T_l].float()).abs()
    off_w, n, k = on._w_off[l - 1]
    a, b = on.g32[off_w:off_w + n * k].view(n, k), off.g32[off_w:off_w + n * k].view(n, k)
    slack = ddp.t() @ off._A(l, 0)[:T_l].float().abs()
    assert bool(((a - b).abs() <= 1e-4 * float(b.abs().max()) + 1.01 * slack).all()), f'dW{l}'
    boff, nb = on._b_off[l - 1]
    a, b = on.g32[boff:boff + nb], off.g32[boff:boff + nb]
    assert bool(((a - b).abs() <= 1e-4 * float(b.abs().max()) + 1.01 * ddp.sum(0)).all()), f'db{l}'
  assert torch.equal(on.step_dev, off.step_dev)


def test_graph_training_matches_and_learns_with_preaggregation(native):
  """30 CUDA-graph steps + flush(): the two schedules give the same losses up to the drift that fp32 atomic order
  causes through Adam (rel. 5e-2 per step), training learns, and evaluation after flush() works."""
  task = _task()
  torch.manual_seed(2)
  batches = [torch.randperm(8000, device=DEV)[:512] for _ in range(31)]
  losses = {}
  for on in (True, False):
    eng = _engine(task, on)
    eng.warmup_and_capture(n_eager=1)
    assert eng.preaggregate == on and eng.kernels_per_step > 0
    ls = []
    for i, s in enumerate(batches):
      loss = eng.train_step(s)
      assert (loss is None) == (i == 0)
      if loss is not None:
        ls.append(float(loss.item()))
    ls.append(float(eng.flush().item()))
    assert eng.flush() is None
    losses[on] = ls
    loss, correct, n = eng.evaluate_batch(torch.randperm(8000, device=DEV)[:512])
    assert n == 512 and loss == loss and correct / n > 0.2, (loss, correct)
    if on:
      kernels_on = eng.kernels_per_step
    else:
      assert eng.kernels_per_step == kernels_on
  a, b = losses[True], losses[False]
  assert len(a) == 31
  for i, (x, y) in enumerate(zip(a, b)):
    assert abs(x - y) <= 5e-2 * max(1.0, abs(y)), (i, x, y)
  assert sum(a[-5:]) / 5 < 0.8 * a[0], (a[0], a[-5:])


def test_preaggregation_survives_regrow(native):
  """An under-calibrated arena regrows (buffers, both layer-1 A buffers, CUDA graphs rebuilt); training and
  evaluate_batch keep working with pre-aggregation on."""
  N = 20000
  ei, topo = rmat_csr(N, 600000, seed=4)
  g = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(0)
  feats = torch.randn(N, 128, device=DEV).to(torch.bfloat16)
  labels = torch.randint(0, 47, (N,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  pool = torch.randperm(N)
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=128, num_nodes=N, fanouts=[8, 6, 4], batch_size=512,
                        hidden=256, num_classes=47, device=DEV, use_cuda_graph=True, seed=5, pipeline=True,
                        use_fused=False, calibration_seeds=pool, calibration_margin=0.35, check_every=4)
  eng._keep = (ut, feats, topo)
  assert eng.preaggregate
  caps0 = list(eng.cap_rows)
  eng.warmup_and_capture(n_eager=1)
  losses = []
  for i in range(40):
    loss = eng.train_step(pool[(i * 512) % (N - 512):][:512].to(DEV))
    if loss is not None:
      losses.append(float(loss.item()))
  losses.append(float(eng.flush().item()))
  assert eng.regrow_count >= 1, (eng.regrow_count, eng.overflow_count(), caps0, eng.cap_rows)
  assert all(l == l and l < 20 for l in losses)
  assert len(eng._A1) == 2 and all(a.shape == eng.A[1].shape and a.shape[0] == eng.cap_T[1] for a in eng._A1)
  loss, correct, n = eng.evaluate_batch(pool[:512].to(DEV))
  assert n == 512 and loss == loss and loss < 20


# --------------------------------------------------------------------------- ticketed tile claiming
def _rand(shape, scale=1.0, seed=0):
  gen = torch.Generator(device=DEV)
  gen.manual_seed(seed)
  return (torch.randn(*shape, device=DEV, generator=gen) * scale).to(torch.bfloat16)


def _counters(idx, val):
  c = torch.zeros(16, dtype=torch.int32, device=DEV)
  c[idx] = val
  return c


def test_ticket_resets_across_graph_replays(native):
  """One CUDA graph launches the same plans twice; a ticket left past the end would make the second launch (or the
  next replay) skip its work, so every output is checked after every replay."""
  T, K, N = 40000, 512, 256                          # 313 row tiles: more items than CTAs
  A = _rand((T, K), seed=1)
  W = _rand((N, K), 0.05, seed=2)
  Z, Z1 = (torch.zeros(T, N, dtype=torch.bfloat16, device=DEV) for _ in range(2))
  c = _counters(1, T)
  fwd = native.TcGemm(0)
  fwd.add_forward(A, W, None, False, Z, c, 1)
  # a two-problem plan (split-K dW + dA): the ticket runs over the combined item space
  dPre = _rand((T, N), 0.1, seed=3)
  gW = torch.zeros(N, K, dtype=torch.float32, device=DEV)
  dA, dA1 = (torch.zeros(T, K, dtype=torch.bfloat16, device=DEV) for _ in range(2))
  bwd = native.TcGemm(0)
  bwd.add_wgrad(dPre, A, gW, c, 1)
  bwd.add_dgrad(dPre, W, dA, c, 1)
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    fwd.run()
    bwd.run()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      for out, keep_, plan in ((Z, Z1, fwd), (dA, dA1, bwd)):
        out.zero_()
        plan.run()
        keep_.copy_(out)
        out.zero_()
        plan.run()
  torch.cuda.current_stream().wait_stream(s)
  ref, absprod = A.double() @ W.double().t(), A.double().abs() @ W.double().abs().t()
  ref_a = dPre.double() @ W.double()
  ref_w, absprod_w = dPre.double().t() @ A.double(), dPre.double().abs().t() @ A.double().abs()
  bound_w = gemm_bound(ref_w, absprod_w, T, bf16_out=False)
  first = None
  for rep in range(4):
    gW.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert bound_ratio(Z, ref, gemm_bound(ref, absprod, K)) <= 1.0, rep
    assert bound_ratio(dA, ref_a, gemm_bound(ref_a, dPre.double().abs() @ W.double().abs(), N)) <= 1.0, rep
    assert torch.equal(Z1, Z) and torch.equal(dA1, dA), rep
    # two launches accumulate into gW
    assert bound_ratio(gW, 2 * ref_w, 2 * bound_w + 2.0 ** -23 * 2 * absprod_w) <= 1.0, rep
    if first is None:
      first = (Z.clone(), dA.clone())
    assert torch.equal(first[0], Z) and torch.equal(first[1], dA), rep


def test_gemm_with_late_starting_ctas_matches_fp32(native):
  """Sleeping kernels on other streams hold SM slots while a GEMM with more items than CTAs starts: whichever CTAs
  start late, the items they did not claim are done by the others and the result is complete."""
  T, K, N = 50000, 512, 256
  A = _rand((T, K), seed=9)
  W = _rand((N, K), 0.05, seed=10)
  b = _rand((N,), seed=11)
  Z = torch.full((T, N), 7.0, dtype=torch.bfloat16, device=DEV)
  c = _counters(1, T)
  pl = native.TcGemm(0)
  pl.add_forward(A, W, b, True, Z, c, 1)
  ref, absprod = A.double() @ W.double().t() + b.double(), A.double().abs() @ W.double().abs().t() + b.double().abs()
  ref = ref.relu()
  bound = gemm_bound(ref, absprod, K)
  sleepers = [torch.cuda.Stream() for _ in range(16)]
  main = torch.cuda.current_stream()
  for rep in range(3):
    Z.fill_(7.0)
    for s in sleepers:
      s.wait_stream(main)
      with torch.cuda.stream(s):
        torch.cuda._sleep(2_000_000 * (1 + rep))
    pl.run()
    for s in sleepers:
      main.wait_stream(s)
    torch.cuda.synchronize()
    assert bound_ratio(Z, ref, bound) <= 1.0, rep
