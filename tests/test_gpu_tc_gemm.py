"""Numerics of the TMA-fed wgmma GEMM kernel (csrc/cuda/tc_gemm.cu) against plain fp32 PyTorch.

Three operand layouts are exercised: K-major x K-major (forward), K-major x MN-major (dA) and MN-major x MN-major
with split-K fp32 reductions (dW); the batch-dependent extent comes from a device counter like in the engine.

Every result is checked against a float64 reference with the bound of `helpers.gemm_bound`: one bf16 ulp plus
K * 2^-22 * (|A| . |W|^T), below the error of one dropped 64-deep k-block or one wrong 8-column group.  The shapes cover
K that is not a multiple of 64, several N tiles of 64 / 128 columns (the bias read at n_tile > 0), ragged row tiles
and an A operand that is a column slice of a wider tensor (as `GraphSageEngine.inference()` passes it)."""
import pytest
import torch

from helpers import bound_ratio, gemm_bound

pytestmark = pytest.mark.gpu


def _counters(dev, idx, val):
  c = torch.zeros(16, dtype=torch.int32, device=dev)
  c[idx] = val
  return c


def _rand(shape, dev, scale=1.0, seed=0):
  g = torch.Generator(device=dev)
  g.manual_seed(seed)
  return (torch.randn(*shape, device=dev, generator=g) * scale).to(torch.bfloat16)


def _case(*vals, a_ld=0):
  """A forward case; a_ld > 0 makes A the first K columns of a [cap, a_ld] tensor."""
  return pytest.param(*vals, a_ld, id='-'.join(str(v) for v in vals) + (f'-ld{a_ld}' if a_ld else ''))


def _ref_forward(A, W, b, relu):
  """float64 act(A . W^T + b) and |A| . |W|^T + |b| (the scale of the accumulation error)."""
  Ad, Wd = A.double(), W.double()
  ref, absprod = Ad @ Wd.t(), Ad.abs() @ Wd.abs().t()
  if b is not None:
    ref, absprod = ref + b.double(), absprod + b.double().abs()
  return (ref.relu() if relu else ref), absprod


@pytest.mark.parametrize('cap,T,K,N,relu,with_bias,a_ld', [
  _case(1000, 777, 512, 256, True, True),
  _case(1024, 1024, 512, 64, False, True),
  _case(40000, 33333, 256, 256, True, False),
  _case(300, 1, 128, 128, False, True),
  _case(512, 0, 512, 256, True, True),
  # K not a multiple of 64 (the last k-block is partly outside the operands)
  _case(300, 257, 8, 64, False, True),
  _case(1000, 777, 200, 256, True, True),
  _case(1000, 129, 400, 128, False, True),
  _case(640, 639, 1032, 192, True, True),
  # N tiles of 64 / 128 columns: several tiles per row block, bias read at n_tile > 0
  _case(1000, 777, 256, 192, True, True),
  _case(512, 500, 128, 320, False, True),
  _case(1000, 1000, 512, 384, True, True),
  _case(700, 650, 256, 640, False, True),
  _case(400, 301, 512, 3008, False, True),
  # row counts at a 128-row tile boundary
  _case(300, 127, 256, 256, True, True),
  _case(300, 128, 256, 256, False, True),
  _case(300, 129, 256, 256, True, True),
  # A as a column slice of a wider tensor
  _case(1000, 777, 256, 256, True, True, a_ld=1024),
  _case(900, 899, 200, 192, False, True, a_ld=512),
])
def test_tc_forward_matches_fp32(native, cap, T, K, N, relu, with_bias, a_ld):
  dev = torch.device('cuda', 0)
  A = _rand((cap, a_ld), dev, seed=1)[:, :K] if a_ld else _rand((cap, K), dev, seed=1)
  W = _rand((N, K), dev, 0.05, seed=2)
  b = _rand((N,), dev, seed=3) if with_bias else None
  Z = torch.full((cap, N), 7.0, dtype=torch.bfloat16, device=dev)
  c = _counters(dev, 2, T)
  pl = native.TcGemm(0)
  pl.add_forward(A, W, b, relu, Z, c, 2)
  pl.run()
  torch.cuda.synchronize()
  ref, absprod = _ref_forward(A[:T], W, b, relu)
  bound = gemm_bound(ref, absprod, K)
  r = bound_ratio(Z[:T], ref, bound)
  print(f'forward {cap}-{T}-{K}-{N} ld={a_ld}: max error / bound = {r:.3f}')
  assert r <= 1.0, r
  # rows of untouched tiles keep their old contents (only tiles below ceil(T/128) are written)
  first_untouched = (T + 127) // 128 * 128
  if first_untouched < cap:
    assert bool((Z[first_untouched:] == 7.0).all())
  # the counter is re-read on every launch: shrink the batch and run the SAME plan again
  if T > 200:
    c[2] = 130
    Z.fill_(7.0)
    pl.run()
    torch.cuda.synchronize()
    assert bound_ratio(Z[:130], ref[:130], bound[:130]) <= 1.0
    assert bool((Z[256:] == 7.0).all())


@pytest.mark.parametrize('cap,T,Kd,N', [(1200, 1000, 256, 512), (1024, 1024, 64, 512), (20000, 12345, 256, 256),
                                        (1000, 999, 96, 192), (1000, 777, 200, 320)])
def test_tc_dgrad_matches_fp32(native, cap, T, Kd, N):
  dev = torch.device('cuda', 0)
  dPre = _rand((cap, Kd), dev, seed=4)
  W = _rand((Kd, N), dev, 0.05, seed=5)
  dA = torch.zeros(cap, N, dtype=torch.bfloat16, device=dev)
  c = _counters(dev, 1, T)
  pl = native.TcGemm(0)
  pl.add_dgrad(dPre, W, dA, c, 1)
  pl.run()
  torch.cuda.synchronize()
  ref, absprod = dPre[:T].double() @ W.double(), dPre[:T].double().abs() @ W.double().abs()
  r = bound_ratio(dA[:T], ref, gemm_bound(ref, absprod, Kd))
  print(f'dgrad {cap}-{T}-{Kd}-{N}: max error / bound = {r:.3f}')
  assert r <= 1.0, r


@pytest.mark.parametrize('cap,T,M,N', [(1200, 1000, 256, 512), (1024, 1024, 64, 512), (50000, 45678, 256, 256),
                                       (4096, 63, 256, 512), (4096, 0, 256, 512),
                                       (1200, 1000, 8, 192), (1200, 1111, 96, 320), (3000, 2999, 200, 192),
                                       (1000, 777, 3008, 320)])
def test_tc_wgrad_split_k_matches_fp32(native, cap, T, M, N):
  dev = torch.device('cuda', 0)
  dPre = _rand((cap, M), dev, 0.1, seed=6)
  dPre[T:] = 0                      # engine invariant: rows beyond the batch are zero up to the capacity
  A = _rand((cap, N), dev, seed=7)  # rows beyond T hold stale (finite) data
  gW = torch.zeros(M, N, dtype=torch.float32, device=dev)
  c = _counters(dev, 3, T)
  pl = native.TcGemm(0)
  pl.add_wgrad(dPre, A, gW, c, 3)
  pl.run()
  torch.cuda.synchronize()
  ref, absprod = dPre[:T].double().t() @ A[:T].double(), dPre[:T].double().abs().t() @ A[:T].double().abs()
  bound = gemm_bound(ref, absprod, T, bf16_out=False)
  r = bound_ratio(gW, ref, bound)
  print(f'wgrad {cap}-{T}-{M}-{N}: max error / bound = {r:.3f}')
  assert r <= 1.0, r
  # red-add semantics: a second run accumulates
  pl.run()
  torch.cuda.synchronize()
  assert bound_ratio(gW, 2 * ref, 2 * bound + 2.0 ** -23 * 2 * absprod) <= 1.0


def test_tc_wgrad_and_dgrad_share_one_launch(native):
  dev = torch.device('cuda', 0)
  cap, T, n_out, two_d = 12000, 9999, 256, 512
  dPre = _rand((cap, n_out), dev, 0.1, seed=8)
  dPre[T:] = 0
  A = _rand((cap, two_d), dev, seed=9)
  W = _rand((n_out, two_d), dev, 0.05, seed=10)
  gW = torch.zeros(n_out, two_d, dtype=torch.float32, device=dev)
  dA = torch.zeros(cap, two_d, dtype=torch.bfloat16, device=dev)
  c = _counters(dev, 2, T)
  pl = native.TcGemm(0)
  pl.add_wgrad(dPre, A, gW, c, 2)
  pl.add_dgrad(dPre, W, dA, c, 2)
  pl.run()
  torch.cuda.synchronize()
  d, a, w = dPre[:T].double(), A[:T].double(), W.double()
  ref_w, ref_a = d.t() @ a, d @ w
  assert bound_ratio(gW, ref_w, gemm_bound(ref_w, d.abs().t() @ a.abs(), T, bf16_out=False)) <= 1.0
  assert bound_ratio(dA[:T], ref_a, gemm_bound(ref_a, d.abs() @ w.abs(), n_out)) <= 1.0


def test_tc_gemm_inside_cuda_graph(native):
  dev = torch.device('cuda', 0)
  A = _rand((2048, 512), dev, seed=11)
  W = _rand((256, 512), dev, 0.05, seed=12)
  Z = torch.zeros(2048, 256, dtype=torch.bfloat16, device=dev)
  c = _counters(dev, 1, 1500)
  pl = native.TcGemm(0)
  pl.add_forward(A, W, None, False, Z, c, 1)
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    pl.run()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      pl.run()
  torch.cuda.synchronize()
  Z.zero_()
  c[1] = 2048
  g.replay()
  torch.cuda.synchronize()
  ref, absprod = _ref_forward(A, W, None, False)
  assert bound_ratio(Z, ref, gemm_bound(ref, absprod, 512)) <= 1.0
