"""The engine bindings check every tensor their kernel dereferences: device, dtype, layout and the extents the host
knows.  Each binding is called once with valid arguments, then with one argument at a time replaced by an invalid one,
which must raise RuntimeError.

Every invalid argument is one the kernel could take without faulting had its check been missing: tensors that are not
on the device are pinned host memory of the full size, a wrong dtype is at least as wide as the right one, a short
tensor is a view into an allocation large enough for the valid call, and index tensors keep valid values.
Misalignment is tested only through TcGemm's add_* methods, which build a plan without launching anything."""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
N_SRC, D, CAP = 600, 64, 400
HOPS = [(50, 4), (300, 3)]


def pinned(t):
  return t.cpu().pin_memory()


def wide(t):
  """The same values in a dtype at least as wide."""
  to = {torch.bfloat16: torch.float32, torch.int32: torch.int64, torch.float32: torch.float64}[t.dtype]
  return t.to(to)


def probe(fn, args, bad):
  """fn(*args) runs; fn with args[i] replaced by any value of bad[i] raises RuntimeError."""
  fn(*args)
  torch.cuda.synchronize()
  for i, alts in bad.items():
    for alt in alts:
      a = list(args)
      a[i] = alt
      with pytest.raises(RuntimeError):
        fn(*a)
  torch.cuda.synchronize()


def bad_tensor(t, short=None):
  """Not on the device, a wider dtype, and optionally a short view."""
  return [pinned(t), wide(t)] + ([short] if short is not None else [])


@pytest.fixture(scope='module')
def batch():
  g = torch.Generator().manual_seed(0)
  cum, degs, ells = [0], [], []
  for rows, k in HOPS:
    degs.append(torch.randint(0, k + 1, (rows,), generator=g).to(torch.int32))
    ells.append(torch.randint(0, N_SRC, (rows * k,), generator=g).to(torch.int32).to(DEV))
    cum.append(cum[-1] + rows)
  ctr = torch.zeros(16, dtype=torch.int32)
  ctr[:len(cum)] = torch.tensor(cum, dtype=torch.int32)
  src = (torch.randn(N_SRC, D, generator=g)).to(torch.bfloat16).to(DEV)
  return dict(ctr=ctr.to(DEV), ell=ells, ks=[k for _, k in HOPS], deg=torch.cat(degs).to(DEV), src=src,
              nh=len(HOPS))


def test_sage_aggregate(native, batch):
  b = batch
  out = torch.zeros(CAP, 2 * D, dtype=torch.bfloat16, device=DEV)
  args = [None, None, b['src'], D, b['ctr'], b['nh'], b['ell'], b['ks'], b['deg'], out]
  probe(native.sage_aggregate, args, {
      2: bad_tensor(b['src']), 4: bad_tensor(b['ctr']), 8: bad_tensor(b['deg']),
      6: [[pinned(e) for e in b['ell']], [wide(e) for e in b['ell']]]})


def test_sage_aggregate_layer1_nodes(native, batch):
  b = batch
  X = torch.randn(N_SRC, D).to(torch.bfloat16)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(X.to(DEV))
  nodes = torch.randperm(N_SRC).to(DEV)
  out = torch.zeros(CAP, 2 * D, dtype=torch.bfloat16, device=DEV)
  probe(native.sage_aggregate, [ut._table(), nodes, None, D, b['ctr'], b['nh'], b['ell'], b['ks'], b['deg'], out],
        {1: [pinned(nodes)]})


def test_sage_block_kernels(native, batch):
  b = batch
  A = torch.zeros(CAP, 3 * D, dtype=torch.bfloat16, device=DEV)
  probe(native.sage_aggregate_block, [None, None, b['src'], D, b['ctr'], b['nh'], b['ell'], b['ks'], b['deg'], A, D],
        {9: [pinned(A), wide(A)], 4: bad_tensor(b['ctr'])})
  dH = torch.zeros(N_SRC, D, device=DEV)
  probe(native.sage_scatter_block, [A, D, D, b['ctr'], b['nh'], b['ell'], b['ks'], b['deg'], dH],
        {0: [wide(A)], 3: bad_tensor(b['ctr']), 7: bad_tensor(b['deg']), 8: [pinned(dH), wide(dH), dH[:, :D - 8]]})
  probe(native.add_block_f32, [A, 2 * D, D, b['ctr'], b['nh'], dH[:CAP]],
        {0: [wide(A)], 3: bad_tensor(b['ctr']), 5: [pinned(dH[:CAP]), wide(dH[:CAP])]})


def test_relu_bwd_cast_and_colsum(native, batch):
  ctr = batch['ctr']
  dH = torch.randn(CAP, D, device=DEV)
  Z = torch.randn(CAP, D, device=DEV).to(torch.bfloat16)
  dPre = torch.zeros(CAP, D, dtype=torch.bfloat16, device=DEV)
  colsum_buf = torch.zeros(D + 8, device=DEV)
  probe(native.relu_bwd_cast, [dH, Z, ctr, 2, dPre, colsum_buf[:D], True, 1.0, True],
        {1: bad_tensor(Z), 2: bad_tensor(ctr), 4: [pinned(dPre), wide(dPre)],
         5: [pinned(colsum_buf[:D]), wide(colsum_buf[:D]), colsum_buf[:D - 4]]})
  out_buf = torch.zeros(D + 8, device=DEV)
  probe(native.colsum_bf16, [Z, ctr, 2, out_buf[:D]],
        {1: bad_tensor(ctr), 3: [pinned(out_buf[:D]), wide(out_buf[:D]), out_buf[:D - 8]]})
  probe(native.zero_rows, [dH, ctr, 2], {1: bad_tensor(ctr)})


def test_softmax_nll(native, batch):
  ctr = batch['ctr']
  C, ld = 47, 64
  logits = torch.randn(CAP, ld, device=DEV).to(torch.bfloat16)
  dl = torch.zeros_like(logits)
  labels = torch.randint(0, C, (N_SRC,), device=DEV)
  nodes = torch.randperm(N_SRC, device=DEV)
  loss, correct = torch.zeros(1, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
  colsum = torch.zeros(ld, device=DEV)
  probe(native.softmax_nll, [logits, C, None, labels, nodes, ctr, loss, dl, correct, colsum, False],
        {3: [pinned(labels)], 4: [pinned(nodes)], 5: bad_tensor(ctr), 6: bad_tensor(loss), 7: [pinned(dl), wide(dl)],
         8: bad_tensor(correct), 9: bad_tensor(colsum)})


def test_zero_grads_and_adam(native):
  n = 1024
  p, g = torch.randn(n, device=DEV), torch.randn(n, device=DEV)
  m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
  p16 = p.to(torch.bfloat16)
  step = torch.zeros(2, dtype=torch.int32, device=DEV)
  loss, correct = torch.zeros(1, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
  probe(native.zero_grads, [g.clone(), loss, correct], {1: bad_tensor(loss), 2: bad_tensor(correct)})
  probe(native.adam_step, [p, g, m, v, p16, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, 1.0],
        {1: [pinned(g)], 2: [pinned(m)], 3: [pinned(v)], 4: [pinned(p16), wide(p16)], 10: bad_tensor(step)})


def test_dropout(native, batch):
  ctr = batch['ctr']
  Z = torch.randn(CAP, D, device=DEV).to(torch.bfloat16)
  step = torch.zeros(2, dtype=torch.int32, device=DEV)
  probe(native.dropout_bf16, [Z, ctr, 2, 0.5, 1, 1, step], {1: bad_tensor(ctr), 6: bad_tensor(step)})


def test_sage_fused(native, batch):
  b = batch
  n_out = 256
  if not native.sage_fused_supported(D, n_out):
    pytest.skip('fused layer shape not supported')
  W = (torch.randn(n_out, 2 * D, device=DEV) * 0.1).to(torch.bfloat16)
  wp = native.pack_weight(W)
  bias_buf = torch.zeros(n_out + 8, dtype=torch.bfloat16, device=DEV)
  z = torch.zeros(CAP, n_out, dtype=torch.bfloat16, device=DEV)
  A = torch.zeros(CAP, 2 * D, dtype=torch.bfloat16, device=DEV)
  args = [None, None, b['src'], D, b['ctr'], b['nh'], b['ell'], b['ks'], b['deg'], wp, bias_buf[:n_out], True, z, A]
  probe(native.sage_fused, args,
        {4: bad_tensor(b['ctr']), 8: bad_tensor(b['deg']), 9: [wide(wp)],   # w_packed is read by TMA: no host memory
         10: [pinned(bias_buf[:n_out]), wide(bias_buf[:n_out]), bias_buf[:n_out - 8]], 13: [pinned(A), wide(A)]})
  probe(native.pack_weight_into, [W, wp], {1: [pinned(wp), wide(wp)]})


def test_gat_and_hgt_elementwise(native, batch):
  ctr = batch['ctr']
  H, heads = 64, 2
  P = torch.randn(CAP, H, device=DEV).to(torch.bfloat16)
  att = torch.randn(H, device=DEV).to(torch.bfloat16)
  out = torch.zeros(CAP, heads, device=DEV)
  probe(lambda *a: native.gat_scores(*a, heads=heads), [P, att, out, ctr, 2],
        {1: [pinned(att), wide(att)], 3: bad_tensor(ctr)})
  X = torch.randn(CAP, H, device=DEV).to(torch.bfloat16)
  Y = torch.zeros_like(X)
  probe(native.hgt_gelu, [X, Y, ctr, 2], {2: bad_tensor(ctr)})
  skip = torch.zeros(1, device=DEV)
  probe(native.hgt_gate, [P, X, Y, skip, ctr, 2], {3: bad_tensor(skip), 4: bad_tensor(ctr)})


def test_link_bce(native, batch):
  ctr = batch['ctr']
  C, Pn, B = 64, 120, 40
  Z = torch.randn(CAP, C, device=DEV).to(torch.bfloat16)
  sl = torch.randint(0, CAP, (2 * Pn,), device=DEV, dtype=torch.int32)
  n_pairs = torch.tensor([Pn], dtype=torch.int32, device=DEV)
  loss, correct = torch.zeros(1, device=DEV), torch.zeros(1, dtype=torch.int32, device=DEV)
  dZ = torch.zeros(CAP, C, device=DEV)
  probe(native.link_bce, [Z, C, sl, Pn, B, n_pairs, loss, correct, dZ],
        {2: [pinned(sl)], 5: bad_tensor(n_pairs), 6: bad_tensor(loss), 7: bad_tensor(correct),
         8: [pinned(dZ), wide(dZ)]})


def test_row_table_gather_into(native):
  X = torch.randn(N_SRC, D).to(torch.bfloat16)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(X.to(DEV))
  tbl = ut._table()
  ids = torch.randint(0, N_SRC, (CAP,), device=DEV)
  n_dev = torch.tensor([CAP], dtype=torch.int32, device=DEV)
  out = torch.zeros(CAP, D, dtype=torch.bfloat16, device=DEV)
  probe(tbl.gather_into, [ids, None, n_dev, out], {0: [pinned(ids)], 2: bad_tensor(n_dev), 3: [pinned(out), wide(out)]})


def test_tc_gemm_plans(native):
  """add_* only encode a plan: every invalid case here, misalignment included, must raise before anything runs."""
  rows, K, N = 256, 128, 128
  ctr = torch.zeros(16, dtype=torch.int32, device=DEV)
  ctr[1] = rows
  A_buf = torch.zeros(rows * K + 8, dtype=torch.bfloat16, device=DEV)
  A = A_buf[:rows * K].view(rows, K)
  A_mis = A_buf[8:].view(rows, K)                             # 16 bytes off: aligned rows
  A_mis2 = A_buf[4:4 + rows * K].view(rows, K)                # 8 bytes off
  W = torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
  bias_buf = torch.zeros(N + 8, dtype=torch.bfloat16, device=DEV)
  Z = torch.zeros(rows, N, dtype=torch.bfloat16, device=DEV)

  def fwd(A, W, bias, Z, c):
    native.TcGemm(0).add_forward(A, W, bias, True, Z, c, 1)

  probe(fwd, [A, W, bias_buf[:N], Z, ctr],
        {0: [pinned(A), wide(A), A_mis2], 1: [pinned(W), wide(W)], 2: [pinned(bias_buf[:N]), bias_buf[4:4 + N],
                                                                      bias_buf[:N - 8]],
         3: [pinned(Z), wide(Z)], 4: bad_tensor(ctr)})
  fwd(A_mis, W, bias_buf[:N], Z, ctr)                         # 16-byte aligned offsets are fine
  dA = torch.zeros(rows, K, dtype=torch.bfloat16, device=DEV)
  dPre = torch.zeros(rows, N, dtype=torch.bfloat16, device=DEV)
  Wt = torch.zeros(N, K, dtype=torch.bfloat16, device=DEV)
  probe(lambda dPre, W, dA: native.TcGemm(0).add_dgrad(dPre, W, dA, ctr, 1), [dPre, Wt, dA],
        {0: [pinned(dPre), wide(dPre)], 2: [pinned(dA), wide(dA), A_mis2]})
  gW = torch.zeros(N, K, device=DEV)
  probe(lambda dPre, A, gW: native.TcGemm(0).add_wgrad(dPre, A, gW, ctr, 1), [dPre, A, gW],
        {1: [pinned(A), wide(A), A_mis2], 2: [pinned(gW), gW.double()]})
