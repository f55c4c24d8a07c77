"""The small kernels of the R-GAT and HGT training steps (csrc/cuda/gat.cu, hgt.cu) at every width the engines use,
against float64 references.

The engine gradient tests run these kernels only inside a whole step, against an fp32 recomputation with loose
relative tolerances.  Here each kernel is called directly on hand-built device buffers:

  gat_act_bwd    dPre = bf16(dH leaky'(Z) keep / (1 - p)) and the bias gradients of every relation of the layer,
                 or (last layer, dH = None) only the bias gradients of a given dPre
  hgt_gelu       exact-erf GELU and its backward
  hgt_gate       the gated skip connection sigma(skip) A + (1 - sigma(skip)) X and its backward (fp32 and bf16 dZ)
  hgt_blocks     the block-diagonal relation images and the inverse map of their dense gradients
  hgt_kqv_cast   the bf16 [dK | dQ | dV] rows and the K/Q/V bias gradient

Every kernel runs at H in {64, 128, ..., 1024} and at row counts T in {0, 1, 127, 128, 129}, at one T large enough
that the launch reaches its grid cap (528 or 1056 CTAs) and CTAs take more than one pass of the grid-stride loop,
and with counters above the buffer's capacity (T clamps to it).  The counters are int32 on the device with three hops; the entries past the last
hop announce more rows than any buffer holds.  Every output buffer holds a sentinel and has spare rows past the
capacity the kernel sees, so three regions are checked apart: rows < T are written, rows [T, round_up(T, 128)) are
zero where the kernel promises it, and every row after that keeps the sentinel.

Bounds.  u = 2^-24 is fp32's unit roundoff, EPS32 = 2u.  A bf16 result is checked to one bf16 ulp of the float64
value plus twice the fp32 error of the expression before the rounding (helpers.bf16_ulp; rounding a value y within d
of the reference r moves it by at most 2^-9 |y| <= ulp(r) / 2 + d / 256).  An fp32 sum of n terms onto a start value
s0 is checked to (n + 2) EPS32 (sum |terms| + |s0|).  That bound grows as n^2 for rows of like size: for unit-normal
rows a whole row missing from a column sum exceeds it up to a few thousand rows (T = 129 here, and the negative
controls at T of about 1000), while at the large T it only bounds the accumulation error.  The fp32 library functions are IEEE-accurate builds (no fast
math): expf and erff are within 2 ulp and the division is correctly rounded, which gives:

  sigmoid   1 / (1 + expf(-s)) is within 2^-22 of sigma(s) (absolute): expf's 2^-22 relative error moves sigma by at
            most sigma (1 - sigma) 2^-22, the add and the division add u each.  1 - sigma is exact above 0.5 (Sterbenz)
            and adds u below.  SIG_ERR = 2^-21 leaves a factor of two.
  gelu      1 + erff(x / sqrt 2) is within 2^-21 of 1 + erf(x / sqrt 2): erff's 2 ulp (<= 2^-23), the rounding of
            the argument (erf' t times 2u t <= 0.5 2^-23) and of the sum (<= 2^-23).  Y = 0.5 x (1 + erf) therefore
            errs by 0.5 |x| 2^-21 plus u |Y|.  Near x = -10 erff returns -1 exactly and Y is 0 where gelu(x) is
            -8e-23: that is inside 0.5 |x| 2^-21.
  gelu'     0.5 (1 + erf) + x 0.39894228 expf(-0.5 x x): the first term errs by 2^-22, the second by
            (0.5 x^2 + 7) u of itself (expf's argument carries the relative error u of x x, which expf scales by
            0.5 x^2), the sum and the product with dY by u each.
"""
import pytest
import torch

from helpers import (act_bwd_ref, bf16_ulp, block_grads, block_images, bound_ratio, colsum_bound, gate_da_ref,
                     gate_dx_ref, gate_ref, gelu_bwd_ref, gelu_ref, skip_g_ref)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
SENTINEL = 7.0
SPARE = 40                        # rows past the capacity the kernel is given; they must keep the sentinel
EPS32 = 2.0 ** -23
WIDTHS = list(range(64, 1025, 64))
SMALL_T = (0, 1, 127, 128, 129)
SEED = 0x1234_5678_9ABC           # both 32-bit halves of the Philox key are non-zero
STEP = 1234567


def _round(n):
  return (n + 127) // 128 * 128


def _cases(big):
  """(rows the counters announce, capacity): the small T and `big` with 64 rows past their last 128-row tile, then
  counters 1000 rows above a capacity that is not a multiple of 128 (the kernel clamps T, and a zeroing end, to it)."""
  return [(T, _round(T) + 64) for T in SMALL_T + (big,)] + [(big + 1000, big)]


def _counters(T, first=None):
  """Three hops ending at T (the first ends at `first`, default T // 3); entries 4 and up hold 2^20."""
  a = T // 3 if first is None else first
  c = torch.full((16,), 1 << 20, dtype=torch.int32)
  c[:4] = torch.tensor([0, a, max(a, T // 2), T], dtype=torch.int32)
  return c.to(DEV)


def _sentinel(rows, d, dtype=torch.bfloat16):
  return torch.full((rows + SPARE, d), SENTINEL, dtype=dtype, device=DEV)


def _check_tail(buf, T, z_end, what):
  """rows [T, z_end) of buf are zero, rows from z_end on keep the sentinel"""
  assert bool((buf[T:z_end] == 0).all()), f'{what}: rows [T, {z_end}) must be zero'
  assert bool((buf[z_end:] == SENTINEL).all()), f'{what}: rows from {z_end} on must not be written'


_sum_bound = colsum_bound


# --------------------------------------------------------------------------- gat_act_bwd
def _act_bwd_big(d):
  # one CTA per 4 passes of rpb = 256 / (d / 8) rows, capped at 528 CTAs: past 2112 rpb rows the grid is capped
  return 132 * 4 * 4 * (256 // (d // 8)) + 100


def _keep(native, ctr, cap, d, p, layer, step_dev):
  """The forward's keep mask, drawn by dropout_bf16 on a ones tensor with the same key and row pitch."""
  ones = torch.ones(cap, d, dtype=torch.bfloat16, device=DEV)
  native.dropout_bf16(ones, ctr, 3, p, SEED, layer, step_dev)
  return ones != 0


def _act_bwd(native, d, Tc, cap, p, step, layer, g):
  """One gat_act_bwd launch with dH and a 2-relation bias gradient; checks it and returns its pieces."""
  T = min(Tc, cap)
  ctr = _counters(Tc)
  step_dev = None if step is None else torch.tensor([step], dtype=torch.int32, device=DEV)
  keep = _keep(native, ctr, cap, d, p, layer, step_dev)[:T]
  dH = torch.randn(cap + 16, d, generator=g, device=DEV) * 4
  z = torch.randn(cap + 16, d, generator=g, device=DEV)
  z[torch.rand(z.shape, generator=g, device=DEV) < 0.05] = 0.0
  z[torch.rand(z.shape, generator=g, device=DEV) < 0.05] = -0.0
  Z = z.to(torch.bfloat16)
  Z[:T][~keep] = 0.0                              # what the forward left where it dropped: Z == 0 is no mask
  buf = _sentinel(cap, d)
  b0 = torch.randn(2 * d, generator=g, device=DEV)
  bias = b0.clone()
  native.gat_act_bwd(dH, Z, buf[:cap], ctr, 3, p=p, seed=SEED, layer=layer, step_dev=step_dev, bias_g=bias)
  torch.cuda.synchronize()
  got = buf[:T]
  ref, bound = act_bwd_ref(dH[:T], Z[:T], keep, 1.0 / (1.0 - p))
  where = (d, Tc, cap, p, step, layer)
  r = bound_ratio(got, ref, bound)
  assert r <= 1.0, ('dPre', where, r)
  assert torch.equal(got != 0, keep & (dH[:T] != 0)), ('the zeros of dPre are the dropped positions', where)
  _check_tail(buf, T, cap, 'dPre')
  x = got.double()
  rb = bound_ratio(bias.view(2, d), (b0.double().view(2, d) + x.sum(0)), _sum_bound(x, b0.view(2, d), T))
  assert rb <= 1.0, ('bias', where, rb)
  return dict(got=got, ref=ref, keep=keep, dH=dH[:T], Z=Z[:T], ctr=ctr, r=max(r, rb))


@pytest.mark.parametrize('d', WIDTHS)
def test_gat_act_bwd_matches_fp64(native, d):
  g = torch.Generator(device=DEV).manual_seed(d)
  ratio = 0.0
  for Tc, cap in _cases(_act_bwd_big(d)):
    for p, step, layer in ((0.0, None, 1), (0.5, None, 1), (0.5, STEP, 1), (0.5, STEP, 2)):
      ratio = max(ratio, _act_bwd(native, d, Tc, cap, p, step, layer, g)['r'])
  print(f'gat_act_bwd d={d}: max error / bound = {ratio:.3f}')


def _act_last(native, d, Tc, cap, n_bias, g):
  """gat_act_bwd without dH: dPre is only read; bias_g [n_bias * d] gains its column sums over rows < T."""
  T = min(Tc, cap)
  x = torch.randn(cap + SPARE, d, generator=g, device=DEV).to(torch.bfloat16)
  x[T:] = 1e30 * torch.sign(torch.randn(cap + SPARE - T, d, generator=g, device=DEV))     # rows the sums must not see
  buf = x
  before = buf.clone()
  b0 = torch.randn(n_bias * d, generator=g, device=DEV)
  bias = b0.clone()
  native.gat_act_bwd(None, None, buf[:cap], _counters(Tc), 3, bias_g=bias)
  torch.cuda.synchronize()
  assert torch.equal(buf.view(torch.int16), before.view(torch.int16)), 'dPre is only read'
  xd = before[:T].double()
  ref = b0.double().view(n_bias, d) + xd.sum(0)
  bound = _sum_bound(xd, b0.view(n_bias, d), T)
  r = bound_ratio(bias.view(n_bias, d), ref, bound)
  assert r <= 1.0, ('bias', d, Tc, cap, n_bias, r)
  return dict(got=bias.view(n_bias, d), ref=ref, bound=bound, x=xd, b0=b0.view(n_bias, d), r=r)


@pytest.mark.parametrize('d', WIDTHS)
def test_gat_act_bwd_last_layer_bias_gradient(native, d):
  g = torch.Generator(device=DEV).manual_seed(d + 1)
  ratio = 0.0
  for Tc, cap in _cases(_act_bwd_big(d)):
    for n_bias in (1, 3):
      ratio = max(ratio, _act_last(native, d, Tc, cap, n_bias, g)['r'])
  print(f'gat_act_bwd (last layer) d={d}: bias gradient error / bound = {ratio:.3f}')


# --------------------------------------------------------------------------- hgt_gelu
def _elementwise_big(d):
  return 132 * 8 * 256 // (d // 8) + 100          # the grid is capped at 1056 CTAs of 256 vectors


def _gelu_inputs(rows, d, g):
  """bf16 X from a pool: +-12 (erf saturates in fp32), a neighbourhood of 0 (exact zeros included), the negative
  lobe around -0.75 where gelu' < 0, and ordinary values."""
  pool = torch.cat([torch.linspace(-12, 12, 2001, device=DEV),
                    -0.75 + 0.2 * (torch.rand(500, generator=g, device=DEV) - 0.5),
                    1e-3 * torch.randn(300, generator=g, device=DEV), torch.zeros(20, device=DEV),
                    2 * torch.randn(1000, generator=g, device=DEV)])
  return pool[torch.randint(0, len(pool), (rows, d), generator=g, device=DEV)].to(torch.bfloat16)


@pytest.mark.parametrize('d', WIDTHS)
def test_hgt_gelu_matches_fp64(native, d):
  g = torch.Generator(device=DEV).manual_seed(d + 2)
  ratio = [0.0, 0.0]
  for Tc, cap in _cases(_elementwise_big(d)):
    T = min(Tc, cap)
    ctr = _counters(Tc)
    X = _gelu_inputs(cap + 16, d, g)
    dY = (torch.randn(cap + 16, d, generator=g, device=DEV) * 3).to(torch.bfloat16)
    Y, dX = _sentinel(cap, d), _sentinel(cap, d)
    native.hgt_gelu(X, Y[:cap], ctr, 3)
    native.hgt_gelu(X, dX[:cap], ctr, 3, dY=dY)
    torch.cuda.synchronize()
    x = X[:T].double()
    ref, bound = gelu_ref(x)
    r0 = bound_ratio(Y[:T], ref, bound)
    assert r0 <= 1.0, ('gelu', d, Tc, cap, r0)
    _check_tail(Y, T, T, 'gelu')
    gy = dY[:T].double()
    ref, bound = gelu_bwd_ref(x, gy)
    r1 = bound_ratio(dX[:T], ref, bound)
    assert r1 <= 1.0, ('gelu backward', d, Tc, cap, r1)
    _check_tail(dX, T, min(cap, _round(T)), 'gelu backward')
    ratio = [max(ratio[0], r0), max(ratio[1], r1)]
  print(f'hgt_gelu d={d}: max error / bound = {ratio[0]:.3f} (forward), {ratio[1]:.3f} (backward)')


# --------------------------------------------------------------------------- hgt_gate
GATE_MODES = [('fp32', True, True), ('bf16', True, True), ('fp32', False, False), ('bf16', False, True)]


def _gate(native, d, Tc, cap, skip, mode, g):
  """hgt_gate forward (mode None) or backward (dZ dtype, with dX, with skip_g); checks it, returns its pieces."""
  T = min(Tc, cap)
  ctr = _counters(Tc)
  A = torch.randn(cap + 16, d, generator=g, device=DEV).to(torch.bfloat16)
  X = torch.randn(cap + 16, d, generator=g, device=DEV).to(torch.bfloat16)
  sk = torch.tensor([skip], dtype=torch.float32, device=DEV)
  sg = torch.sigmoid(sk.double())
  a, x = A[:T].double(), X[:T].double()
  out = _sentinel(cap, d)
  where = (d, Tc, cap, skip, mode)
  if mode is None:
    native.hgt_gate(A, X, out[:cap], sk, ctr, 3)
    torch.cuda.synchronize()
    ref, bound = gate_ref(a, x, sg)
    r = bound_ratio(out[:T], ref, bound)
    assert r <= 1.0, ('gate', where, r)
    _check_tail(out, T, T, 'gate')
    return dict(r=r)
  kind, with_dx, with_sg = mode
  dZ = torch.randn(cap + 16, d, generator=g, device=DEV) * 2
  if kind == 'bf16':
    dZ = dZ.to(torch.bfloat16)
  dX0 = torch.randn(cap + SPARE, d, generator=g, device=DEV)
  dX = dX0.clone()
  s0 = torch.tensor([0.37], device=DEV)
  skip_g = s0.clone()
  native.hgt_gate(A, X, out[:cap], sk, ctr, 3, dZ=dZ, dX=dX[:cap] if with_dx else None,
                  skip_g=skip_g if with_sg else None)
  torch.cuda.synchronize()
  gz = dZ[:T].double()
  ref, bound = gate_da_ref(gz, sg)
  r = bound_ratio(out[:T], ref, bound)
  assert r <= 1.0, ('gate dA', where, r)
  _check_tail(out, T, min(cap, _round(T)), 'gate dA')
  if with_dx:
    ref, bound = gate_dx_ref(dX0[:T].double(), gz, sg)
    rx = bound_ratio(dX[:T], ref, bound)
    assert rx <= 1.0, ('gate dX', where, rx)
    r = max(r, rx)
  assert torch.equal(dX[T:] if with_dx else dX, dX0[T:] if with_dx else dX0), 'dX rows >= T are untouched'
  t = gz * (a - x)
  dsg = sg * (1 - sg)
  # fp32 sum of T d terms onto s0, and sigma'(skip) within 2^-20 (two factors within SIG_ERR)
  ref_s, bound_s = skip_g_ref(s0, sg, t, T * d)
  if with_sg:
    rs = bound_ratio(skip_g, ref_s, bound_s)
    assert rs <= 1.0, ('skip_g', where, rs)
    r = max(r, rs)
  else:
    assert torch.equal(skip_g, s0)
  return dict(r=r, t=t, s0=s0, dsg=dsg, sg=sg, skip_g=skip_g, ref_s=ref_s, bound_s=bound_s)


@pytest.mark.parametrize('d', WIDTHS)
def test_hgt_gate_matches_fp64(native, d):
  g = torch.Generator(device=DEV).manual_seed(d + 3)
  ratio = 0.0
  for Tc, cap in _cases(_elementwise_big(d)):
    for skip in (0.0, 8.0, -8.0):
      for mode in [None] + GATE_MODES:
        ratio = max(ratio, _gate(native, d, Tc, cap, skip, mode, g)['r'])
  print(f'hgt_gate d={d}: max error / bound = {ratio:.3f}')


# --------------------------------------------------------------------------- hgt_blocks
def _heads(H):
  """heads = 1, H / 64 and H / 8 (head widths H, 64 and 8); at H = 1024 also 8 and 16 heads"""
  hs = {1, max(1, H // 64), H // 8}
  return sorted(hs | ({8, 16} if H == 1024 else set()))


@pytest.mark.parametrize('H', WIDTHS)
def test_hgt_blocks_match_block_diag(native, H):
  g = torch.Generator(device=DEV).manual_seed(H + 4)
  for heads in _heads(H):
    D = H // heads
    for R in (1, 3, 8):
      att = torch.randn(R, heads, D, D, generator=g, device=DEV).to(torch.bfloat16)
      msg = torch.randn(R, heads, D, D, generator=g, device=DEV).to(torch.bfloat16)
      att_img = torch.full((R * H, H), SENTINEL, dtype=torch.bfloat16, device=DEV)
      msg_img = torch.full((H, R * H), SENTINEL, dtype=torch.bfloat16, device=DEV)
      native.hgt_blocks(att, msg, att_img, msg_img)
      torch.cuda.synchronize()
      where = (H, heads, D, R)
      # att_img rows r H .. (r + 1) H: block h is att[r, h];  msg_img columns r H ..: block h is msg[r, h]^T
      ref_a, ref_m = block_images(att, msg)
      assert torch.equal(att_img.view(torch.int16), ref_a.view(torch.int16)), ('att image', where)
      assert torch.equal(msg_img.view(torch.int16), ref_m.view(torch.int16)), ('msg image', where)

      # gradient mode: the diagonal blocks of the dense fp32 gradients are added onto att_g / msg_g
      att_g0 = torch.randn(R, heads, D, D, generator=g, device=DEV)
      msg_g0 = torch.randn(R, heads, D, D, generator=g, device=DEV)
      att_d = torch.randn(R * H, H, generator=g, device=DEV)
      msg_d = torch.randn(H, R * H, generator=g, device=DEV)
      blk_a, blk_m = block_grads(att_d, msg_d, R, heads, D)
      exp_a, exp_m = att_g0 + blk_a, msg_g0 + blk_m               # one fp32 add, as in the kernel
      att_g, msg_g = att_g0.clone(), msg_g0.clone()
      att_img.fill_(SENTINEL)
      msg_img.fill_(SENTINEL)
      native.hgt_blocks(att, msg, att_img, msg_img, att_d, msg_d, att_g, msg_g)
      torch.cuda.synchronize()
      assert torch.equal(att_g, exp_a) and torch.equal(msg_g, exp_m), ('gradient blocks', where)
      assert bool((att_d == 0).all()) and bool((msg_d == 0).all()), ('dense gradients are re-zeroed', where)
      assert bool((att_img == SENTINEL).all()) and bool((msg_img == SENTINEL).all()), ('images untouched', where)


# --------------------------------------------------------------------------- hgt_kqv_cast
def _kqv_big(H):
  # one CTA per 4 passes of rpb = 256 / cw rows (cw vectors per blockIdx.y chunk), capped at 528 CTAs
  cw = min(3 * H // 8, 128)
  return 132 * 4 * 4 * (256 // cw) + 100


def _kqv(native, H, Tc, cap, with_dq, g, q_rows=None):
  """One hgt_kqv_cast launch (rows < n of dkv, rows < nq of dq; dq has q_rows rows, default cap + 16, and rows
  past them hold 1e30); checks it and returns its pieces."""
  first = 2 * Tc // 3
  n = min(Tc, cap)
  q_rows = cap + 16 if q_rows is None else q_rows
  nq = min(first, n, q_rows) if with_dq else 0
  ctr = _counters(Tc, first)
  ex = torch.exp2(torch.randint(-20, 21, (cap + SPARE, 2 * H), generator=g, device=DEV).float())
  dkv = torch.randn(cap + SPARE, 2 * H, generator=g, device=DEV) * ex
  dkv0 = dkv.clone()
  dq = (torch.randn(cap + SPARE, H, generator=g, device=DEV) * 3).to(torch.bfloat16)
  dq[q_rows:] = 1e30
  out = _sentinel(cap, 3 * H)
  b0 = torch.randn(3 * H, generator=g, device=DEV)
  bias = b0.clone()
  native.hgt_kqv_cast(dkv[:cap], dq[:q_rows] if with_dq else None, out[:cap], bias, ctr, 3, 1)
  torch.cuda.synchronize()
  where = (H, Tc, cap, with_dq)
  got = out[:n]
  bits = lambda t: t.contiguous().view(torch.int16)   # noqa: E731
  assert torch.equal(bits(got[:, :H]), bits(dkv0[:n, :H].to(torch.bfloat16))), ('dK', where)
  assert torch.equal(bits(got[:, 2 * H:]), bits(dkv0[:n, H:].to(torch.bfloat16))), ('dV', where)
  assert torch.equal(got[:nq, H:2 * H], dq[:nq]), ('dQ', where)
  assert bool((got[nq:, H:2 * H] == 0).all()), ('dQ rows >= nq are zero', where)
  _check_tail(out, n, min(cap, _round(n)), 'kqv out')
  assert bool((dkv[:n] == 0).all()), ('dkv rows < n are re-zeroed', where)
  assert torch.equal(dkv[n:], dkv0[n:]), ('dkv rows >= n are untouched', where)
  x = got.double()
  ref = b0.double() + x.sum(0)
  bound = _sum_bound(x, b0, n)
  r = bound_ratio(bias, ref, bound)
  assert r <= 1.0, ('kqv bias', where, r)
  return dict(got=bias, ref=ref, bound=bound, x=x, b0=b0, r=r)


@pytest.mark.parametrize('dq', ['dq', 'no_dq'])
@pytest.mark.parametrize('H', WIDTHS)
def test_hgt_kqv_cast_matches_fp64(native, H, dq):
  g = torch.Generator(device=DEV).manual_seed(H + 5 + (dq == 'dq'))
  ratio = 0.0
  for Tc, cap in _cases(_kqv_big(H)):
    ratio = max(ratio, _kqv(native, H, Tc, cap, dq == 'dq', g)['r'])
  chunks = (3 * H // 8 + 127) // 128
  print(f'hgt_kqv_cast H={H} ({chunks} column chunks) {dq}: bias gradient error / bound = {ratio:.3f}')


@pytest.mark.parametrize('H', [64, 384, 704, 1024])
def test_hgt_kqv_cast_reads_dq_only_to_its_rows(native, H):
  """dQ shorter than the rows the counter gives it (the engine passes a dQ sized for the layer's targets): nq clamps
  to dQ's rows, like every extent read from a counter, and the rows of dQ's segment past them are zero."""
  g = torch.Generator(device=DEV).manual_seed(H + 7)
  for q_rows in (1, 300):
    _kqv(native, H, 1000, 1100, True, g, q_rows=q_rows)


# --------------------------------------------------------------------------- the bounds have teeth
def test_bounds_reject_plausible_defects(native):
  """The defects these kernels could plausibly have, applied in float64 to their results or references, each
  exceed their bound.  The summation bounds grow with the number of terms, so each is shown at a row count where
  the defect is the size a real one would be."""
  g = torch.Generator(device=DEV).manual_seed(99)

  def col_defects(res, c0):
    """one row missing from every column sum, and the 8-column group at c0 missing entirely"""
    no_row = bound_ratio(res['got'] - res['x'][-1], res['ref'], res['bound'])
    no_group = res['got'].clone()
    no_group[..., c0:c0 + 8] = res['b0'][..., c0:c0 + 8]
    return no_row, bound_ratio(no_group, res['ref'], res['bound'])

  # gat_act_bwd, last layer: 3 relation biases, 1093 rows
  res = _act_last(native, 1024, 1093, 1200, 3, g)
  act_row, act_group = col_defects(res, 1016)
  # hgt_kqv_cast at H = 704: the third column chunk holds one 8-column group, the last of dV
  res = _kqv(native, 704, 1000, 1100, True, g)
  kqv_row, kqv_group = col_defects(res, 3 * 704 - 8)

  # hgt_gate: one CTA's partial of skip_g dropped, and sigma in place of sigma'
  d, T, cap = 64, 129, 320
  res = _gate(native, d, T, cap, 0.0, ('fp32', True, True), g)
  nvec = d // 8
  grid = min(1056, (cap * nvec + 255) // 256)
  vec = torch.arange(T * nvec, device=DEV)
  cta = (vec % (grid * 256)) // 256
  part = torch.zeros(grid, dtype=torch.float64, device=DEV).index_add_(0, cta, res['t'].view(-1, 8).sum(1))
  worst = int(part.abs().argmax())
  no_cta = bound_ratio(res['skip_g'] - res['dsg'] * part[worst], res['ref_s'], res['bound_s'])
  sig = bound_ratio(res['s0'].double() + res['sg'] * res['t'].sum(), res['ref_s'], res['bound_s'])

  # gat_act_bwd: the keep mask of the neighbouring step
  d, T = 128, 1000
  res = _act_bwd(native, d, T, _round(T), 0.5, STEP, 1, g)
  near = _keep(native, res['ctr'], _round(T), d, 0.5, 1, torch.tensor([STEP + 1], dtype=torch.int32, device=DEV))[:T]
  ref = res['dH'].double() * torch.where(res['Z'] > 0, 1.0, 0.01).double() * near.double() * 2.0
  step_r = bound_ratio(res['got'], ref, bf16_ulp(ref))
  print(f'defects: error / bound = {act_row:.1f} / {act_group:.1f} (gat_act_bwd bias: row / 8-column group missing), '
        f'{kqv_row:.1f} / {kqv_group:.1f} (hgt_kqv_cast bias: row / last 8-column group missing), '
        f'{no_cta:.1f} (skip_g: one CTA dropped), {sig:.1f} (skip_g: sigma for sigma\'), '
        f'{step_r:.3g} (keep mask of step + 1)')
  assert min(act_row, act_group, kqv_row, kqv_group, no_cta, sig, step_r) > 1.0
