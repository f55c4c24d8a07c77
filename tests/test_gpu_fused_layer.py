"""The fused GraphSAGE layer kernel (k_sage_fused3, csrc/cuda/sage_tc.cu) at every shape, source and degree it accepts,
against float64 references.

One launch gathers the rows of a sampled batch, takes the neighbour mean, multiplies [mean | self] with W on wgmma and
applies bias and ReLU.  Each test builds the sampler's layout by hand -- per-hop ELL blocks, `deg`, int32 counters,
source rows -- so that every edge case is placed on purpose, and checks the launch in two stages through `a_save`, the
A tile the kernel multiplies:

  1. A.  The mean half against the float64 mean of the rows the kernel reads: a -1 slot, or a node id the feature
     table does not hold, adds zero and still counts in the degree.  The self half equals the source row (zeros for a
     missing id).  Both halves equal `sage_aggregate`'s output bit for bit: both kernels sum in fp32 in ELL-slot order
     and round once.
  2. Z given A.  Against act(A W^T + b) in float64, within helpers.gemm_bound.  Z from a launch without `a_save` is
     the same bits.

The degrees sit on both sides of every loader boundary: the bf16 loader takes the self row and neighbours 0-4 in its
first batch, then batches of 5, up to the 15 slots of the resolvers' handle table; the MXFP8 loader takes 1 + 7, then
8; both chase slots 15 and up themselves.
"""
import pytest
import torch

from graphlearn_for_pytorch_b200.data import dequantize_mxfp8, quantize_mxfp8
from helpers import bf16_ulp, bound_ratio, gemm_bound

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
SENTINEL = 7.0
EPS32 = 2.0 ** -23

# (k, degrees of the first rows): a hub hop, a hop wider than the handle table, one exactly as wide, one narrower
HOPS = [(512, [512, 0, 1, 16, 17, 200]),
        (20, [0, 1, 5, 6, 7, 8, 10, 11, 14, 15, 16, 17, 20]),
        (15, [0, 1, 5, 6, 7, 8, 10, 11, 14, 15]),
        (7, [0, 1, 5, 6, 7])]
HOP_ROWS = (6, 200, 300)          # rows of the first three hops (boundaries inside tiles); the last hop takes the rest
RESIDUES = (1, 63, 64, 65, 127)   # T mod 128: one row, both 64-row halves of a tile, the ragged last tile
SHAPES = [(d, n) for d in (64, 128) for n in range(32, 257, 32)]
N_OUT = list(range(32, 257, 32))
MISS_STRIDE = 29                  # table sources: batch node s is missing from the table when s % 29 == 0


class Batch:
  """Per-hop ELL blocks of HOPS for T target rows over sources [0, n_src) (targets are sources 0 .. T-1).  Slots past
  a row's degree hold valid ids that must not be read; about 5% of the slots inside it hold -1 (a neighbour the
  sampler dropped: it adds nothing but still counts in the mean's divisor)."""

  def __init__(self, T, seed):
    g = torch.Generator().manual_seed(seed)
    self.T, self.n_src = T, T + 200
    rows = list(HOP_ROWS) + [T - sum(HOP_ROWS)]
    self.cum, degs, self.ells = [0], [], []
    for (k, heads), n in zip(HOPS, rows):
      deg = torch.randint(0, k + 1, (n,), generator=g)
      deg[:len(heads)] = torch.tensor(heads)
      ell = torch.randint(0, self.n_src, (n, k), generator=g)
      ell[torch.rand(n, k, generator=g) < 0.05] = -1
      self.ells.append(ell.to(torch.int32))
      degs.append(deg.to(torch.int32))
      self.cum.append(self.cum[-1] + n)
    m = MISS_STRIDE
    hub, wide = self.ells[0], self.ells[1]
    # -1 and missing ids inside the degree, below and from slot 15 on: the hub row (degree 512) and hop 1's degree-17
    # row (head 11); hop 1's degree-16 row (head 10) keeps a present row in slot 15, the first slot the loaders chase
    hub[0, 2], hub[0, 100], hub[0, 3], hub[0, 200] = -1, -1, m, 2 * m
    wide[11, 5], wide[11, 16], wide[11, 4], wide[11, 15] = -1, -1, 3 * m, 4 * m
    wide[10, 15] = 1
    self.deg = torch.cat(degs)
    self.ks = [k for k, _ in HOPS]
    self.ell_d = [e.flatten().to(DEV) for e in self.ells]
    self.deg_d = self.deg.to(DEV)

  def counters(self, total=None):
    c = torch.zeros(16, dtype=torch.int32)
    c[:len(self.cum)] = torch.tensor(self.cum, dtype=torch.int32)
    if total is not None:
      c[len(self.cum) - 1] = total
    return c.to(DEV)

  def edges(self, T):
    """(target, source) of every slot of the first T rows that adds a row: inside the degree, not -1."""
    tg, sr = [], []
    for h, (k, _) in enumerate(HOPS):
      n = max(0, min(T, self.cum[h + 1]) - self.cum[h])
      if n == 0:
        continue
      e = self.ells[h][:n].long()
      mask = (torch.arange(k).unsqueeze(0) < self.deg[self.cum[h]:self.cum[h] + n].long().unsqueeze(1)) & (e >= 0)
      tg.append((torch.arange(n).unsqueeze(1) + self.cum[h]).expand(n, k)[mask])
      sr.append(e[mask])
    return torch.cat(tg).to(DEV), torch.cat(sr).to(DEV)


class Source:
  """The rows the kernel reads.  `Xs[s]` (bf16 [n_src, d]) is what batch node s contributes: its feature row, the
  bf16 value of its de-quantised MXFP8 row, or zeros for an id the table does not hold.

  kind: 'local'  dense bf16 rows (deeper layers: the self row of target t is row t)
        'hbm'    a one-part table in HBM          'split'       one part in HBM, one in pinned host memory
        'parts16' 16 uneven parts (a 1-row part first) alternating between HBM and pinned host memory
        'mxfp8'  a one-part MXFP8 table in HBM    'mxfp8_split' an MXFP8 table split between HBM and host memory
  Table sources map every 29th batch node to an id past the table's last row."""

  def __init__(self, native, kind, n_src, d, seed):
    g = torch.Generator().manual_seed(seed)
    self.kind = kind
    if kind == 'local':
      self.Xs = (torch.randn(n_src, d, generator=g) * 2).to(torch.bfloat16).to(DEV)
      self.feat, self.nodes, self.local = None, None, self.Xs
      return
    n_glob = n_src + 97
    if kind.startswith('mxfp8'):
      x = torch.randn(n_glob, d, generator=g) * torch.exp2(
          torch.randint(-6, 7, (n_glob, d // 32), generator=g).float()).repeat_interleave(32, 1)
      rows = quantize_mxfp8(x)
      X = dequantize_mxfp8(rows, d).to(torch.bfloat16)
    else:
      X = (torch.randn(n_glob, d, generator=g) * 2).to(torch.bfloat16)
      rows = X
    if kind in ('hbm', 'mxfp8'):
      bounds = [0, n_glob]
    elif kind in ('split', 'mxfp8_split'):
      bounds = [0, n_glob // 3, n_glob]
    else:
      cuts = torch.randperm(n_glob - 2, generator=g)[:14] + 2
      bounds = [0, 1] + sorted(cuts.tolist()) + [n_glob]
    self.feat = native.RowTableHandle(0)
    for p in range(len(bounds) - 1):
      part = rows[bounds[p]:bounds[p + 1]]
      self.feat.append(part.to(DEV) if p % 2 == 0 else part.clone().pin_memory(), False)
    assert self.feat.num_rows() == n_glob and self.feat.num_parts == len(bounds) - 1
    nodes = torch.randperm(n_glob, generator=g)[:n_src]
    miss = torch.arange(0, n_src, MISS_STRIDE)
    nodes[miss] = n_glob + torch.arange(len(miss))
    Xs = torch.zeros(n_src, d, dtype=torch.bfloat16)
    present = nodes < n_glob
    Xs[present] = X[nodes[present]]
    self.Xs, self.nodes, self.local = Xs.to(DEV), nodes.to(DEV), None


def _weights(n_out, d, seed):
  g = torch.Generator().manual_seed(seed)
  W = (torch.randn(n_out, 2 * d, generator=g) / (2 * d) ** 0.5).to(torch.bfloat16).to(DEV)
  bias = (torch.randn(n_out, generator=g) * 0.5).to(torch.bfloat16).to(DEV)
  return W, bias


def _mean_oracle(b, Xs, T):
  """float64 sums, means and bounds of the first T rows: one bf16 ulp of the mean, plus the fp32 sum of dg rows and
  the multiplication by the fp32 1/dg (the bound of test_sage_aggregate_matches_fp64_mean)."""
  d = Xs.shape[1]
  tg, sr = b.edges(T)
  Xd = Xs.double()
  s = torch.zeros(T, d, dtype=torch.float64, device=DEV).index_add_(0, tg, Xd[sr])
  a = torch.zeros(T, d, dtype=torch.float64, device=DEV).index_add_(0, tg, Xd[sr].abs())
  dg = b.deg[:T].to(DEV).double().unsqueeze(1)
  ref = s / dg.clamp(min=1)
  bound = torch.where(dg > 0, bf16_ulp(ref) + (dg + 2) * EPS32 * a / dg.clamp(min=1), torch.zeros_like(ref))
  return s, ref, bound


def _z_oracle(A, W, bias, relu):
  """act(A W^T + b) in float64 and its bound: a bf16 GEMM with fp32 accumulation over k = 2d products plus the bias."""
  Ad, Wd, bd = A.double(), W.double(), bias.double()
  ref = Ad @ Wd.t() + bd
  if relu:
    ref = ref.clamp(min=0)
  return ref, gemm_bound(ref, Ad.abs() @ Wd.abs().t() + bd.abs(), A.shape[1] + 1)


def _launch(native, b, src, d, wp, bias, relu, ctr, z, a_save=None):
  native.sage_fused(src.feat, src.nodes, src.local, d, ctr, len(HOPS), b.ell_d, b.ks, b.deg_d, wp, bias, relu, z,
                    a_save)


def _case(native, d, n_out, kind, T, relu, seed):
  """Runs the kernel on one batch with spare rows above it, then with counters above the capacity (T is clamped to
  z's rows); checks both stages.  Returns the first run's results and references, and the largest ratios."""
  b = Batch(T, seed)
  src = Source(native, kind, b.n_src, d, seed + 1)
  W, bias = _weights(n_out, d, seed + 2)
  wp = native.pack_weight(W)
  ratios = [0.0, 0.0]
  first = None
  for cap, total in ((T + 37, None), (T - 50, T + 1000)):
    ctr = b.counters(total)
    Te = min(T if total is None else total, cap)
    z = torch.full((cap, n_out), SENTINEL, dtype=torch.bfloat16, device=DEV)
    A = torch.full((cap + 3, 2 * d), SENTINEL, dtype=torch.bfloat16, device=DEV)
    z2 = torch.full_like(z, SENTINEL)
    agg = torch.full((cap, 2 * d), SENTINEL, dtype=torch.bfloat16, device=DEV)
    _launch(native, b, src, d, wp, bias, relu, ctr, z, A)
    _launch(native, b, src, d, wp, bias, relu, ctr, z2)
    native.sage_aggregate(src.feat, src.nodes, src.local, d, ctr, len(HOPS), b.ell_d, b.ks, b.deg_d, agg)
    torch.cuda.synchronize()
    where = (d, n_out, kind, relu, cap, Te)

    s, ref_m, bound_m = _mean_oracle(b, src.Xs, Te)
    rm = bound_ratio(A[:Te, :d], ref_m, bound_m)
    assert rm <= 1.0, ('mean', where, rm)
    assert torch.equal(A[:Te, d:], src.Xs[:Te]), ('the self half must be the source row', where)
    assert torch.equal(A[:Te].view(torch.int16), agg[:Te].view(torch.int16)), \
        ('the A tile must be sage_aggregate\'s output, bit for bit', where)
    assert bool((A[Te:] == SENTINEL).all()), ('a_save rows at and above T must not be written', where)

    ref_z, bound_z = _z_oracle(A[:Te], W, bias, relu)
    rz = bound_ratio(z[:Te], ref_z, bound_z)
    assert rz <= 1.0, ('z', where, rz)
    assert torch.equal(z.view(torch.int16), z2.view(torch.int16)), ('z must not depend on a_save', where)
    assert bool((z[Te:] == SENTINEL).all()), ('z rows at and above T must not be written', where)
    ratios = [max(ratios[0], rm), max(ratios[1], rz)]
    if first is None:
      first = dict(b=b, src=src, W=W, bias=bias, A=A[:Te], z=z[:Te], s=s, ref_m=ref_m, bound_m=bound_m,
                   ref_z=ref_z, bound_z=bound_z)
  print(f'fused d={d} n_out={n_out} {kind} relu={relu} T={T}: max error / bound = {ratios[0]:.3f} (mean), '
        f'{ratios[1]:.3f} (z)')
  return first


# --------------------------------------------------------------------------- every shape and source
CASES = [(d, n, kind) for kind in ('local', 'hbm', 'split', 'parts16') for d, n in SHAPES] + \
        [(128, n, kind) for kind in ('mxfp8', 'mxfp8_split') for n in N_OUT]


@pytest.mark.parametrize('d,n_out,kind', CASES)
def test_fused_layer_matches_fp64(native, d, n_out, kind):
  i = CASES.index((d, n_out, kind))
  T = 8 * 128 + RESIDUES[i % len(RESIDUES)]
  relu = (n_out // 32 + d // 64 + i // len(SHAPES)) % 2 == 0    # alternates along n_out, flips with d and source
  _case(native, d, n_out, kind, T, relu, seed=1000 + i)


@pytest.mark.parametrize('d,n_out,kind', [(128, 160, 'hbm'), (64, 224, 'local'), (128, 96, 'mxfp8')])
def test_fused_layer_many_tiles_per_cta(native, d, n_out, kind):
  """At least five tiles per CTA: every CTA reuses both handle-table stages and wraps every mbarrier parity."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  T = 5 * 128 * sms + 63
  _case(native, d, n_out, kind, T, relu=True, seed=7)


@pytest.mark.parametrize('kind', ['local', 'hbm'])
def test_fused_layer_zero_counters_write_nothing(native, kind):
  d, n_out, cap = 128, 96, 300
  b = Batch(1100, seed=3)
  src = Source(native, kind, b.n_src, d, seed=4)
  W, bias = _weights(n_out, d, seed=5)
  z = torch.full((cap, n_out), SENTINEL, dtype=torch.bfloat16, device=DEV)
  A = torch.full((cap, 2 * d), SENTINEL, dtype=torch.bfloat16, device=DEV)
  _launch(native, b, src, d, native.pack_weight(W), bias, True, torch.zeros(16, dtype=torch.int32, device=DEV), z, A)
  torch.cuda.synchronize()
  assert bool((z == SENTINEL).all()) and bool((A == SENTINEL).all())


# --------------------------------------------------------------------------- the bounds have teeth
def test_bounds_reject_plausible_defects(native):
  """The defects this kernel could plausibly have, applied in Python to its results, each exceed their bound."""
  d, n_out = 128, 96
  r = _case(native, d, n_out, 'hbm', 8 * 128 + 65, relu=False, seed=11)
  b, Xs, A, z = r['b'], r['src'].Xs, r['A'], r['z']
  assert bound_ratio(A[:, :d], r['ref_m'], r['bound_m']) <= 1.0
  assert bound_ratio(z, r['ref_z'], r['bound_z']) <= 1.0
  deg = b.deg.tolist()

  def mean_ratio(t, row):
    bad = A[:, :d].clone()
    bad[t] = row.to(torch.bfloat16)
    return bound_ratio(bad, r['ref_m'], r['bound_m'])

  # a 16-neighbour row whose slot 15 is a present node: drop slot 15 from its mean
  t = b.cum[1] + 10
  s15 = int(b.ells[1][10, 15])
  assert deg[t] == 16 and s15 >= 0 and bool(Xs[s15].abs().sum() > 0)
  drop = mean_ratio(t, (r['s'][t] - Xs[s15].double()) / 16)
  # divide a mean by dg - 1 (hop 1's degree-5 row)
  t = b.cum[1] + 2
  assert deg[t] == 5
  off_by_one = mean_ratio(t, r['s'][t] / 4)
  # zero the 32-column tail block of a row; swap two columns of one 64-column block of a row
  t = 700
  tail = z.clone()
  tail[t, 64:96] = 0
  c0, c1 = 5, 41
  t_sw = int((z[:, c0].double() - z[:, c1].double()).abs().argmax())
  swap = z.clone()
  swap[t_sw, c0], swap[t_sw, c1] = z[t_sw, c1], z[t_sw, c0]
  tail_r = bound_ratio(tail, r['ref_z'], r['bound_z'])
  swap_r = bound_ratio(swap, r['ref_z'], r['bound_z'])
  print(f'defects: error / bound = {drop:.1f} (slot 15 dropped), {off_by_one:.1f} (mean / (dg - 1)), '
        f'{tail_r:.1f} (tail block zeroed), {swap_r:.1f} (two columns swapped)')
  assert drop > 1.0 and off_by_one > 1.0 and tail_r > 1.0 and swap_r > 1.0


# --------------------------------------------------------------------------- the contract of the binding
def test_sage_fused_supported_is_exactly_the_grid(native):
  for d in (0, 8, 32, 63, 64, 65, 96, 128, 192, 256):
    for n_out in (0, 8, 16, 31, 32, 48, 64, 80, 96, 112, 128, 160, 192, 224, 240, 256, 264, 288, 320, 512):
      want = int(d in (64, 128) and n_out % 32 == 0 and 32 <= n_out <= 256)
      assert int(native.sage_fused_supported(d, n_out)) == want, (d, n_out)


def test_sage_fused_rejects_unsupported_shapes(native):
  b = Batch(1100, seed=21)

  def call(d, n_out, kind='local'):
    src = Source(native, kind, b.n_src, d, seed=22)
    W, bias = _weights(n_out, d, seed=23)
    wp = W.flatten().clone()             # right size; never read by a launch that is rejected
    z = torch.full((64, n_out), SENTINEL, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError):
      _launch(native, b, src, d, wp, bias, True, b.counters(), z)
    torch.cuda.synchronize()
    assert bool((z == SENTINEL).all()), (d, n_out, kind)

  for d in (32, 96, 192, 256):
    call(d, 64)
  for n_out in (16, 48, 80, 240, 288, 320):
    call(64, n_out)
  for d in (64, 256):
    call(d, 64, 'mxfp8')


@pytest.mark.parametrize('d,n_out', SHAPES)
def test_pack_weight_roundtrip_on_the_grid(native, d, n_out):
  """W [N, K] -> [K/64][N][64] with the 16-byte chunks of row n XOR-swizzled by (n & 7); undone here."""
  K = 2 * d
  w = torch.randn(n_out, K, generator=torch.Generator().manual_seed(K + n_out)).to(torch.bfloat16).to(DEV)
  p = native.pack_weight(w).view(K // 64, n_out, 8, 8)
  rows = torch.arange(n_out, device=DEV)
  out = torch.empty_like(p)
  for cv in range(8):
    out[:, rows, cv] = p[:, rows, cv ^ (rows & 7)]
  assert torch.equal(out.permute(1, 0, 2, 3).reshape(n_out, K), w)
