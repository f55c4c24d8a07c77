"""The GraphSAGE backward of the mean aggregation (csrc/cuda/transpose.cu) against exact and float64 references.

Every training step of GraphSageEngine / GraphSageLinkEngine runs it in two pieces: the sampler transposes the batch's
adjacency (k_tr_count, the three-phase scan, k_tr_fill, k_tr_meta), and k_sage_gather_bwd walks it per source row:
dPre[s] = relu'(Z[s]) * gscale * (dA[s, d:2d] if s < T + sum_t dA[t, :d] / deg[t]), with the bias column sums fused.

* The transposed adjacency is checked exactly (integers and fp32 1/deg bit for bit) on batches laid into the arena by
  hand: ELL slots past a row's degree holding valid ids, -1 entries inside the degree, duplicate sources, 1 to 4
  transposed hops, counters above `cap_rows` and above `cap_nodes`, more than 1024 scan blocks, and a second build on
  the same arena.
* k_sage_gather_bwd is checked at every lane-group shape against a float64 reference on one hand-built batch whose
  in-batch in-degrees sit on every branch of the kernel: the record path (0-2 in-edges), the batches of in-edges past
  the first two, the kHeavy = 24 threshold, rows split over a team of warps (hubs of up to 5000 in-edges, several in
  one 32-row chunk, a chunk of 32 hubs, a hub as the last source) and rows past one grid sweep.
* The engine's own step is checked layer by layer against the same reference, built from the arena it trained on.

Each comparison is a bound (tests/helpers.py): one bf16 ulp of the result plus (n + 3) * 2^-23 * gscale * sum|terms| for
an fp32 sum of n terms; masked rows, rows past the batch and rows past the buffer are compared exactly.
"""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageEngine
from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges
from helpers import bound_ratio, colsum_ratio, gather_ref
from test_gpu_kernel_widths import AGG_WIDTHS

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
SENTINEL = 7.0


# --------------------------------------------------------------------------- hand-built batches
def _hop(rows, k, design, pool_hi, exclude, g, deg_lo=0, holes=0.03):
  """deg [rows] and ELL block [rows, k] of one hop.  Sources in `design` get exactly their in-degree; the other slots
  inside the degrees draw sources from [0, pool_hi) minus `exclude` (a few of them -1, which the kernels skip); slots
  past a row's degree hold valid ids.  The first three rows have degree 0, 1 and k."""
  deg = torch.randint(deg_lo, k + 1, (rows,), generator=g)
  deg[:3] = torch.tensor([0, 1, k])
  n_slots = int(deg.sum())
  fixed = torch.repeat_interleave(torch.tensor(list(design.keys()), dtype=torch.int64),
                                  torch.tensor(list(design.values()), dtype=torch.int64))
  assert fixed.numel() <= n_slots
  pool = torch.ones(pool_hi, dtype=torch.bool)
  pool[[s for s in exclude if s < pool_hi]] = False
  pool = pool.nonzero().squeeze(1)
  fill = pool[torch.randint(0, pool.numel(), (n_slots - fixed.numel(),), generator=g)]
  fill[torch.rand(fill.numel(), generator=g) < holes] = -1
  vals = torch.cat([fixed, fill])[torch.randperm(n_slots, generator=g)]
  ell = torch.randint(0, pool_hi, (rows, k), generator=g)
  ell[torch.arange(k).unsqueeze(0) < deg.unsqueeze(1)] = vals
  return deg.to(torch.int32), ell.to(torch.int32)


def _lay_out(ar, cum, hops, g):
  """Writes a batch into the arena's sampler state: counters[:len(cum)] = cum and, per hop h, the degrees of the
  frontier rows from cum[h] on and the ELL rows (up to cap_rows[h]; the ELL rows after them keep random valid ids)."""
  c = torch.zeros(16, dtype=torch.int32)
  c[:len(cum)] = torch.tensor(cum, dtype=torch.int32)
  ar.counters.copy_(c)
  ar.deg.zero_()
  for h, (deg, ell) in enumerate(hops):
    cap = ar.cap_rows[h] * ar.fanouts[h]
    full = torch.randint(0, ar.cap_nodes, (cap,), generator=g, dtype=torch.int32)
    e = ell.flatten()[:cap]
    full[:e.numel()] = e
    ar.ell[h].copy_(full)
    ar.deg[cum[h]:cum[h] + deg.numel()].copy_(deg)


def _edges(cum, hops, cap_rows, cap_nodes):
  """(hop, target, source) of every edge of the batch: frontier rows clamped to cap_rows, slots inside the degree,
  sources in [0, cap_nodes)."""
  hs, ts, ss = [], [], []
  for h, (deg, ell) in enumerate(hops):
    n = min(cum[h + 1] - cum[h], cap_rows[h])
    k = ell.shape[1]
    e = ell[:n].long()
    m = (torch.arange(k).unsqueeze(0) < deg[:n].long().unsqueeze(1)) & (e >= 0) & (e < cap_nodes)
    ts.append((torch.arange(n).unsqueeze(1) + cum[h]).expand(n, k)[m])
    ss.append(e[m])
    hs.append(torch.full((ss[-1].numel(),), h, dtype=torch.int64))
  return torch.cat(hs), torch.cat(ts), torch.cat(ss)


# --------------------------------------------------------------------------- transposed adjacency
def _check_transpose(ar, cum, hops):
  """Exact check of tr_cnt, tr_off, the segments, tr_meta and tr_meta_inv against the batch's edges."""
  torch.cuda.synchronize()
  H, N = ar.tr_hops, ar.cap_nodes
  hop, tgt, src = _edges(cum, hops[:H], ar.cap_rows, N)
  cnt_exp = torch.zeros(H, N, dtype=torch.int64)
  cnt_exp.index_put_((hop, src), torch.ones_like(src), accumulate=True)
  cnt_exp = cnt_exp.cumsum(0)                                   # cumulative over hops 0..h
  assert torch.equal(ar.tr_cnt.cpu().long(), cnt_exp), 'tr_cnt[h][s] must be the in-count over hops 0..h'
  total = cnt_exp[-1]
  off_exp = torch.zeros(N + 1, dtype=torch.int64)
  off_exp[1:] = total.cumsum(0)
  off = ar.tr_off.cpu().long()
  assert torch.equal(off, off_exp), 'tr_off must be the exclusive scan of the in-counts, tr_off[cap_nodes] the total'
  E = int(off_exp[-1])
  tg_all = ar.tr_tgt.cpu().long()
  seg = tg_all[:E]
  # every slot of the segments: its source, and the hop its rank falls in ([cnt[h-1][s], cnt[h][s]) is hop h)
  owner = torch.repeat_interleave(torch.arange(N), total)
  rank = torch.arange(E) - off_exp[owner]
  slot_hop = (rank.unsqueeze(0) >= cnt_exp[:, owner]).sum(0)
  got = torch.sort((owner * H + slot_hop) * N + seg).values
  exp = torch.sort((src * H + hop) * N + tgt).values
  assert torch.equal(got, exp), 'the first tr_cnt[h][s] entries of a segment must be the targets of hops 0..h'
  # records {segment start, first two targets, total} and their fp32 1/deg, for the sources of the batch
  n_nodes = min(cum[H + 1], N)
  first = torch.where(total > 0, tg_all[off[:N].clamp(max=tg_all.numel() - 1)], -1)
  second = torch.where(total > 1, tg_all[(off[:N] + 1).clamp(max=tg_all.numel() - 1)], -1)
  meta_exp = torch.stack([off[:N], first, second, total], 1)
  meta_exp[n_nodes:] = torch.tensor([0, -1, -1, 0])
  assert torch.equal(ar.tr_meta.cpu().long(), meta_exp), 'tr_meta[s] must be {off, seg[0], seg[1], total}'
  degf = ar.deg.cpu().float()
  inv = lambda t: torch.where(t >= 0, 1.0 / degf[t.clamp(min=0)], torch.zeros(()))   # fp32 division, as the kernel's
  inv_exp = torch.stack([inv(first), inv(second)], 1)
  inv_exp[n_nodes:] = 0.0
  assert torch.equal(ar.tr_meta_inv.cpu().view(torch.int32), inv_exp.view(torch.int32)), \
      'tr_meta_inv must be fp32 1/deg of the first two targets, bit for bit'
  return E


TRANSPOSE_CASES = [
    # name, max_seeds, fanouts, cap_override, transposed hops, counters
    ('1hop-k512', 64, [512], [], 1, [0, 64, 20000]),
    # cap_nodes = 1,082,368 > 1024 * 1024: the scan carries across more than 1024 block sums; hop 1 has more rows than
    # cap_rows[1] = 32768 and the batch more nodes than cap_nodes
    ('2hops-1M-nodes', 1024, [32, 32], [], 2, [0, 1024, 40000, 1082368 + 5000]),
    # calibrated capacities cap_rows = [256, 1000, 2000, 3000], cap_nodes = 6256: hop 2 and the batch exceed them
    ('3hops-calibrated', 256, [8, 4, 3], [256, 1000, 2000, 3000], 3, [0, 256, 1100, 3500, 6500]),
    ('4hops', 64, [4, 3, 3, 2], [], 4, [0, 64, 300, 1000, 3000, 7000]),
    ('4hop-arena-2-transposed', 64, [4, 3, 3, 2], [], 2, [0, 64, 300, 1000, 3000, 7000]),
]


@pytest.mark.parametrize('case', TRANSPOSE_CASES, ids=[c[0] for c in TRANSPOSE_CASES])
def test_transposed_adjacency_is_exact(native, case):
  """Integer-exact transposed adjacency and per-source records; the second batch is built on the same arena (the
  per-build memsets of the counts and cursors) and must come out as a fresh build would."""
  name, max_seeds, fanouts, cap_override, tr_hops, cum = case
  ar = native.SamplerArena(0, max_seeds, fanouts, False, 0, cap_override)
  ar.enable_transpose(tr_hops)
  g = torch.Generator().manual_seed(len(name))
  for rebuild in (False, True):
    if rebuild:                                              # a different, smaller batch into the same buffers
      cum = [0] + [c * 4 // 5 for c in cum[1:]]
    hops = []
    for h in range(tr_hops):
      k = fanouts[h]
      deg, ell = _hop(cum[h + 1] - cum[h], k, {}, min(cum[h + 2], ar.cap_nodes), (), g)
      deg[3] = k
      ell[3] = ell[3, 0]                                     # a row sampling one source k times (with replacement)
      hops.append((deg, ell))
    _lay_out(ar, cum, hops, g)
    ar.build_transpose()
    E = _check_transpose(ar, cum, hops)
    print(f'transpose {name} rebuild={rebuild}: {E} transposed edges over {ar.cap_nodes} nodes exact')


# --------------------------------------------------------------------------- sage_gather_bwd
# counters of the gather batch: 600 seeds, hop-1 frontier to 3000, hop-2 frontier to 33000, 310,000 nodes in all
# (S % 32 == 16); one grid sweep of the kernel covers 67,584 / 135,168 / 270,336 rows for 4 / 2 / 1 warps per 32 rows
CUM = [0, 600, 3000, 33000, 310000]
# in-batch in-degrees placed on purpose (hop 0, sources < 3000), exact for every prefix of hops: every count 0..40
# (the record path, U, the batches of in-edges past the first two at 2 + {HB, LPR} +- 1, kHeavy = 24 / 25); hubs at
# lanes 0, 10, 20 and 31 of the chunk [64, 96), one of 5000 in-edges; a chunk [96, 128) of 32 hubs; 63, 65 and 257
HOP0_DESIGN = {s: s for s in range(41)}
HOP0_DESIGN.update({64: 129, 74: 25, 84: 64, 95: 5000})
HOP0_DESIGN.update({96 + i: 25 + i for i in range(32)})
HOP0_DESIGN.update({200: 63, 201: 65, 202: 257})
# hop 2: hubs past one grid sweep of every lane-group shape, lane 31 of a chunk, and the last source of the batch
HOP2_DESIGN = {70000: 200, 140001: 130, 280031: 27, 290000: 40, CUM[4] - 1: 30}

GATHER_CONFIGS = [
    # n_hops_targets, rows of dA (None: cum[n]), rows of dPre, with Z, gscale, bias sums
    (3, None, CUM[4] + 40, True, 1.0 / (1.0 - 0.3), 'prezeroed'),
    (3, CUM[3] - 300, CUM[4] - 50, True, 1.0, 'memset'),      # counters above both buffers
    (2, None, CUM[3] + 33, False, 1.0 / (1.0 - 0.3), 'memset'),  # no ReLU mask: the dropout scale alone
    (1, CUM[1] - 100, CUM[2] + 7, True, 1.0 / (1.0 - 0.3), None),
    (2, CUM[2] - 1, CUM[3], False, 1.0, 'prezeroed'),
]


@pytest.fixture(scope='module')
def gather_batch(native):
  ar = native.SamplerArena(0, 1024, [32, 16, 2], False, 0)
  ar.enable_transpose(3)
  g = torch.Generator().manual_seed(11)
  excl = set(HOP0_DESIGN) | set(HOP2_DESIGN)
  hops = [_hop(CUM[1] - CUM[0], 32, HOP0_DESIGN, CUM[2], excl, g, deg_lo=8),
          _hop(CUM[2] - CUM[1], 16, {}, CUM[3], excl, g),
          _hop(CUM[3] - CUM[2], 2, HOP2_DESIGN, CUM[4], excl, g)]
  _lay_out(ar, CUM, hops, g)
  ar.build_transpose()
  _check_transpose(ar, CUM, hops)
  hop, tgt, src = _edges(CUM, hops, ar.cap_rows, ar.cap_nodes)
  indeg = torch.bincount(src, minlength=CUM[4])
  for s, n in {**HOP0_DESIGN, **HOP2_DESIGN}.items():
    assert int(indeg[s]) == n, (s, n)
  yield ar, hop.to(DEV), tgt.to(DEV), src.to(DEV)
  del ar
  torch.cuda.empty_cache()


@pytest.mark.parametrize('d', AGG_WIDTHS)
def test_sage_gather_bwd_matches_fp64(native, gather_batch, d):
  ar, hop, tgt, src = gather_batch
  g = torch.Generator(device=DEV).manual_seed(d)
  ratios = []
  for n_hops, rows_dA, cap_src, with_z, gscale, bias in GATHER_CONFIGS:
    rows_dA = CUM[n_hops] if rows_dA is None else rows_dA
    T, S = min(CUM[n_hops], rows_dA), min(CUM[n_hops + 1], cap_src)
    dA = (torch.randn(rows_dA, 2 * d, device=DEV, generator=g) * 0.5).to(torch.bfloat16)
    Z = None
    if with_z:
      Z = torch.randn(cap_src + 16, d, device=DEV, generator=g).to(torch.bfloat16)
      r = torch.rand(Z.shape, device=DEV, generator=g)
      Z.masked_fill_(r < 0.1, 0.0)
      Z.masked_fill_((r >= 0.1) & (r < 0.2), -0.0)
      assert bool((Z.view(torch.int16) == -32768).any()), 'Z must hold -0.0'
    full = torch.full((cap_src + 64, d), SENTINEL, dtype=torch.bfloat16, device=DEV)
    dPre = full[:cap_src]
    init = {'prezeroed': 0.25, 'memset': 12345.0, None: 0.0}[bias]
    cbuf = torch.full((d + 8,), init, dtype=torch.float32, device=DEV)
    colsum = cbuf[:d] if bias else None
    native.sage_gather_bwd(dA, d, ar, n_hops, Z, dPre, colsum, bias == 'prezeroed', gscale)
    torch.cuda.synchronize()
    sel = hop < n_hops
    ref, bound = gather_ref(dA, d, Z, tgt[sel], src[sel], ar.deg, T, S, cap_src, gscale)
    case = (d, n_hops, rows_dA, cap_src, with_z, round(gscale, 4), bias)
    r = bound_ratio(dPre, ref, bound)
    assert r <= 1.0, f'dPre off its float64 reference {case}: error / bound = {r}'
    assert bool((full[cap_src:] == SENTINEL).all()), f'rows past dPre must stay untouched {case}'
    rc = 0.0
    if bias:
      rc = colsum_ratio(colsum, dPre, S, init if bias == 'prezeroed' else 0.0)
      assert rc <= 1.0, f'bias column sums off {case}: error / bound = {rc}'
      assert bool((cbuf[d:] == init).all()), f'columns past d must stay untouched {case}'
    ratios.append((n_hops, r, rc))
  print(f'gather_bwd d={d}: max error / bound per config (hops, dPre, bias) = '
        + ', '.join(f'({n}, {r:.3f}, {rc:.2e})' for n, r, rc in ratios))


# --------------------------------------------------------------------------- the engine's step
def _hub_engine(fanouts, hidden, dropout, pipeline, calibrated):
  """GraphSageEngine over an RMAT graph plus one node adjacent to every other, so that a batch holds sources with
  far more than 128 in-batch in-edges."""
  N, hub = 6000, 17
  ei = rmat_edges(N, 30000, seed=3)
  v = torch.arange(N)
  ei = torch.cat([ei, torch.stack([v, torch.full_like(v, hub)]), torch.stack([torch.full_like(v, hub), v])], 1)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=N)
  g = glt.data.Graph(topo, 'CUDA', 0)
  torch.manual_seed(0)
  feats = torch.randn(N, 128, device=DEV).to(torch.bfloat16)
  labels = torch.randint(0, 47, (N,), device=DEV)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageEngine(g, ut._table(), labels, in_dim=128, num_nodes=N, fanouts=fanouts, batch_size=256,
                        hidden=hidden, num_classes=47, device=DEV, use_fused=(hidden <= 256), use_cuda_graph=False,
                        seed=5, pipeline=pipeline, dropout=dropout,
                        calibration_seeds=torch.arange(N) if calibrated else None)
  assert eng.calibrated == calibrated
  eng._keep = (ut, feats, topo)
  return eng, N


def _arena_hops(ar, c, n):
  hops = []
  for h in range(n):
    k = ar.fanouts[h]
    rows = max(0, min(c[h + 1] - c[h], ar.cap_rows[h]))
    hops.append((ar.deg[c[h]:c[h] + rows].cpu(), ar.ell[h][:rows * k].view(rows, k).cpu()))
  return hops


ENGINE_CASES = [
    # fanouts, hidden, dropout, pipeline, calibrated
    ([5, 4, 3], 64, 0.3, False, False),
    ([5, 4, 3], 128, 0.0, True, False),
    ([5, 4, 3, 2], 256, 0.3, False, True),
    ([5, 4, 3], 512, 0.3, True, False),
    ([5, 4, 3, 2], 1024, 0.3, False, False),
    ([5, 4, 3, 2], 128, 0.3, True, True),
]


@pytest.mark.parametrize('fanouts,hidden,dropout,pipeline,calibrated', ENGINE_CASES)
def test_engine_gather_backward_matches_fp64(native, fanouts, hidden, dropout, pipeline, calibrated):
  """dPre[l-1] and the bias gradient of layer l-1 of a real step, for every layer l >= 2, recomputed in float64 from
  the step's own dA[l], Z[l-1] (after dropout) and the arena it sampled: checks the hop prefix L - l + 1, the buffer
  row counts and the dropout scale the engine hands to the kernel.  Pipelined engines are checked on both arenas."""
  eng, N = _hub_engine(fanouts, hidden, dropout, pipeline, calibrated)
  L = eng.L
  gscale = 1.0 / (1.0 - dropout)
  out = []
  for parity in ((0, 1) if pipeline else (0,)):
    eng._cur = parity
    eng.seeds_dev.copy_(torch.randperm(N, device=DEV)[:eng.bs])
    eng._sample(); eng._forward(); eng._backward()
    torch.cuda.synchronize()
    ar = eng.arena
    c = ar.counters[:L + 2].cpu().tolist()
    S2 = min(c[L], eng.dPre[1].shape[0])
    hub_in = int(ar.tr_cnt[L - 2, :S2].max())
    assert hub_in > 128, f'the batch must hold a source with more than 128 in-edges (max {hub_in})'
    for l in range(2, L + 1):
      n = L - l + 1
      dA, Z, dPre = eng.dA[l], eng.Z[l - 1], eng.dPre[l - 1]
      T, S = min(c[n], dA.shape[0]), min(c[n + 1], dPre.shape[0])
      _, tgt, src = _edges(c, _arena_hops(ar, c, n), ar.cap_rows, ar.cap_nodes)
      ref, bound = gather_ref(dA, hidden, Z, tgt.to(DEV), src.to(DEV), ar.deg, T, S, dPre.shape[0], gscale)
      r = bound_ratio(dPre, ref, bound)
      assert r <= 1.0, f'layer {l} (parity {parity}): dPre[{l - 1}] error / bound = {r}'
      boff, bn = eng._b_off[l - 2]
      rc = colsum_ratio(eng.g32[boff:boff + bn], dPre, S, 0.0)
      assert rc <= 1.0, f'layer {l} (parity {parity}): bias gradient of layer {l - 1} error / bound = {rc}'
      out.append(f'l={l}/p{parity}: {r:.3f} {rc:.2e}')
  print(f'engine fanouts={fanouts} hidden={hidden} dropout={dropout} pipeline={pipeline} calibrated={calibrated} '
        f'(max in-degree {hub_in}): dPre / bias error / bound ' + ', '.join(out))
