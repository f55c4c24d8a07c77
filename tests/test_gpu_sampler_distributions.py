"""The neighbour samplers against their exact draw distributions (float64), at every fanout bucket.

The CPU/GPU equality tests prove that both planes run the same algorithm; these prove that the algorithm draws what
it claims.  Every case samples a "star" CSR: N rows with the same local neighbourhood, row v's columns being
base[v] + position, so each pick maps back to a position.  Philox is keyed by the row id, so one launch is N
independent draws of one distribution; their counts are compared with the exact probabilities by chi-square (cells
with an expected count below 5 merged), or per position / per pair for rows too wide to enumerate.

Every statistical check prints its p-value and asserts p > 1e-6.  Seeds are fixed and Philox makes every outcome
deterministic, so a correct sampler cannot flake.  Picks of a row are compared as sorted subsets: the order of a
row's picks is not a uniform permutation (Floyd's output favours low positions first), and nothing relies on it.

Fanout buckets of the CUDA kernels (GLT_DISPATCH_FANOUT, cuda/sampling.cu): k <= 8 / 16 / 32 run one pick per lane on
8 / 16 / 32 lanes per row; k <= 128 / 512 run 4 / 16 picks per lane on 32 lanes.
"""
import itertools
import math

import numpy as np
import pytest
import torch
from scipy import integrate, stats

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.sampler import NeighborSampler

DEV = torch.device('cuda', 0)
PLANES = ['cpu', pytest.param('gpu', marks=pytest.mark.gpu)]
P_MIN = 1e-6
SEED = 0x5EED2026
KS = [1, 3, 8, 9, 16, 17, 32, 33, 128, 129, 512]
# weights spanning a 1e3 ratio, cycled over a row's positions
W7 = np.array([1.0, 1e-3 ** 0.5, 3.0, 1e3 ** 0.5, 0.1, 10.0, 1.0 / 3.0], dtype=np.float32)


# --------------------------------------------------------------------------- graphs
class Star:
  """CSR whose row v has deg[v] columns base[v] + (0, 1, ...), optional per-position weights (cycled)."""

  def __init__(self, deg, base=None, weights=None):
    self.deg = np.asarray(deg, dtype=np.int64)
    n = self.deg.size
    self.indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(self.deg, out=self.indptr[1:])
    self.base = self.indptr[:-1].copy() if base is None else np.asarray(base, dtype=np.int64)
    E = int(self.indptr[-1])
    pos = np.arange(E, dtype=np.int64) - np.repeat(self.indptr[:-1], self.deg)
    self.indices = np.repeat(self.base, self.deg) + pos
    self.weights = None
    if weights is not None:
      weights = np.asarray(weights, dtype=np.float32)
      self.weights = weights[pos % weights.size]
    self._graphs = {}

  @property
  def n(self):
    return self.deg.size

  def topo(self):
    return glt.data.Topology((torch.from_numpy(self.indptr), torch.from_numpy(self.indices)),
                             edge_weights=None if self.weights is None else torch.from_numpy(self.weights),
                             input_layout='CSR', layout='CSR')

  def graph(self, mode='CUDA'):
    if mode not in self._graphs:
      self._graphs[mode] = glt.data.Graph(self.topo(), mode, 0 if mode != 'CPU' else None)
    return self._graphs[mode]

  def handle(self, mode='CUDA'):
    return self.graph(mode).graph_handler

  def handle_int64(self):
    """A device graph keeping int64 column ids (the 'CUDA' mode narrows them to int32 when they fit)."""
    if 'int64' not in self._graphs:
      h = glt.ops.require_native().GraphHandle(0)
      w = None if self.weights is None else torch.from_numpy(self.weights).to(DEV)
      h.add_shard(torch.from_numpy(self.indptr).to(DEV), torch.from_numpy(self.indices).to(DEV),
                  torch.arange(self.indices.size, device=DEV), w, 0, self.n)
      self._graphs['int64'] = h
    return self._graphs['int64']

  def positions(self, rows, nbrs):
    """Positions of global neighbour ids `nbrs` in rows `rows` (row indices into this CSR)."""
    p = nbrs - self.base[rows]
    assert np.all((p >= 0) & (p < self.deg[rows])), 'a pick outside its row'
    return p


def padded(row_idx, vals, n, k):
  """[n, k] int64 of each row's values in their output order, -1 padded; plus the per-row counts."""
  row_idx = np.asarray(row_idx, dtype=np.int64)
  order = np.argsort(row_idx, kind='stable')
  row_idx, vals = row_idx[order], np.asarray(vals)[order]
  cnt = np.bincount(row_idx, minlength=n)
  assert cnt.max(initial=0) <= k
  start = np.zeros(n + 1, dtype=np.int64)
  np.cumsum(cnt, out=start[1:])
  out = np.full((n, k), -1, dtype=np.int64)
  out[row_idx, np.arange(row_idx.size) - start[row_idx]] = vals
  return out, cnt


def one_hop(plane, star, k, weighted=False, replace=False, stream=0, seed=SEED, rows=None, mode='CUDA'):
  """Positions [n, k] (draw order, -1 padded) and counts of one one-hop call on `star`'s rows."""
  rows = np.arange(star.n, dtype=np.int64) if rows is None else np.asarray(rows, dtype=np.int64)
  n = rows.size
  if plane == 'cpu':
    nat = glt.ops.require_native()
    t = star.topo()
    seeds = torch.from_numpy(rows)
    if weighted:
      nbr, cnt, _ = nat.cpu_sample_neighbors_weighted(t.indptr, t.indices, None, t.edge_weights, seeds, k, False,
                                                      seed, stream, replace)
    else:
      nbr, cnt, _ = nat.cpu_sample_neighbors(t.indptr, t.indices, None, seeds, k, False, replace, seed, stream)
    cnt = cnt.numpy()
    r = np.repeat(np.arange(n), cnt)
    pos, c2 = padded(r, star.positions(rows[r], nbr.numpy()), n, k)
    assert np.array_equal(c2, cnt)
    return pos, cnt
  h = star.handle_int64() if mode == 'int64' else star.handle(mode)
  nbr, cnt, _ = h.sample_one_hop(torch.from_numpy(rows).to(DEV), k, False, weighted, replace, seed, stream)
  nbr, cnt = nbr.cpu().numpy(), cnt.cpu().numpy().astype(np.int64)
  have = nbr >= 0
  assert np.array_equal(have.sum(1), cnt) and np.all(have == (np.arange(k)[None, :] < cnt[:, None]))
  pos = np.full_like(nbr, -1)
  rr = np.nonzero(have)
  pos[rr] = star.positions(rows[rr[0]], nbr[rr])
  return pos, cnt


def sorted_picks(pos):
  big = np.iinfo(np.int64).max
  s = np.sort(np.where(pos < 0, big, pos), axis=1)
  return np.where(s == big, -1, s)


def assert_no_duplicates(pos, label):
  s = sorted_picks(pos)
  dup = (s[:, 1:] == s[:, :-1]) & (s[:, 1:] >= 0)
  assert not dup.any(), f'{label}: {int(dup.any(1).sum())} rows hold a position twice'


# --------------------------------------------------------------------------- statistics
def chisq(obs, expected, label):
  """Chi-square of counts against expected counts; cells expecting < 5 are pooled."""
  obs = np.asarray(obs, dtype=np.float64).ravel()
  exp = np.asarray(expected, dtype=np.float64).ravel()
  assert abs(exp.sum() - obs.sum()) <= 1e-6 * obs.sum(), (label, exp.sum(), obs.sum())
  assert np.all(obs[exp == 0] == 0), f'{label}: an outcome of probability 0 was drawn'
  small = exp < 5
  o = list(obs[~small])
  e = list(exp[~small])
  if small.any():
    if exp[small].sum() >= 5 or not e:
      o.append(obs[small].sum()); e.append(exp[small].sum())
    else:
      j = int(np.argmin(e))
      o[j] += obs[small].sum(); e[j] += exp[small].sum()
  o, e = np.array(o), np.array(e)
  if o.size < 2:
    print(f'{label}: one cell, nothing to test')
    return
  e *= o.sum() / e.sum()
  stat, p = stats.chisquare(o, e)
  print(f'{label}: chi2 {stat:.1f} over {o.size} cells, p = {p:.3g}')
  assert p > P_MIN, f'{label}: p = {p:.3g}'


def binom_check(hits, n, q, label):
  p = stats.binomtest(int(hits), int(n), float(q)).pvalue
  print(f'{label}: {hits} of {n} against {q * n:.1f}, p = {p:.3g}')
  assert p > P_MIN, f'{label}: p = {p:.3g}'


def subset_codes(pos):
  """Bitmask of each row's picked positions (d <= 62)."""
  s = np.where(pos >= 0, np.left_shift(np.int64(1), np.maximum(pos, 0)), 0)
  return np.bitwise_or.reduce(s, axis=1)


def uniform_subset_probs(d, k):
  return {sum(1 << i for i in c): 1.0 / math.comb(d, k) for c in itertools.combinations(range(d), k)}


def weighted_subset_probs(w, k):
  """P(subset) of successive draws without replacement in proportion to w: sum over its orderings."""
  w = np.asarray(w, dtype=np.float64)
  W = w.sum()
  out = {}
  for t in itertools.permutations(range(w.size), k):
    p, rest = 1.0, W
    for i in t:
      p *= w[i] / rest
      rest -= w[i]
    code = sum(1 << i for i in t)
    out[code] = out.get(code, 0.0) + p
  return out


def check_subsets(pos, probs, label):
  codes = subset_codes(pos)
  keys = np.array(sorted(probs), dtype=np.int64)
  assert np.all(np.isin(codes, keys)), f'{label}: a subset of probability 0 (or of the wrong size) was drawn'
  obs = np.searchsorted(keys, codes)
  chisq(np.bincount(obs, minlength=keys.size), np.array([probs[c] for c in keys]) * codes.size, label)


def weighted_exclusion_probs(w):
  """d = k + 1, weighted without replacement: P(position j is the one left out) = P(j's exponential key is the
  largest) = int w_j e^{-w_j t} prod_{i != j} (1 - e^{-w_i t}) dt, integrated per distinct weight."""
  w = np.asarray(w, dtype=np.float64)
  vals, inv, cnt = np.unique(w, return_inverse=True, return_counts=True)
  p_val = np.empty(vals.size)
  for a, wa in enumerate(vals):
    c = cnt.copy()
    c[a] -= 1

    def f(t, wa=wa, c=c):
      return wa * math.exp(-wa * t) * float(np.prod((-np.expm1(-vals * t)) ** c))
    # split the range at the scales of the smallest and largest weights
    pts = sorted({0.0, 1.0 / vals.max(), 1.0 / vals.min(), 10.0 / vals.min(), 60.0 / vals.min()})
    p_val[a] = sum(integrate.quad(f, lo, hi, limit=200, epsabs=1e-13, epsrel=1e-10)[0]
                   for lo, hi in zip(pts[:-1], pts[1:]))
  p = p_val[inv]
  assert abs(p.sum() - 1.0) < 1e-7, p.sum()
  return p


def weighted_inclusion(w, k):
  """Inclusion probability of every position in a weighted k-sample without replacement (exponential race):
  P(key_j among the k smallest) = int w_j e^{-w_j t} P(at most k - 1 other keys below t) dt.  Positions of equal
  weight are exchangeable, so the count of other keys below t is a sum of one binomial per distinct weight."""
  w = np.asarray(w, dtype=np.float64)
  vals, inv, cnt = np.unique(w, return_inverse=True, return_counts=True)
  pts = [0.0] + list(np.geomspace(1e-4 / vals.max(), 60.0 / vals.min(), 16))
  p_val = np.empty(vals.size)
  for a, wa in enumerate(vals):
    c = cnt.copy()
    c[a] -= 1

    def f(t, wa=wa, c=c):
      pmf = np.ones(1)
      for wv, n in zip(vals, c):
        if n:
          pmf = np.convolve(pmf, stats.binom.pmf(np.arange(min(n, k - 1) + 1), n, -math.expm1(-wv * t)))[:k]
      return wa * math.exp(-wa * t) * pmf.sum()
    p_val[a] = sum(integrate.quad(f, lo, hi, limit=100, epsabs=1e-13, epsrel=1e-10)[0]
                   for lo, hi in zip(pts[:-1], pts[1:]))
  p = p_val[inv]
  assert abs(p.sum() - k) < 1e-6 * k, (p.sum(), k)
  return p


def check_inclusion(pos, d, pi, label, bins=64):
  """Picks per position (grouped into contiguous bins when few) against the inclusion probabilities `pi`."""
  n = pos.shape[0]
  hits = np.bincount(pos[pos >= 0], minlength=d).astype(np.float64)
  exp = np.broadcast_to(np.asarray(pi, dtype=np.float64), (d,)) * n
  if exp.min() < 20 and d > bins:
    edges = np.linspace(0, d, bins + 1).astype(np.int64)
    hits = np.add.reduceat(hits, edges[:-1])
    exp = np.add.reduceat(exp, edges[:-1])
  chisq(hits, exp, label)


def check_pairs(pos, d, k, label):
  """Co-inclusion of fixed position pairs against k(k-1)/(d(d-1)) (uniform without replacement)."""
  n = pos.shape[0]
  q = k * (k - 1) / (d * (d - 1))
  for a, b in [(0, 1), (0, d - 1), (d // 2 - 1, d // 2), (1, d - 2), (k - 1, k)]:
    both = ((pos == a).any(1) & (pos == b).any(1)).sum()
    binom_check(both, n, q, f'{label} pair ({a},{b})')


# --------------------------------------------------------------------------- graphs shared by the cases
def rows_for(d, cells):
  """Enough rows for about 64 expected draws per cell, between 2^14 and 2^17 (and at most 2^24 edges)."""
  n = 1 << 14
  while n < (1 << 17) and n < 64 * cells and 2 * n * d <= (1 << 24):
    n *= 2
  return n


_STARS = {}


def star(n, d, weights=None):
  key = (n, d, None if weights is None else tuple(np.asarray(weights).tolist()))
  if key not in _STARS:
    _STARS[key] = Star(np.full(n, d), weights=weights)
  return _STARS[key]


HUB_D, HUB_ROWS = 4096, 1 << 12


# --------------------------------------------------------------------------- uniform without replacement
@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', KS)
def test_uniform_floyd_boundary(plane, k):
  """d = k + 1: exactly one position is left out, uniformly."""
  d = k + 1
  s = star(rows_for(d, d), d)
  pos, cnt = one_hop(plane, s, k, stream=3)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'k={k} d={d}')
  left_out = d * (d - 1) // 2 - pos.sum(1)
  chisq(np.bincount(left_out, minlength=d), np.full(d, s.n / d), f'{plane} uniform k={k} d={d} left-out position')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('d,k', [(6, 3), (5, 4), (9, 8), (40, 2), (7, 1), (12, 5)])
def test_uniform_subsets(plane, d, k):
  s = star(1 << 17, d)
  pos, cnt = one_hop(plane, s, k, stream=4)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'd={d} k={k}')
  if math.comb(d, k) <= 5000:
    check_subsets(pos, uniform_subset_probs(d, k), f'{plane} uniform d={d} k={k} subsets')
  else:
    check_inclusion(pos, d, k / d, f'{plane} uniform d={d} k={k} inclusion')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', [3, 16, 32, 128, 512])
def test_uniform_hub(plane, k):
  """One hub per bucket: d = 4096 over 4096 rows."""
  s = star(HUB_ROWS, HUB_D)
  pos, cnt = one_hop(plane, s, k, stream=5)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'hub k={k}')
  check_inclusion(pos, HUB_D, k / HUB_D, f'{plane} uniform hub k={k} inclusion')
  check_pairs(pos, HUB_D, k, f'{plane} uniform hub k={k}')


@pytest.mark.parametrize('plane', PLANES)
def test_uniform_widest_row(plane):
  """256 rows of degree 100,000 at k = 512 (2.56e7 edges)."""
  d, k = 100_000, 512
  s = star(256, d)
  pos, cnt = one_hop(plane, s, k, stream=6)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, 'd=1e5 k=512')
  check_inclusion(pos, d, k / d, f'{plane} uniform d=1e5 k=512 inclusion')
  check_pairs(pos, d, k, f'{plane} uniform d=1e5 k=512')


# --------------------------------------------------------------------------- weighted without replacement
@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('d,k,w', [(6, 3, [1, 1, 2, 4, 0.5, 8]), (7, 5, W7), (5, 2, [1e-3, 1, 1e3, 1, 30]),
                                   (9, 4, [1, 2, 3, 4, 5, 6, 7, 8, 9])])
def test_weighted_subsets(plane, d, k, w):
  w = np.asarray(w, dtype=np.float32)
  s = star(1 << 17, d, w)
  pos, cnt = one_hop(plane, s, k, weighted=True, stream=7)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'weighted d={d} k={k}')
  check_subsets(pos, weighted_subset_probs(w.astype(np.float64), k), f'{plane} weighted d={d} k={k} subsets')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', KS)
def test_weighted_floyd_boundary(plane, k):
  """d = k + 1 with weights over a 1e3 ratio: which position is left out, against the exponential race's law."""
  d = k + 1
  s = star(rows_for(d, d), d, W7)
  pos, cnt = one_hop(plane, s, k, weighted=True, stream=8)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'weighted k={k}')
  left_out = d * (d - 1) // 2 - pos.sum(1)
  p = weighted_exclusion_probs(W7[np.arange(d) % W7.size].astype(np.float64))
  chisq(np.bincount(left_out, minlength=d), p * s.n, f'{plane} weighted k={k} d={d} left-out position')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', [8, 16, 32, 128, 512])
def test_weighted_hub(plane, k):
  """d = 4096 in blocks of 64 positions alternating weight 1 and 4: inclusion per block against the exact law."""
  w = np.repeat(np.array([1.0, 4.0], dtype=np.float32), 64)
  s = star(HUB_ROWS, HUB_D, w)
  pos, cnt = one_hop(plane, s, k, weighted=True, stream=9)
  assert np.all(cnt == k)
  assert_no_duplicates(pos, f'weighted hub k={k}')
  pi = weighted_inclusion(s.weights[:HUB_D], k)
  check_inclusion(pos, HUB_D, pi, f'{plane} weighted hub k={k} inclusion', bins=64)


@pytest.mark.parametrize('plane', PLANES)
def test_weighted_zero_weights(plane):
  """Zero-weight neighbours are never picked while positive ones remain, and fill the rest in position order."""
  w = np.array([0, 3, 0, 1, 0, 2, 0, 0], dtype=np.float32)   # 3 positive weights
  s = star(1 << 15, 8, w)
  pos, cnt = one_hop(plane, s, 2, weighted=True, stream=10)
  assert np.all(cnt == 2) and np.all(w[pos] > 0)
  check_subsets(pos, weighted_subset_probs(w.astype(np.float64), 2),
                f'{plane} weighted zero-weights k=2 subsets')
  pos, cnt = one_hop(plane, s, 5, weighted=True, stream=11)
  assert np.all(cnt == 5)
  assert np.array_equal(sorted_picks(pos), np.tile([0, 1, 2, 3, 5], (s.n, 1)))   # all positives, then 0 and 2
  pos, cnt = one_hop(plane, s, 7, weighted=True, stream=12)
  # keys order the picks: the positive weights first, then the zero weights in position order
  assert np.all(np.sort(pos[:, :3], axis=1) == [1, 3, 5]) and np.all(pos[:, 3:] == [0, 2, 4, 6])


# --------------------------------------------------------------------------- with replacement
def check_draws(pos, d, probs, label, w=None):
  """k independent draws of law `probs`: the marginal of every draw and the joints of draws (0, 1), (0, k-1)."""
  n, k = pos.shape
  assert np.all(pos >= 0)
  bins = min(d, 16)
  edges = np.linspace(0, d, bins + 1).astype(np.int64)
  pb = np.add.reduceat(probs, edges[:-1])
  binned = np.searchsorted(edges, pos, side='right') - 1
  if d <= 64:
    chisq(np.bincount(pos.ravel(), minlength=d), probs * pos.size, f'{label} marginal')
  else:
    check_inclusion(pos, d, probs * k, f'{label} marginal')
  if w is not None:
    # per distinct weight: a CDF whose running sum rounds coarser than the small weights skews exactly these
    vals, inv = np.unique(w[:d], return_inverse=True)
    chisq(np.bincount(inv[pos.ravel()], minlength=vals.size), np.bincount(inv, weights=probs) * pos.size,
          f'{label} per weight')
  for j in sorted({j for j in (1, k - 1) if 0 < j < k}):
    cells = binned[:, 0] * bins + binned[:, j]
    chisq(np.bincount(cells, minlength=bins * bins), np.outer(pb, pb).ravel() * n, f'{label} joint of draws 0, {j}')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k,d', [(1, 5), (3, 5), (8, 11), (16, 17), (17, 40), (33, 60), (129, 300), (512, 4096),
                                 (512, 100_000)])
@pytest.mark.parametrize('weighted', [False, True])
def test_with_replacement(plane, k, d, weighted):
  w = W7 if weighted else None
  s = star(rows_for(d, 256) if d < 4096 else HUB_ROWS if d == 4096 else 256, d, w)
  pos, cnt = one_hop(plane, s, k, weighted=weighted, replace=True, stream=13)
  assert np.all(cnt == k)
  probs = np.full(d, 1.0 / d) if not weighted else s.weights[:d].astype(np.float64) / s.weights[:d].sum(dtype=np.float64)
  check_draws(pos, d, probs, f'{plane} {"weighted" if weighted else "uniform"} replace k={k} d={d}',
              s.weights if weighted else None)


@pytest.mark.parametrize('plane', PLANES)
def test_weighted_replace_wide_row_small_weights(plane):
  """1e5 weights alternating 1 and 1000: the row sums to 5e7, where one fp32 ulp (4) exceeds the small weights.
  Their share of the draws must still be 1/1001: the CDF has to be summed finer than fp32."""
  d, k = 100_000, 512
  s = star(256, d, np.array([1.0, 1000.0], dtype=np.float32))
  small = 0
  for stream in range(120, 128):
    pos, cnt = one_hop(plane, s, k, weighted=True, replace=True, stream=stream)
    assert np.all(cnt == k)
    small += int((pos % 2 == 0).sum())
  total = 8 * s.n * k
  chisq([small, total - small], np.array([1.0, 1000.0]) / 1001.0 * total, f'{plane} weighted replace d=1e5 small weights')


@pytest.mark.parametrize('plane', PLANES)
def test_weighted_replace_edges(plane):
  """Rows of degree <= k are copied; a row whose weights are all 0 picks nothing; zero weights are never drawn."""
  w = np.array([0, 2, 0, 0, 1, 0], dtype=np.float32)
  deg = np.tile([6, 4, 3, 6, 0], 2000)
  s = Star(deg, weights=w)
  zero = Star(np.full(64, 6), weights=np.zeros(6, dtype=np.float32))
  pos, cnt = one_hop(plane, s, 4, weighted=True, replace=True, stream=14)
  assert np.array_equal(cnt, np.minimum(deg, 4))
  small = (deg <= 4)
  assert np.all(pos[small & (deg > 0)][:, :3] == [0, 1, 2])
  big = pos[deg > 4]
  assert np.all((big == 1) | (big == 4))
  chisq(np.bincount(big.ravel() == 4, minlength=2), np.array([2 / 3, 1 / 3]) * big.size,
        f'{plane} weighted replace with zero weights')
  pos, cnt = one_hop(plane, zero, 4, weighted=True, replace=True, stream=14)
  assert np.all(cnt == 0) and np.all(pos == -1)


# --------------------------------------------------------------------------- mixed warps
@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', [3, 12, 40])
@pytest.mark.parametrize('weighted', [False, True])
def test_mixed_warp_rows(plane, k, weighted):
  """Rows of degree 0, d <= k (copied) and d > k interleaved in one launch (4 / 2 / 1 rows per warp at
  k = 3 / 12 / 40): the copies are exact, and the sampled rows draw exactly what a launch of them alone draws,
  with the exact law."""
  d_big = k + 3
  pattern = np.array([d_big, 0, max(k - 1, 1), d_big, k, d_big, 1, d_big])
  deg = np.tile(pattern, 1 << 14)
  s = Star(deg, weights=W7 if weighted else None)
  pos, cnt = one_hop(plane, s, k, weighted=weighted, stream=15)
  assert np.array_equal(cnt, np.minimum(deg, k))
  for dd in np.unique(deg[deg <= k]):
    rows = pos[deg == dd]
    assert np.all(rows[:, :dd] == np.arange(dd)) and np.all(rows[:, dd:] == -1), f'copied row of degree {dd}'
  big_rows = np.nonzero(deg == d_big)[0]
  alone, _ = one_hop(plane, s, k, weighted=weighted, stream=15, rows=big_rows)
  assert np.array_equal(pos[big_rows], alone), 'sampled rows depend on the rows sharing their warp'
  big = pos[big_rows]
  assert_no_duplicates(big, 'mixed')
  pi = weighted_inclusion(W7[np.arange(d_big) % W7.size], k) if weighted else np.full(d_big, k / d_big)
  check_inclusion(big, d_big, pi, f'{plane} {"weighted" if weighted else "uniform"} mixed warp k={k} inclusion')


# --------------------------------------------------------------------------- device arenas
def arena_hop_picks(star, node, rows, cols, ne, hop, k):
  """Positions [n_targets, k] (ELL order) of hop `hop` of an arena's COO, and the targets' global ids."""
  e0 = sum(ne[:hop])
  sl = slice(e0, e0 + ne[hop])
  tgt = node[cols[sl]]
  nbr = node[rows[sl]]
  targets, t_idx = np.unique(tgt, return_inverse=True)
  pos, _ = padded(t_idx, star.positions(targets[t_idx], nbr), targets.size, k)
  return targets, pos


def coo_np(out):
  return [x.cpu().numpy() if torch.is_tensor(x) else x for x in out]


@pytest.mark.gpu
@pytest.mark.parametrize('k,weighted', [(3, False), (16, True), (33, False), (129, True), (512, False)])
def test_sampler_arena_one_hop(k, weighted):
  """SamplerArena.sample reads back through to_coo: d = k + 1, the left-out position against its exact law."""
  d = k + 1
  s = star(min(rows_for(d, d), 1 << 15), d, W7 if weighted else None)
  nat = glt.ops.require_native()
  arena = nat.SamplerArena(0, s.n, [k], False, int(s.indices.max()) + 1)
  arena.sample(s.handle(), torch.arange(s.n, device=DEV), None, SEED, 40, weighted, False, False)
  node, rows, cols, _, nn, ne = coo_np(arena.to_coo())
  targets, pos = arena_hop_picks(s, node, rows, cols, ne, 0, k)
  assert np.array_equal(targets, np.arange(s.n)) and ne[0] == s.n * k
  assert_no_duplicates(pos, f'arena k={k}')
  left_out = d * (d - 1) // 2 - pos.sum(1)
  p = weighted_exclusion_probs(W7[np.arange(d) % W7.size].astype(np.float64)) if weighted else np.full(d, 1 / d)
  chisq(np.bincount(left_out, minlength=d), p * s.n, f'arena {"weighted" if weighted else "uniform"} k={k} left-out')
  # the arena draws what the one-hop kernel draws for the same (seed, stream)
  ref, _ = one_hop('gpu', s, k, weighted=weighted, stream=40)
  assert np.array_equal(sorted_picks(pos), sorted_picks(ref))


def two_level(n, d0, d1):
  """Seeds 0..n-1 with d0 children each (ids n + ...); every child has a row of d1 leaves (ids past all rows)."""
  n_mid = n * d0
  deg = np.concatenate([np.full(n, d0), np.full(n_mid, d1)])
  base = np.concatenate([n + np.arange(n) * d0, n + n_mid + np.arange(n_mid) * d1])
  return Star(deg, base=base)


@pytest.mark.gpu
@pytest.mark.parametrize('replace', [False, True])
def test_sampler_arena_two_hops_independent(replace):
  """Hop 1 rows draw independently of hop 0: the joint of a seed's subset and its first child's subset is the
  product of two uniform laws."""
  n, d0, k0, d1, k1 = 1 << 15, 4, 2, 5, 2
  s = two_level(n, d0, d1)
  nat = glt.ops.require_native()
  arena = nat.SamplerArena(0, n, [k0, k1], False, int(s.indices.max()) + 1)
  arena.sample(s.handle(), torch.arange(n, device=DEV), None, SEED, 48, False, replace, False)
  node, rows, cols, _, nn, ne = coo_np(arena.to_coo())
  t0, p0 = arena_hop_picks(s, node, rows, cols, ne, 0, k0)
  t1, p1 = arena_hop_picks(s, node, rows, cols, ne, 1, k1)
  assert np.array_equal(t0, np.arange(n))
  first_child = n + np.arange(n) * d0 + p0[:, 0]
  i1 = np.searchsorted(t1, first_child)
  assert np.array_equal(t1[i1], first_child)
  label = f'arena 2-hop replace={replace}'
  if replace:
    a = p0[:, 0] * d0 + p0[:, 1]
    b = p1[i1, 0] * d1 + p1[i1, 1]
    pa, pb = np.full(d0 * d0, 1 / d0 ** 2), np.full(d1 * d1, 1 / d1 ** 2)
  else:
    ka = np.array(sorted(uniform_subset_probs(d0, k0)))
    kb = np.array(sorted(uniform_subset_probs(d1, k1)))
    a = np.searchsorted(ka, subset_codes(p0))
    b = np.searchsorted(kb, subset_codes(p1[i1]))
    pa, pb = np.full(ka.size, 1 / ka.size), np.full(kb.size, 1 / kb.size)
  chisq(np.bincount(a * pb.size + b, minlength=pa.size * pb.size), np.outer(pa, pb).ravel() * n,
        f'{label} joint of hop 0 and hop 1')


@pytest.mark.gpu
def test_sampler_arena_device_steps_independent():
  """Consecutive device steps (use_dev_step, step_inc = 1, as under CUDA-graph replay): the joint of a row's subsets
  in two steps is the product, and the step advances the stream by 8 per step."""
  d, k = 5, 2
  s = star(1 << 16, d)
  nat = glt.ops.require_native()
  arena = nat.SamplerArena(0, s.n, [k], False, int(s.indices.max()) + 1)
  keys = np.array(sorted(uniform_subset_probs(d, k)))
  codes = []
  for step in range(2):
    arena.sample(s.handle(), torch.arange(s.n, device=DEV), None, SEED, 56, False, False, True, 1)
    node, rows, cols, _, nn, ne = coo_np(arena.to_coo())
    _, pos = arena_hop_picks(s, node, rows, cols, ne, 0, k)
    assert int(arena.step.item()) == step + 1
    ref, _ = one_hop('gpu', s, k, stream=56 + 8 * (step + 1))
    assert np.array_equal(sorted_picks(pos), sorted_picks(ref))
    codes.append(np.searchsorted(keys, subset_codes(pos)))
  m = keys.size
  chisq(np.bincount(codes[0] * m + codes[1], minlength=m * m), np.full(m * m, s.n / m ** 2),
        'arena consecutive device steps joint')


@pytest.mark.gpu
@pytest.mark.parametrize('weighted', [False, True])
def test_hetero_arena_two_relations(weighted):
  """Two relations out of one node type with k = 3 (d = 5) and k = 40 (d = 41): the grouped kernel runs both under
  the 32-lane, 4-picks template chosen from max k.  Each relation's law, and the joint of both relations' picks on
  the same row against the product."""
  n = 1 << 16
  w5 = np.array([1, 2, 0.25, 4, 1], dtype=np.float32)
  r0 = Star(np.full(n, 5), base=np.arange(n) * 5, weights=w5 if weighted else None)
  r1 = Star(np.full(n, 41), base=n * 5 + np.arange(n) * 41, weights=W7 if weighted else None)
  n_nbr = n * 5 + n * 41
  nat = glt.ops.require_native()
  arena = nat.HeteroArena(0, 2, [r0.handle(), r1.handle()], [0, 0], [1, 1], [[3], [40]], [n, n_nbr], [n, 0],
                          False, SEED, weighted, False, 0, [])
  arena.step.fill_(64)
  arena.sample([0], [torch.arange(n, device=DEV)], 0)
  nodes, rows, cols, _, nn, ne = arena.to_coo()
  seeds = nodes[0].cpu().numpy()
  assert np.array_equal(seeds, np.arange(n))
  picks = []
  for r, (st, k) in enumerate([(r0, 3), (r1, 40)]):
    nbr = nodes[1].cpu().numpy()[rows[r].cpu().numpy()]
    tgt = seeds[cols[r].cpu().numpy()]
    assert ne[r] == [n * k]
    pos, _ = padded(tgt, st.positions(tgt, nbr), n, k)
    assert_no_duplicates(pos, f'hetero relation {r}')
    picks.append(pos)
  kind = 'weighted' if weighted else 'uniform'
  p0 = weighted_subset_probs(w5.astype(np.float64), 3) if weighted else uniform_subset_probs(5, 3)
  check_subsets(picks[0], p0, f'hetero {kind} relation 0 (k=3) subsets')
  left_out = 41 * 40 // 2 - picks[1].sum(1)
  p1 = weighted_exclusion_probs(W7[np.arange(41) % 7].astype(np.float64)) if weighted else np.full(41, 1 / 41)
  chisq(np.bincount(left_out, minlength=41), p1 * n, f'hetero {kind} relation 1 (k=40) left-out position')
  keys = np.array(sorted(p0))
  a = np.searchsorted(keys, subset_codes(picks[0]))
  pa = np.array([p0[c] for c in keys])
  chisq(np.bincount(a * 41 + left_out, minlength=keys.size * 41), np.outer(pa, p1).ravel() * n,
        f'hetero {kind} joint of the two relations')


# --------------------------------------------------------------------------- keying and memory tiers
@pytest.mark.parametrize('plane', PLANES)
def test_consecutive_streams_independent(plane):
  d, k = 5, 2
  s = star(1 << 16, d)
  keys = np.array(sorted(uniform_subset_probs(d, k)))
  a = np.searchsorted(keys, subset_codes(one_hop(plane, s, k, stream=70)[0]))
  b = np.searchsorted(keys, subset_codes(one_hop(plane, s, k, stream=71)[0]))
  m = keys.size
  chisq(np.bincount(a * m + b, minlength=m * m), np.full(m * m, s.n / m ** 2), f'{plane} streams 70, 71 joint')
  again = np.searchsorted(keys, subset_codes(one_hop(plane, s, k, stream=70)[0]))
  assert np.array_equal(a, again)


@pytest.mark.gpu
@pytest.mark.parametrize('weighted', [False, True])
def test_memory_tiers_draw_the_same(weighted):
  """ZERO_COPY (pinned host, int64 ids), CUDA with int32 ids and CUDA with int64 ids pick the same positions."""
  s = Star(np.tile([50, 3, 200, 0, 17], 4000), weights=W7 if weighted else None)
  for k in (8, 40, 512):
    ref, cnt = one_hop('gpu', s, k, weighted=weighted, stream=80)
    for mode in ('ZERO_COPY', 'int64'):
      got, c2 = one_hop('gpu', s, k, weighted=weighted, stream=80, mode=mode)
      assert np.array_equal(cnt, c2) and np.array_equal(got, ref), (mode, k)


@pytest.mark.gpu
@pytest.mark.parametrize('k,d', [(3, 7), (16, 40), (129, 300), (512, 4096)])
def test_weighted_gpu_matches_cpu(k, d):
  """Same seed, same stream: the planes' weighted picks.  Without replacement they rank keys computed with device
  and host logf, and pick the same subsets (measured on an H100: no row differs at these shapes).  With replacement
  they sum the fp64 CDF in different orders, so a draw landing on a boundary may differ: all but a tiny fraction of
  rows must agree."""
  s = star(HUB_ROWS if d >= 4096 else 1 << 15, d, W7)
  for replace in (False, True):
    g, _ = one_hop('gpu', s, k, weighted=True, replace=replace, stream=90)
    c, _ = one_hop('cpu', s, k, weighted=True, replace=replace, stream=90)
    if not replace:
      g, c = sorted_picks(g), sorted_picks(c)
    differ = int((g != c).any(1).sum())
    print(f'weighted replace={replace} k={k} d={d}: {differ} of {s.n} rows differ between GPU and CPU')
    assert differ <= (max(2, s.n // 10000) if replace else 0)


@pytest.mark.parametrize('plane', PLANES)
def test_neighbor_sampler_weighted_with_replacement(plane):
  """NeighborSampler(with_weight=True, replace=True) draws k independent neighbours in proportion to the weights,
  on CPU and CUDA graphs alike."""
  d, k = 7, 5
  s = star(1 << 15, d, W7)
  g = s.graph('CPU' if plane == 'cpu' else 'CUDA')
  ns = NeighborSampler(g, [k], with_weight=True, replace=True, seed=SEED,
                       device=DEV if plane == 'gpu' else None)
  seeds = torch.arange(s.n, device=DEV if plane == 'gpu' else 'cpu')
  out = ns.sample_one_hop(seeds, k, stream=100)
  cnt = out.nbr_num.cpu().numpy()
  assert np.all(cnt == k)
  nbr = out.nbr.cpu().numpy().reshape(s.n, k)
  pos = nbr - s.base[:, None]
  probs = W7.astype(np.float64) / W7.sum(dtype=np.float64)
  check_draws(pos, d, probs, f'{plane} NeighborSampler weighted replace', s.weights)
  if plane == 'gpu':
    ref = NeighborSampler(s.graph('CPU'), [k], with_weight=True, replace=True, seed=SEED)
    c = ref.sample_one_hop(seeds.cpu(), k, stream=100).nbr.numpy().reshape(s.n, k)
    differ = int((c != nbr).any(1).sum())
    print(f'NeighborSampler weighted replace: {differ} of {s.n} rows differ between GPU and CPU')
    assert differ <= max(2, s.n // 10000)


# --------------------------------------------------------------------------- negatives
@pytest.mark.parametrize('plane', PLANES)
def test_strict_negatives_uniform_over_non_edges(plane):
  n = 30
  rng = np.random.default_rng(7)
  cells = rng.choice(n * n, size=300, replace=False)
  adj = np.zeros(n * n, dtype=bool)
  adj[cells] = True
  ei = torch.from_numpy(np.stack(np.divmod(np.sort(cells), n)))
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=n)
  req = 1 << 18
  if plane == 'cpu':
    rows, cols = glt.ops.require_native().cpu_negative_sample(topo.indptr, topo.indices, n, n, req, 20, False, True,
                                                            SEED, 110)
  else:
    h = glt.data.Graph(topo, 'CUDA', 0).graph_handler
    rows, cols, count = h.negative_sample(n, n, req, 20, False, SEED, 110)
    c = int(count.item())
    rows, cols = rows[:c], cols[:c]
  pair = rows.cpu().numpy() * n + cols.cpu().numpy()
  assert pair.size > req * 0.999
  assert not adj[pair].any(), 'an edge was returned as a negative'
  obs = np.bincount(pair, minlength=n * n)[~adj]
  chisq(obs, np.full(obs.size, pair.size / obs.size), f'{plane} strict negatives over {obs.size} non-edges')
