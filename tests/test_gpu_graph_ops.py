"""The public graph operations against exact references: random walks (uniform and node2vec p / q), induced
subgraphs, full neighbourhoods and degrees, hotness propagation and padded negative sampling.

The CPU/GPU equality tests prove that both planes run the same algorithm; these prove that the algorithm computes
what it claims.  Where the CPU plane implements the same operation a test runs on both planes (PLANES), so its CPU
half also runs without a GPU.

Statistical checks follow test_gpu_sampler_distributions.py: fixed seeds (Philox makes every outcome
deterministic, so a correct kernel cannot flake), a printed p-value and `assert p > 1e-6`.  Deterministic checks are
exact; hotness entries are bounded by their float32 rounding.
"""
import math

import numpy as np
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.sampler import NeighborSampler, NodeSamplerInput
from test_gpu_sampler_distributions import DEV, PLANES, SEED, binom_check, chisq

U32 = np.uint64(0xFFFFFFFF)


def nat():
  return glt.ops.require_native()


# --------------------------------------------------------------------------- graphs
def csr_graph(indptr, indices, eids=None):
  indptr = torch.as_tensor(np.asarray(indptr, dtype=np.int64))
  indices = torch.as_tensor(np.asarray(indices, dtype=np.int64))
  eids = None if eids is None else torch.as_tensor(np.asarray(eids, dtype=np.int64))
  return glt.data.Topology((indptr, indices), edge_ids=eids, input_layout='CSR', layout='CSR')


def from_rows(rows):
  """CSR (indptr, indices) of a list of per-row column lists (each row sorted here)."""
  deg = np.array([len(r) for r in rows], dtype=np.int64)
  indptr = np.zeros(deg.size + 1, dtype=np.int64)
  np.cumsum(deg, out=indptr[1:])
  indices = np.concatenate([np.sort(np.asarray(r, dtype=np.int64)) for r in rows]) if indptr[-1] else \
      np.zeros(0, dtype=np.int64)
  return indptr, indices


def two_shards(topo, split, eids=True):
  """A two-shard device table (int64 column ids) holding `topo`'s rows [0, split) and [split, n)."""
  ip, ind, ei = topo.indptr, topo.indices, topo.edge_ids
  n = ip.numel() - 1
  shards = []
  for b, e in ((0, split), (split, n)):
    lo, hi = int(ip[b]), int(ip[e])
    s = {'indptr': (ip[b:e + 1] - lo).to(DEV), 'indices': ind[lo:hi].to(DEV), 'row_begin': b, 'row_end': e}
    if eids:
      s['eids'] = ei[lo:hi].to(DEV)
    shards.append(s)
  return glt.data.Graph.from_shards(shards, 0)


def int64_graph(topo):
  """A one-shard device table that keeps int64 column ids ('CUDA' mode narrows them to int32)."""
  n = topo.indptr.numel() - 1
  return glt.data.Graph.from_shards([{'indptr': topo.indptr.to(DEV), 'indices': topo.indices.to(DEV),
                                      'eids': topo.edge_ids.to(DEV), 'row_begin': 0, 'row_end': n}], 0)


TIERS = ['CUDA', 'ZERO_COPY', 'int64', 'shards']


def tier_graph(topo, tier):
  if tier in ('CUDA', 'ZERO_COPY'):
    return glt.data.Graph(topo, tier, 0)
  if tier == 'int64':
    return int64_graph(topo)
  return two_shards(topo, (topo.indptr.numel() - 1) // 2)


# --------------------------------------------------------------------------- Philox (csrc/philox.h) in numpy
def philox_draw(seed, stream, row, i):
  """philox_draw(seed, stream, row, i) of csrc/philox.h, vectorised over `row` and `i`."""
  row = np.asarray(row, dtype=np.uint64)
  i = np.broadcast_to(np.asarray(i, dtype=np.uint64), row.shape)
  x, y = row & U32, row >> np.uint64(32)
  z, w = i >> np.uint64(2), np.full_like(row, np.uint64(stream) & U32)
  k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
  for _ in range(10):
    p0, p1 = np.uint64(0xD2511F53) * x, np.uint64(0xCD9E8D57) * z
    x, y, z, w = (p1 >> np.uint64(32)) ^ y ^ k0, p1 & U32, (p0 >> np.uint64(32)) ^ w ^ k1, p0 & U32
    k0, k1 = (k0 + np.uint64(0x9E3779B9)) & U32, (k1 + np.uint64(0xBB67AE85)) & U32
  return np.choose((i & np.uint64(3)).astype(np.int64), [x, y, z, w])


def bounded(r, n):
  return ((np.asarray(r, dtype=np.uint64) * np.asarray(n, dtype=np.uint64)) >> np.uint64(32)).astype(np.int64)


# --------------------------------------------------------------------------- random walks
def walk(plane, topo_or_graph, starts, length, p=1.0, q=1.0, stream=0, seed=SEED):
  starts = torch.as_tensor(np.asarray(starts, dtype=np.int64))
  if plane == 'cpu':
    t = topo_or_graph
    return nat().cpu_random_walk(t.indptr, t.indices, starts, length, p, q, seed, stream).numpy()
  g = topo_or_graph if isinstance(topo_or_graph, glt.data.Graph) else glt.data.Graph(topo_or_graph, 'CUDA', 0)
  return g.graph_handler.random_walk(starts.to(DEV), length, p, q, seed, stream).cpu().numpy()


CIRC_N = 1 << 16
CIRC_OFFS = np.array([1, 2, 2, 3, 7, 7, 7, 40], dtype=np.int64)   # repeated columns: 2 twice, 7 three times


def circulant():
  """Row v holds (v + o) mod N for o in CIRC_OFFS, plus node N with no out-edges."""
  n = CIRC_N
  v = np.arange(n, dtype=np.int64)
  indptr = np.zeros(n + 2, dtype=np.int64)
  indptr[1:n + 1] = np.arange(1, n + 1) * CIRC_OFFS.size
  indptr[n + 1] = indptr[n]
  cols = np.sort((v[:, None] + CIRC_OFFS[None, :]) % n, axis=1).ravel()
  return csr_graph(indptr, cols)


@pytest.mark.parametrize('plane', PLANES)
def test_uniform_walk_steps(plane):
  """Every step is uniform over the row's positions (a repeated column counts once per position), and consecutive
  steps are independent."""
  topo = circulant()
  L = 4
  w = walk(plane, topo, np.arange(CIRC_N), L, stream=11)
  assert w.shape == (CIRC_N, L + 1) and np.array_equal(w[:, 0], np.arange(CIRC_N))
  inc = (w[:, 1:] - w[:, :-1]) % CIRC_N
  vals, mult = np.unique(CIRC_OFFS, return_counts=True)
  assert np.all(np.isin(inc, vals)), 'a step left its row'
  code = np.searchsorted(vals, inc)
  probs = mult / CIRC_OFFS.size
  for s in range(L):
    chisq(np.bincount(code[:, s], minlength=vals.size), probs * CIRC_N, f'{plane} uniform walk step {s + 1}')
  m = vals.size
  chisq(np.bincount(code[:, 0] * m + code[:, 1], minlength=m * m), np.outer(probs, probs).ravel() * CIRC_N,
        f'{plane} uniform walk steps 1, 2 joint')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('pq', [(1.0, 1.0), (0.25, 4.0), (0.3, 1.7)])
def test_walk_edges(plane, pq):
  """A node with no out-edges keeps the walker in place, start ids outside every row stay where they are, and
  walk_length = 0 returns the start column."""
  topo = circulant()
  p, q = pq
  dead, outside = CIRC_N, [CIRC_N + 1, CIRC_N + 1000, 1 << 40, -3]
  starts = np.array([dead] + outside + [5, 9], dtype=np.int64)
  w = walk(plane, topo, starts, 6, p, q, stream=12)
  for i, s in enumerate(starts[:-2]):
    assert np.all(w[i] == s), (s, w[i])
  assert np.all(w[-2:, 1:] != w[-2:, :-1])
  z = walk(plane, topo, starts, 0, p, q, stream=12)
  assert z.shape == (starts.size, 1) and np.array_equal(z[:, 0], starts)
  e = walk(plane, topo, np.zeros(0), 5, p, q, stream=12)
  assert e.shape == (0, 6)


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('pq', [(1.0, 1.0), None])
def test_uniform_walk_replays_philox(plane, pq):
  """Uniform walks (p = q = 1 included) take one Philox draw per step that leaves a row, keyed (seed, stream,
  walker, step): the walk is exactly that replay.  Rows of mixed degree, dead ends and ids outside the graph."""
  rng = np.random.default_rng(5)
  n = 3000
  deg = rng.integers(0, 40, n)
  deg[::97] = 0
  deg[5] = 3000
  rows = [rng.integers(0, n + 50, d) for d in deg]      # columns n .. n + 49 have no row: dead ends
  indptr, indices = from_rows(rows)
  topo = csr_graph(indptr, indices)
  starts = np.concatenate([np.arange(n), [n + 7, -1, 5, 5]])
  L, stream = 7, 13
  p, q = pq if pq else (1.0, 1.0)
  got = walk(plane, topo, starts, L, p, q, stream=stream)
  cur = starts.copy()
  draws = np.zeros(starts.size, dtype=np.int64)
  ref = [cur.copy()]
  for _ in range(L):
    inside = (cur >= 0) & (cur < n)
    d = np.where(inside, indptr[np.clip(cur, 0, n - 1) + 1] - indptr[np.clip(cur, 0, n - 1)], 0)
    r = philox_draw(SEED, stream, np.arange(starts.size), draws)
    pos = bounded(r, d)
    nxt = np.where(d > 0, indices[np.where(d > 0, indptr[np.clip(cur, 0, n - 1)] + pos, 0)], cur)
    draws += d > 0
    cur = nxt
    ref.append(cur.copy())
  ref = np.stack(ref, 1)
  bad = int((got != ref).any(1).sum())
  assert bad == 0, f'{plane}: {bad} of {starts.size} walks differ from the Philox replay'


# node2vec: gadget a -> {b} + X, b -> {a x n_ret} + X + Y; X, Y have no out-edges.  A walker from a reaches b with
# probability 1 / (1 + |X|), and its second step is then the node2vec law with previous node a: weight 1/p for a,
# 1 for the members of X (a's neighbours), 1/q for Y, per position.
PQ = [(0.25, 4.0), (4.0, 0.25), (0.125, 8.0), (8.0, 0.125), (0.3, 1.7), (1.0, 1.0)]
# (n_ret, n_in, n_out) of b's row; the widest row is directed (a is not in it)
SHAPES_OUT = [(1, 0, 1), (1, 1, 31), (1, 1, 998), (0, 1, 4999)]
SHAPES_RET = [(1, 0, 1), (31, 1, 1), (998, 1, 1), (0, 1, 4999)]
N2V_WALKERS = 1 << 17
N2V_COPIES = 8


def n2v_weights(p, q):
  return {'ret': 1.0 / p, 'in': 1.0, 'out': 1.0 / q}


def shapes_for(p, q):
  w = n2v_weights(p, q)
  return SHAPES_RET if w['ret'] < min(w['in'], w['out']) else SHAPES_OUT


def gadget(n_ret, n_in, n_out, copies=N2V_COPIES):
  """N2V_COPIES disjoint gadgets; node a of copy c is c * G, b is c * G + 1, X follows, then Y."""
  G = 2 + n_in + n_out
  rows = []
  for c in range(copies):
    B = c * G
    X = list(range(B + 2, B + 2 + n_in))
    Y = list(range(B + 2 + n_in, B + G))
    rows += [[B + 1] + X, [B] * n_ret + X + Y] + [[]] * (n_in + n_out)
  return csr_graph(*from_rows(rows)), G


def n2v_law(p, q, n_ret, n_in, n_out, bins=64):
  """Cells (node a, each X member, Y in <= `bins` contiguous groups) of b's row and their exact float64 probabilities,
  plus a map from a local id (node - c * G) to its cell."""
  w = n2v_weights(p, q)
  Z = n_ret * w['ret'] + n_in * w['in'] + n_out * w['out']
  G = 2 + n_in + n_out
  cell = np.full(G, -1, dtype=np.int64)
  probs = [n_ret * w['ret'] / Z]
  cell[0] = 0
  for j in range(n_in):
    cell[2 + j] = len(probs)
    probs.append(w['in'] / Z)
  nb = min(bins, n_out)
  edges = np.linspace(0, n_out, nb + 1).astype(np.int64)
  group = np.searchsorted(edges, np.arange(n_out), side='right') - 1
  cell[2 + n_in:] = len(probs) + group
  probs += list(np.diff(edges) * w['out'] / Z)
  return np.array(probs), cell


def check_n2v(w, G, p, q, shape, label):
  n_ret, n_in, n_out = shape
  B = (np.arange(w.shape[0]) % N2V_COPIES) * G
  assert np.array_equal(w[:, 0], B)
  first = w[:, 1] - B
  assert np.all((first == 1) | ((first >= 2) & (first < 2 + n_in))), f'{label}: step 1 left a\'s row'
  at_b = first == 1
  if n_in:
    binom_check(int(at_b.sum()), w.shape[0], 1.0 / (1 + n_in), f'{label} step 1 reaches b')
  assert np.array_equal(w[~at_b, 2], w[~at_b, 1]), f'{label}: a walker left a node without out-edges'
  second = w[at_b, 2] - B[at_b]
  probs, cell = n2v_law(p, q, *shape)
  ok = (second >= 0) & (second < G)
  assert ok.all() and np.all(cell[second] >= 0), f'{label}: step 2 left b\'s row'
  chisq(np.bincount(cell[second], minlength=probs.size), probs * at_b.sum(), f'{label} step 2')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('pq', PQ, ids=lambda pq: f'p{pq[0]}-q{pq[1]}')
@pytest.mark.parametrize('wide', range(4))
def test_node2vec_second_step_law(plane, pq, wide):
  """The second step of a p / q walk against its exact float64 law, on rows of degree 2, 33, 1000 and 5000 whose
  candidates almost all carry the smallest weight (the rejection sampler's worst case), the widest one directed."""
  p, q = pq
  shape = shapes_for(p, q)[wide]
  topo, G = gadget(*shape)
  starts = (np.arange(N2V_WALKERS) % N2V_COPIES) * G
  w = walk(plane, topo, starts, 2, p, q, stream=20 + wide)
  check_n2v(w, G, p, q, shape, f'{plane} p={p} q={q} row {shape}')


@pytest.mark.gpu
@pytest.mark.parametrize('pq', [(0.25, 4.0), (0.3, 1.7), (8.0, 0.125), (1.0, 1.0)])
def test_node2vec_gpu_matches_cpu(pq):
  """Same seed, same stream: the planes' p / q walks are bit-identical, at dyadic and non-dyadic p and q."""
  rng = np.random.default_rng(3)
  n = 4000
  deg = rng.integers(0, 24, n)
  deg[7] = 4000
  rows = [rng.integers(0, n, d) for d in deg]
  for v in range(0, n, 3):                            # make many edges reciprocal: 'in' candidates
    for c in rows[v][:4]:
      rows[c] = np.append(rows[c], v)
  topo = csr_graph(*from_rows(rows))
  starts = np.concatenate([np.arange(n), np.full(2000, 7)])
  a = walk('cpu', topo, starts, 10, *pq, stream=30)
  b = walk('gpu', topo, starts, 10, *pq, stream=30)
  bad = int((a != b).any(1).sum())
  assert bad == 0, f'{bad} of {starts.size} walks differ between GPU and CPU'
  shape = (998, 1, 1) if pq[0] > 1 else (1, 1, 998)
  topo, _ = gadget(*shape)
  s = (np.arange(1 << 14) % N2V_COPIES) * (2 + sum(shape[1:]))
  assert np.array_equal(walk('cpu', topo, s, 2, *pq, stream=31), walk('gpu', topo, s, 2, *pq, stream=31))


@pytest.mark.gpu
@pytest.mark.parametrize('pq', [(1.0, 1.0), (0.3, 1.7), (0.125, 8.0)])
def test_walk_memory_tiers(pq):
  """HBM with int32 and int64 column ids, ZERO_COPY and a two-shard table walk the same walks."""
  rng = np.random.default_rng(4)
  n = 3000
  deg = rng.integers(0, 30, n)
  deg[1500] = 3000                                    # a hub right at the shard boundary
  rows = [rng.integers(0, n, d) for d in deg]
  topo = csr_graph(*from_rows(rows))
  starts = np.concatenate([np.arange(n), np.full(1000, 1500), [n + 3, -2]])
  ref = walk('cpu', topo, starts, 8, *pq, stream=40)
  for tier in TIERS:
    got = walk('gpu', tier_graph(topo, tier), starts, 8, *pq, stream=40)
    assert np.array_equal(got, ref), tier


@pytest.mark.parametrize('plane', PLANES)
def test_walk_argument_errors(plane):
  """r = max(1, 1/p, 1/q) / min(1, 1/p, 1/q) > 64, p or q <= 0 or not finite, and a negative length raise on both
  planes, from NeighborSampler (ValueError) and from the bindings (RuntimeError); r = 64 is accepted."""
  topo = circulant()
  g = glt.data.Graph(topo, 'CPU' if plane == 'cpu' else 'CUDA', None if plane == 'cpu' else 0)
  ns = NeighborSampler(g, [2], seed=SEED, device=DEV if plane == 'gpu' else None)
  starts = torch.arange(8, device=DEV if plane == 'gpu' else 'cpu')
  bad = [(0.0625, 8.0), (8.0, 0.0625), (0.125, 16.0), (0.01, 1.0), (1.0, 100.0), (0.0, 1.0), (1.0, 0.0),
         (-1.0, 1.0), (1.0, -2.0), (math.nan, 1.0), (1.0, math.nan), (math.inf, 1.0), (1.0, math.inf)]
  for p, q in bad:
    with pytest.raises(ValueError):
      ns.random_walk(starts, 3, p, q)
    with pytest.raises(RuntimeError):
      walk(plane, topo if plane == 'cpu' else g, np.arange(8), 3, p, q)
  with pytest.raises(ValueError):
    ns.random_walk(starts, -1)
  with pytest.raises(RuntimeError):
    walk(plane, topo if plane == 'cpu' else g, np.arange(8), -1)
  for p, q in [(0.125, 8.0), (8.0, 0.125), (0.125, 1.0), (64.0, 1.0), (1.0, 1 / 64)]:
    assert ns.random_walk(starts, 3, p, q).shape == (8, 4)


# --------------------------------------------------------------------------- induced subgraphs
SUB_ROWS, SUB_COLS = 6000, 6100                       # columns 6000 .. 6099 have no row


def subgraph_case():
  """Rows at the warp-ballot boundary (31, 32, 33), a hub of 5000, a row entirely outside the node set, repeated
  columns, columns with no row; the node set has duplicates, is unsorted and holds ids with no row."""
  rng = np.random.default_rng(6)
  in_set = rng.random(SUB_COLS) < 0.5
  in_set[:9] = True
  in_set[[6000, 6001, 6002]] = True
  inside, outside = np.nonzero(in_set)[0], np.nonzero(~in_set)[0]
  rows = [rng.integers(0, SUB_COLS, 5000)]
  rows += [rng.choice(inside, d) for d in (31, 32, 33)]
  rows += [rng.integers(0, SUB_COLS, d) for d in (31, 32, 33)]
  rows += [rng.choice(outside, 40)]
  rows += [np.array([3, 3, 3, 6001, 6001, 2])]
  rows += [rng.integers(0, SUB_COLS, d) for d in rng.integers(0, 12, SUB_ROWS - 9)]
  indptr, indices = from_rows(rows)
  eids = np.arange(indices.size, dtype=np.int64) * 7 + 3
  topo = csr_graph(indptr, indices, eids)
  nodes = np.concatenate([np.nonzero(in_set)[0], [10 ** 9, 10 ** 9 + 1]])
  nodes = np.concatenate([nodes, rng.choice(nodes, 500)])
  rng.shuffle(nodes)
  return topo, nodes


def subgraph_reference(topo, nodes, num_seeds):
  ip, ind, ei = topo.indptr.numpy(), topo.indices.numpy(), topo.edge_ids.numpy()
  uniq = np.unique(nodes)
  row = np.repeat(np.arange(ip.size - 1), np.diff(ip))
  keep = np.isin(row, uniq) & np.isin(ind, uniq)
  # CSR order is (row, position in row): rows ascending == local ids ascending
  return uniq, np.searchsorted(uniq, ind[keep]), np.searchsorted(uniq, row[keep]), ei[keep], \
      np.searchsorted(uniq, nodes[:num_seeds])


def check_subgraph(out, ref, label):
  names = ['node', 'row', 'col', 'eids', 'mapping']
  for name, a, b in zip(names, out, ref):
    a = a.cpu().numpy()
    assert a.shape == b.shape and np.array_equal(a, b), f'{label}: {name} differs'


@pytest.mark.parametrize('tier', ['CPU'] + [pytest.param(t, marks=pytest.mark.gpu) for t in TIERS])
def test_node_subgraph_exact(tier):
  """NeighborSampler.node_subgraph against a brute-force filter of the COO: the sorted unique node list, edges in
  (row, position) order, reversed orientation, edge ids and the seeds' mapping."""
  topo, nodes = subgraph_case()
  g = glt.data.Graph(topo, 'CPU') if tier == 'CPU' else tier_graph(topo, tier)
  dev = DEV if tier != 'CPU' else torch.device('cpu')
  ns = NeighborSampler(g, None, with_edge=True, seed=SEED, device=DEV if tier != 'CPU' else None)
  out = ns.node_subgraph(torch.from_numpy(nodes).to(dev), 100)
  check_subgraph(out, subgraph_reference(topo, nodes, 100), tier)
  ns = NeighborSampler(g, None, with_edge=False, seed=SEED, device=DEV if tier != 'CPU' else None)
  node, row, col, eids, _ = ns.node_subgraph(torch.from_numpy(nodes).to(dev), 0)
  assert eids is None
  ref = subgraph_reference(topo, nodes, 0)
  check_subgraph((node, row, col), ref[:3], f'{tier} without edge ids')
  sub = ns.subgraph(NodeSamplerInput(torch.from_numpy(nodes[:50]).to(dev)))
  ref = subgraph_reference(topo, nodes[:50], 50)
  check_subgraph((sub.node, sub.row, sub.col, sub.metadata), (ref[0], ref[1], ref[2], ref[4]), f'{tier} subgraph()')
  empty = ns.node_subgraph(torch.zeros(0, dtype=torch.int64, device=dev), 0)
  assert all(t.numel() == 0 for t in empty[:3])


@pytest.mark.gpu
def test_device_table_subgraph_ballot_rows():
  """DeviceTable.subgraph on node sets that hold only rows of degree 31 / 32 / 33 / 5000 and all their columns, so
  every lane of a ballot hits, and on one that holds none of a row's columns."""
  topo, _ = subgraph_case()
  g = glt.data.Graph(topo, 'CUDA', 0)
  ip, ind = topo.indptr.numpy(), topo.indices.numpy()
  for rows in ([1], [2], [3], [0], [1, 2, 3, 0], [7]):
    nodes = np.unique(np.concatenate([rows] + [ind[ip[r]:ip[r + 1]] for r in rows]))
    if rows == [7]:
      nodes = np.array([7])
    t = nat().DeviceTable(0, nodes.size)
    t.init_ordered(torch.from_numpy(nodes).to(DEV))
    r, c, e = t.subgraph(g.graph_handler, t.size(), True)
    ref = subgraph_reference(topo, nodes, 0)
    assert np.array_equal(r.cpu().numpy(), ref[2]) and np.array_equal(c.cpu().numpy(), ref[1]), rows
    assert np.array_equal(e.cpu().numpy(), ref[3]), rows


# --------------------------------------------------------------------------- full neighbourhoods and degrees
def full_reference(topo, ids):
  ip, ind, ei = topo.indptr.numpy(), topo.indices.numpy(), topo.edge_ids.numpy()
  n = ip.size - 1
  deg = np.array([ip[v + 1] - ip[v] if 0 <= v < n else 0 for v in ids], dtype=np.int64)
  pos = [np.arange(ip[v], ip[v + 1]) for v, d in zip(ids, deg) if d]
  pos = np.concatenate(pos) if pos else np.zeros(0, dtype=np.int64)
  return ind[pos], deg, ei[pos]


def full_ids(topo):
  n = topo.indptr.numel() - 1
  rng = np.random.default_rng(8)
  return [np.zeros(0, dtype=np.int64), np.array([0]), np.array([0, 0, 1, 2, 3, 0]),
          np.concatenate([rng.permutation(n), rng.integers(0, n, 500), [n, n + 5, 10 ** 9, -1, 0]])]


@pytest.mark.gpu
@pytest.mark.parametrize('tier', TIERS)
def test_full_neighbors_and_degrees(tier):
  """GraphHandle.lookup_degree and full_neighbors, with and without edge ids, exact against the CSR: empty input,
  repeated ids, ids outside every shard (degree 0), a hub of 5000."""
  topo, _ = subgraph_case()
  h = tier_graph(topo, tier).graph_handler
  for ids in full_ids(topo):
    nbr, deg, eid = full_reference(topo, ids)
    d = torch.from_numpy(ids).to(DEV)
    assert np.array_equal(h.lookup_degree(d).cpu().numpy(), deg)
    for with_edge in (False, True):
      a, c, e = h.full_neighbors(d, with_edge)
      assert np.array_equal(c.cpu().numpy(), deg) and np.array_equal(a.cpu().numpy(), nbr), (tier, ids.size)
      if with_edge:
        assert np.array_equal(e.cpu().numpy(), eid), (tier, ids.size)


@pytest.mark.parametrize('tier', ['CPU'] + [pytest.param(t, marks=pytest.mark.gpu) for t in TIERS])
def test_neighbor_sampler_full_fanout(tier):
  """NeighborSampler with fanout -1 returns exactly the CSR neighbourhoods, with edge ids."""
  topo, _ = subgraph_case()
  g = glt.data.Graph(topo, 'CPU') if tier == 'CPU' else tier_graph(topo, tier)
  dev = DEV if tier != 'CPU' else torch.device('cpu')
  ns = NeighborSampler(g, [-1], with_edge=True, seed=SEED, device=DEV if tier != 'CPU' else None)
  for ids in full_ids(topo):
    nbr, deg, eid = full_reference(topo, ids)
    out = ns.sample_one_hop(torch.from_numpy(ids).to(dev), -1)
    assert np.array_equal(out.nbr_num.cpu().numpy(), deg), (tier, ids.size)
    assert np.array_equal(out.nbr.cpu().numpy(), nbr) and np.array_equal(out.edge.cpu().numpy(), eid)


@pytest.mark.gpu
def test_missing_edge_ids_raise():
  """A device table built without edge ids refuses every call that would return them, and answers the rest."""
  topo, nodes = subgraph_case()
  g = two_shards(topo, 3000, eids=False)
  h = g.graph_handler
  ids = torch.arange(0, 6000, 7, device=DEV)
  with pytest.raises(RuntimeError, match='graph has no edge ids'):
    h.full_neighbors(ids, True)
  with pytest.raises(RuntimeError, match='graph has no edge ids'):
    h.sample_one_hop(ids, 4, True, False, False, SEED, 0)
  t = nat().DeviceTable(0, 16)
  t.init_ordered(ids[:16].contiguous())
  with pytest.raises(RuntimeError, match='graph has no edge ids'):
    t.subgraph(h, t.size(), True)
  with pytest.raises(RuntimeError):
    NeighborSampler(g, [-1], with_edge=True, device=DEV).sample_one_hop(ids, -1)
  nbr, deg, _ = full_reference(topo, ids.cpu().numpy())
  a, c, e = h.full_neighbors(ids, False)
  assert e is None and np.array_equal(a.cpu().numpy(), nbr) and np.array_equal(c.cpu().numpy(), deg)
  out = NeighborSampler(g, None, with_edge=False, device=DEV).node_subgraph(torch.from_numpy(nodes).to(DEV), 0)
  check_subgraph(out[:3], subgraph_reference(topo, nodes, 0)[:3], 'no edge ids')


# --------------------------------------------------------------------------- hotness
def nbr_prob_reference(topo, nbr_topo, last, nbr_last, k):
  """float64 cur[v] = 1 - (1 - last[v]) prod_u (1 - p_u min(1, k / deg(u))) over v's columns u with deg(u) > 0 and
  u < len(nbr_last); 0 for rows of degree 0 and entries past the graph's rows.  Also each entry's float32 bound."""
  ip, ind, nip = topo.indptr.numpy(), topo.indices.numpy(), nbr_topo.indptr.numpy()
  last, nbr_last = last.astype(np.float64), nbr_last.astype(np.float64)
  n, nn, nrows = last.size, nbr_last.size, nip.size - 1
  rows = min(n, ip.size - 1)
  deg = np.diff(ip)[:rows]
  u = ind[:ip[rows]]
  ok = (u >= 0) & (u < nn)
  du = np.where(ok & (u < nrows), nip[np.clip(u + 1, 0, nrows)] - nip[np.clip(u, 0, nrows)], 0)
  ok &= du > 0
  pu = np.where(ok, nbr_last[np.clip(u, 0, nn - 1)], 0.0)
  scale = np.ones_like(pu) if k < 0 else np.minimum(1.0, k / np.maximum(du, 1))
  fac = 1.0 - pu * scale                              # skipped neighbours have p_u = 0: a factor of 1
  prod = np.ones(rows)
  for v in np.nonzero(deg)[0]:
    prod[v] = np.prod(fac[ip[v]:ip[v + 1]])
  cur = np.zeros(n)
  cur[:rows] = np.where(deg > 0, 1.0 - (1.0 - last[:rows]) * prod, 0.0)
  bound = np.zeros(n)
  bound[:rows] = (deg + 4) * 2.0 ** -24
  return cur, bound


def hot_graph():
  """Rows of degree 0, hubs above 32 (the cross-lane product), columns past every row and past nbr_last."""
  rng = np.random.default_rng(9)
  n = 3000
  deg = rng.integers(0, 20, n)
  deg[::50] = 0
  deg[[3, 4, 5]] = [33, 700, 4000]
  rows = [rng.integers(0, n + 200, d) for d in deg]
  return csr_graph(*from_rows(rows))


def run_nbr_prob(plane, topo, last, nbr_last, k, nbr_topo=None):
  nbr_topo = topo if nbr_topo is None else nbr_topo
  if plane == 'cpu':
    return nat().cpu_nbr_prob(topo.indptr, topo.indices, nbr_topo.indptr, torch.from_numpy(last),
                              torch.from_numpy(nbr_last), k).numpy()
  g, ng = glt.data.Graph(topo, 'CUDA', 0), glt.data.Graph(nbr_topo, 'CUDA', 0)
  return g.graph_handler.nbr_prob(ng.graph_handler, torch.from_numpy(last).to(DEV),
                                  torch.from_numpy(nbr_last).to(DEV), k).cpu().numpy()


def check_bound(got, ref, bound, label):
  err = np.abs(got.astype(np.float64) - ref)
  worst = int(np.argmax(err / np.maximum(bound, 1e-30)))
  print(f'{label}: max error {err.max():.3g}, worst entry {worst} at {err[worst] / max(bound[worst], 1e-30):.3g} '
        f'of its bound')
  assert np.all(err <= bound), f'{label}: entry {worst} off by {err[worst]:.3g} > {bound[worst]:.3g}'


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('k', [-1, 1, 5, 5000])
@pytest.mark.parametrize('n_last,n_nbr', [(3000, 3000), (3300, 3100), (3100, 2900), (2500, 3300)])
def test_nbr_prob_formula(plane, k, n_last, n_nbr):
  """One hotness hop against its float64 formula: k < 0 (all neighbours), k = 1, 5 and k >= every degree; `last`
  longer and shorter than the graph's rows, `nbr_last` shorter than the largest column id."""
  topo = hot_graph()
  rng = np.random.default_rng(k + 7 * n_last)
  last = rng.random(n_last).astype(np.float32)
  nbr_last = rng.random(n_nbr).astype(np.float32)
  nbr_last[::11] = 1.0
  nbr_last[::13] = 0.0
  got = run_nbr_prob(plane, topo, last, nbr_last, k)
  ref, bound = nbr_prob_reference(topo, topo, last, nbr_last, k)
  assert got.shape == (n_last,)
  check_bound(got, ref, bound, f'{plane} nbr_prob k={k} last {n_last} nbr_last {n_nbr}')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('fanouts', [[-1, 3], [5, 5000]])
def test_sample_prob_two_hops(plane, fanouts):
  """NeighborSampler.sample_prob over two hops against the float64 chain; hop 2's bound adds hop 1's bounds of the
  row and of its neighbours (every partial derivative of the formula lies in [0, 1])."""
  topo = hot_graph()
  node_cnt = 3150
  seeds = np.arange(0, 3000, 17)
  g = glt.data.Graph(topo, 'CPU') if plane == 'cpu' else glt.data.Graph(topo, 'CUDA', 0)
  dev = DEV if plane == 'gpu' else torch.device('cpu')
  ns = NeighborSampler(g, fanouts, seed=SEED, device=DEV if plane == 'gpu' else None)
  got = ns.sample_prob(NodeSamplerInput(torch.from_numpy(seeds).to(dev)), node_cnt).cpu().numpy()
  last = np.full(node_cnt, np.float32(0.01), dtype=np.float32)
  last[seeds] = 1.0
  ref1, b1 = nbr_prob_reference(topo, topo, last, last, fanouts[0])
  ref2, b2 = nbr_prob_reference(topo, topo, ref1, ref1, fanouts[1])
  ip, ind = topo.indptr.numpy(), topo.indices.numpy()
  rows = ip.size - 1
  prop = np.zeros(node_cnt)
  for v in range(rows):
    if ip[v + 1] > ip[v]:
      u = ind[ip[v]:ip[v + 1]]
      prop[v] = b1[v] + b1[u[u < node_cnt]].sum()
  check_bound(got, ref2, b2 + prop + 2.0 ** -24, f'{plane} sample_prob {fanouts}')


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('ks', [(-1, 2), (3, 40)])
def test_hetero_sample_prob(plane, ks):
  """_hetero_sample_prob on a user -> item / item -> user schema: one hop per relation against float64, each node
  type's count past its relation's rows."""
  rng = np.random.default_rng(10)
  nu, ni = 300, 500
  udeg = rng.integers(0, 40, nu)
  udeg[[0, 1]] = [0, 450]
  src = np.repeat(np.arange(nu), udeg)
  dst = np.concatenate([rng.choice(ni, d, replace=False) for d in udeg])
  fwd = glt.data.Topology(torch.from_numpy(np.stack([src, dst])), layout='CSR', num_nodes=None)
  rev = glt.data.Topology(torch.from_numpy(np.stack([dst, src])), layout='CSR', num_nodes=None)
  uto, rto = ('u', 'to', 'i'), ('i', 'rev', 'u')
  mode = 'CPU' if plane == 'cpu' else 'CUDA'
  graphs = {uto: glt.data.Graph(fwd, mode, None if plane == 'cpu' else 0),
            rto: glt.data.Graph(rev, mode, None if plane == 'cpu' else 0)}
  ns = NeighborSampler(graphs, {uto: [ks[0]], rto: [ks[1]]}, seed=SEED, device=DEV if plane == 'gpu' else None)
  dev = DEV if plane == 'gpu' else torch.device('cpu')
  seeds = torch.arange(0, nu, 7, device=dev)
  cnt = {'u': nu + 20, 'i': ni + 10}
  got = {k: v.cpu().numpy() for k, v in ns.sample_prob(NodeSamplerInput(seeds, input_type='u'), cnt).items()}
  pu = np.full(cnt['u'], np.float32(0.005), dtype=np.float32)
  pu[seeds.cpu().numpy()] = 1.0
  pi = np.full(cnt['i'], np.float32(0.005), dtype=np.float32)
  cu, bu = nbr_prob_reference(fwd, rev, pu, pi, ks[1])      # k of the relation pointing back (i -> u)
  ci, bi = nbr_prob_reference(rev, fwd, pi, pu, ks[0])
  check_bound(got['u'], np.maximum(pu, cu), bu + 2.0 ** -23, f'{plane} hetero users {ks}')
  check_bound(got['i'], np.maximum(pi, ci), bi + 2.0 ** -23, f'{plane} hetero items {ks}')


# --------------------------------------------------------------------------- negative sampling, padded
def negatives(plane, topo, num_rows, num_cols, req, trials, padding, stream):
  if plane == 'cpu':
    r, c = nat().cpu_negative_sample(topo.indptr, topo.indices, num_rows, num_cols, req, trials, padding, True,
                                     SEED, stream)
    return r.numpy(), c.numpy()
  h = glt.data.Graph(topo, 'CUDA', 0).graph_handler
  r, c, count = h.negative_sample(num_rows, num_cols, req, trials, padding, SEED, stream)
  n = int(count.item())
  return r[:n].cpu().numpy(), c[:n].cpu().numpy()


def dense_graph():
  """20 rows over 40 columns, 70 % of the cells edges."""
  rng = np.random.default_rng(12)
  adj = rng.random((20, 40)) < 0.7
  r, c = np.nonzero(adj)
  return glt.data.Topology(torch.from_numpy(np.stack([r, c])), layout='CSR', num_nodes=None), adj


@pytest.mark.parametrize('plane', PLANES)
@pytest.mark.parametrize('num_rows,num_cols,trials', [(20, 40, 0), (25, 40, 0), (25, 31, 0), (20, 40, 2),
                                                     (28, 40, 3)])
def test_padded_negatives(plane, num_rows, num_cols, trials):
  """padding=True returns exactly req pairs; a pair is a strict negative with probability 1 - f^trials (f the share
  of the rectangle that is edges) and otherwise a uniform cell of the whole rectangle, rows past the graph included
  (trials = 0: only padded draws)."""
  topo, adj = dense_graph()
  full = np.zeros((num_rows, num_cols), dtype=bool)
  full[:20, :min(40, num_cols)] = adj[:, :min(40, num_cols)]
  req = 1 << 18
  r, c = negatives(plane, topo, num_rows, num_cols, req, trials, True, 140 + trials)
  assert r.size == req and c.size == req
  assert r.min() >= 0 and r.max() < num_rows and c.min() >= 0 and c.max() < num_cols
  R = num_rows * num_cols
  f = full.sum() / R
  pad = f ** trials / R
  probs = np.where(full.ravel(), pad, pad + (1 - f ** trials) / (R - full.sum()))
  assert abs(probs.sum() - 1) < 1e-9
  chisq(np.bincount(r * num_cols + c, minlength=R), probs * req,
        f'{plane} padded negatives {num_rows}x{num_cols} trials={trials}')
  sampler = glt.sampler.RandomNegativeSampler(
    glt.data.Graph(topo, 'CPU') if plane == 'cpu' else glt.data.Graph(topo, 'CUDA', 0),
    'CPU' if plane == 'cpu' else 'CUDA', seed=SEED)
  assert sampler.sample(1000, trials_num=trials, padding=True).shape == (2, 1000)
