"""sm_90a kernels vs. the CPU reference ops / plain PyTorch fp32 (needs an H100)."""
import sys

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.sampler import NeighborSampler, NodeSamplerInput
from helpers import adjacency_sets, canonical_edges, ring_dataset, rmat_csr

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _graphs(num_nodes=3000, num_edges=60000, weights=False, seed=0):
  ei, topo = rmat_csr(num_nodes, num_edges, seed)
  if weights:
    w = (torch.arange(ei.shape[1]) % 7 + 1).float()
    topo = glt.data.Topology(ei, edge_weights=w, layout='CSR', num_nodes=num_nodes)
  return topo, glt.data.Graph(topo, 'CPU'), glt.data.Graph(topo, 'CUDA', 0)


@pytest.mark.parametrize('k', [3, 10, 25, 40])
def test_one_hop_matches_cpu(native, k):
  topo, gc, gg = _graphs()
  seeds = torch.randperm(3000)[:700]
  for with_edge in (False, True):
    sc = NeighborSampler(gc, [k], with_edge=with_edge, seed=11)
    sg = NeighborSampler(gg, [k], with_edge=with_edge, seed=11, device=DEV)
    a = sc.sample_one_hop(seeds, k, stream=5)
    b = sg.sample_one_hop(seeds.to(DEV), k, stream=5)
    assert torch.equal(a.nbr_num, b.nbr_num.cpu())
    assert torch.equal(a.nbr, b.nbr.cpu())          # same Philox streams -> identical picks
    if with_edge:
      assert torch.equal(a.edge, b.edge.cpu())


def test_one_hop_zero_copy_and_full(native):
  topo, gc, _ = _graphs(500, 9000)
  gz = glt.data.Graph(topo, 'ZERO_COPY', 0)
  seeds = torch.arange(0, 500, 3)
  a = NeighborSampler(gc, [4], seed=1).sample_one_hop(seeds, 4, stream=0)
  b = NeighborSampler(gz, [4], seed=1, device=DEV).sample_one_hop(seeds.to(DEV), 4, stream=0)
  assert torch.equal(a.nbr, b.nbr.cpu())
  a = NeighborSampler(gc, [-1], with_edge=True).sample_one_hop(seeds, -1)
  b = NeighborSampler(gz, [-1], with_edge=True, device=DEV).sample_one_hop(seeds.to(DEV), -1)
  assert torch.equal(a.nbr, b.nbr.cpu()) and torch.equal(a.edge, b.edge.cpu())
  assert torch.equal(a.nbr_num, b.nbr_num.cpu())


def test_weighted_one_hop_statistics(native):
  indptr = torch.tensor([0, 4])
  topo = glt.data.Topology((indptr, torch.tensor([10, 11, 12, 13])), edge_weights=torch.tensor([1., 1., 2., 4.]),
                           input_layout='CSR', layout='CSR')
  g = glt.data.Graph(topo, 'CUDA', 0)
  s = NeighborSampler(g, [1], with_weight=True, seed=3, device=DEV)
  hits = torch.zeros(4)
  seeds = torch.zeros(1, dtype=torch.int64, device=DEV)
  for t in range(3000):
    o = s.sample_one_hop(seeds, 1, stream=t)
    hits[o.nbr.item() - 10] += 1
  p = hits / 3000
  assert (p - torch.tensor([1., 1., 2., 4.]) / 8).abs().max() < 0.04


@pytest.mark.parametrize('fanouts', [[3, 2], [15, 10, 5], [40, 2]])
def test_arena_multihop_matches_cpu(native, fanouts):
  topo, gc, gg = _graphs(5000, 100000)
  seeds = torch.randperm(5000)[:333]
  sc = NeighborSampler(gc, fanouts, with_edge=True, seed=21)
  sg = NeighborSampler(gg, fanouts, with_edge=True, seed=21, device=DEV)
  a = sc.sample_from_nodes(seeds)
  b = sg.sample_from_nodes(seeds.to(DEV))
  assert a.num_sampled_nodes == b.num_sampled_nodes
  assert a.num_sampled_edges == b.num_sampled_edges
  assert torch.equal(a.node[:333], b.node[:333].cpu())            # seeds keep their order
  # hop-contiguous node sets match; ids inside a hop may be permuted
  off = 0
  for n in a.num_sampled_nodes:
    assert set(a.node[off:off + n].tolist()) == set(b.node[off:off + n].cpu().tolist())
    off += n
  assert canonical_edges(a) == canonical_edges(b)
  eb = dict(zip(zip(b.node[b.row].cpu().tolist(), b.node[b.col].cpu().tolist()), b.edge.cpu().tolist()))
  ea = dict(zip(zip(a.node[a.row].tolist(), a.node[a.col].tolist()), a.edge.tolist()))
  assert ea == eb
  # per-hop edge blocks: targets of hop h are nodes of hop h-1
  cum = [0]
  for n in b.num_sampled_nodes:
    cum.append(cum[-1] + n)
  e0 = 0
  for h, ne in enumerate(b.num_sampled_edges):
    cols = b.col[e0:e0 + ne]
    assert int(cols.min()) >= cum[h] and int(cols.max()) < cum[h + 1]
    e0 += ne


def test_generic_path_on_gpu_with_full_fanout(native):
  ds = ring_dataset(40, graph_mode='CUDA', device=0)
  s = NeighborSampler(ds.graph, [-1, 2], device=DEV)
  out = s.sample_from_nodes(torch.tensor([0, 10], device=DEV))
  assert set(out.node.cpu().tolist()) == {0, 1, 2, 3, 4, 10, 11, 12, 13, 14}
  src, dst = out.node[out.row], out.node[out.col]
  assert torch.all(((src - dst) % 40 == 1) | ((src - dst) % 40 == 2))


@pytest.mark.parametrize('dtype,width', [(torch.float32, 100), (torch.bfloat16, 128), (torch.float16, 7),
                                         (torch.int64, 1), (torch.uint8, 33), (torch.float64, 16),
                                         (torch.float32, 1024)])
def test_unified_tensor_gather(native, dtype, width):
  n = 5000
  if dtype.is_floating_point:
    full = torch.randn(n, width).to(dtype)
  else:
    full = torch.randint(0, 100, (n, width)).to(dtype)
  ut = glt.data.UnifiedTensor(0, dtype)
  ut.init_from([full[:2000], full[2000:3500], full[3500:]], [0, 0, -1])   # 2 HBM parts + pinned host
  ids = torch.randint(0, n, (3000,))
  got = ut[ids.to(DEV)]
  assert torch.equal(got.cpu(), full[ids])
  assert ut.shape == [n, width]


@pytest.mark.parametrize('dtype,width', [(torch.bfloat16, 128), (torch.float32, 128), (torch.float32, 1024),
                                         (torch.int64, 2)])
def test_gather_large_lookup_four_rows_in_flight(native, dtype, width):
  """Large lookups take the 4-rows-per-group variant of k_gather_vec: also cover negative ids,
  the id2index indirection, a device-side row count and a ragged tail."""
  n, m = 20000, 150_001
  full = (torch.randn(n, width) * 50).to(dtype)
  ut = glt.data.UnifiedTensor(0, dtype)
  ut.init_from([full[:9000], full[9000:15000], full[15000:]], [0, 0, -1])
  ids = torch.randint(0, n, (m,))
  ids[::97] = -1
  perm = torch.randperm(n)
  table = ut._table()
  got = table.gather(ids.to(DEV), perm.to(DEV), 0).cpu()
  exp = full[perm[ids.clamp(min=0)]]
  exp[ids < 0] = 0
  assert torch.equal(got, exp)
  out = torch.full((m, width), 7, dtype=dtype, device=DEV)
  n_dev = torch.tensor([100_000], dtype=torch.int32, device=DEV)
  table.gather_into(ids.to(DEV), None, n_dev, out)
  exp2 = full[ids.clamp(min=0)]
  exp2[ids < 0] = 0
  exp2[100_000:] = 0                       # rows past the device-side count are zero-filled
  assert torch.equal(out.cpu(), exp2)
  # ids beyond the id2index table are answered with zero rows, not an out-of-bounds read
  oob = table.gather(torch.tensor([5, n + 10, 2 ** 40], device=DEV), perm.to(DEV), 0).cpu()
  assert torch.equal(oob[0], full[perm[5]]) and oob[1:].abs().sum() == 0


def test_feature_split_and_reorder(native):
  ei, topo = rmat_csr(2000, 30000)
  feat = glt.utils.id_features(2000, 16)
  for ratio in (0.0, 0.3, 1.0):
    sorted_feat, id2idx = glt.data.sort_by_in_degree(feat, ratio, topo)
    f = glt.data.Feature(sorted_feat, id2idx, split_ratio=ratio, device=0)
    ids = torch.randint(0, 2000, (777,), device=DEV)
    out = f[ids]
    assert torch.equal(out[:, 0].long(), ids)
    assert torch.equal(f.cpu_get(ids.cpu())[:, 0].long(), ids.cpu())


def test_negative_sampler_gpu(native):
  ei, topo = rmat_csr(300, 6000)
  g = glt.data.Graph(topo, 'CUDA', 0)
  edges = set(zip(ei[0].tolist(), ei[1].tolist()))
  ns = glt.sampler.RandomNegativeSampler(g, 'CUDA')
  out = ns.sample(2000, trials_num=5)
  assert 1500 < out.shape[1] <= 2000
  assert all((r, c) not in edges for r, c in zip(out[0].tolist(), out[1].tolist()))
  out = ns.sample(2000, trials_num=1, padding=True)
  assert out.shape[1] == 2000
  # rows and columns are drawn independently (the reference correlates them)
  assert abs(torch.corrcoef(out.float().cpu())[0, 1]) < 0.2


def test_subgraph_gpu_matches_cpu(native):
  topo, gc, gg = _graphs(800, 16000)
  seeds = torch.randperm(800)[:50]
  a = NeighborSampler(gc, [3], with_edge=True, seed=4).subgraph(NodeSamplerInput(seeds))
  b = NeighborSampler(gg, [3], with_edge=True, seed=4, device=DEV).subgraph(NodeSamplerInput(seeds.to(DEV)))
  assert set(a.node.tolist()) == set(b.node.cpu().tolist())
  assert canonical_edges(a) == canonical_edges(b)
  assert torch.equal(b.node[b.metadata].cpu(), seeds)
  assert sorted(a.edge.tolist()) == sorted(b.edge.cpu().tolist())


def test_random_walk_gpu_matches_cpu(native):
  topo, gc, gg = _graphs(600, 12000)
  starts = torch.arange(0, 600, 3)
  for p, q in ((1.0, 1.0), (0.25, 4.0)):
    a = NeighborSampler(gc, [1], seed=9)
    b = NeighborSampler(gg, [1], seed=9, device=DEV)
    wa = a.random_walk(starts, 8, p, q)
    wb = b.random_walk(starts.to(DEV), 8, p, q)
    assert torch.equal(wa, wb.cpu())


def test_sample_prob_gpu_matches_cpu(native):
  topo, gc, gg = _graphs(700, 9000)
  seeds = torch.arange(0, 700, 9)
  pa = NeighborSampler(gc, [5, 3]).sample_prob(NodeSamplerInput(seeds), 700)
  pb = NeighborSampler(gg, [5, 3], device=DEV).sample_prob(NodeSamplerInput(seeds.to(DEV)), 700)
  assert torch.allclose(pa, pb.cpu(), atol=1e-5)


def test_device_table(native):
  t = native.DeviceTable(0, 1000)
  keys = torch.tensor([7, 3, 7, 9, 3, 100], device=DEV)
  ids = t.init_ordered(keys)
  assert ids.tolist() == [0, 1, 0, 2, 1, 3] and t.size() == 4
  assert t.nodes[:4].tolist() == [7, 3, 9, 100]
  more = t.insert(torch.tensor([9, 55, 56, 55, -1], device=DEV))
  assert more[0].item() == 2 and more[4].item() == -1 and more[1].item() == more[3].item()
  assert sorted(more[1:3].tolist()) == [4, 5] and t.size() == 6
  assert t.lookup(torch.tensor([100, 12345], device=DEV)).tolist() == [3, -1]
  t.clear()
  assert t.size() == 0 and t.lookup(torch.tensor([7], device=DEV)).tolist() == [-1]


def test_neighbor_loader_cuda_ring(native):
  from test_loaders_cpu import check_homo_batch
  ds = ring_dataset(40, graph_mode='CUDA', with_gpu=True, device=0, split_ratio=0.5)
  loader = glt.loader.NeighborLoader(ds, [2, 2], torch.arange(40), batch_size=8, shuffle=True, with_edge=True,
                                     device=DEV, seed=1)
  seen = []
  for b in loader:
    assert b.x.is_cuda and b.edge_index.is_cuda
    b = b.to('cpu')
    check_homo_batch(b)
    seen += b.batch.tolist()
  assert sorted(seen) == list(range(40))


def test_arena_capacity_guard(native):
  """Calibrated (too small) capacities: excess nodes are dropped and counted, nothing overflows."""
  topo, gc, gg = _graphs(5000, 100000)
  caps = [256, 300, 500, 700]
  arena = native.SamplerArena(0, 256, [10, 5, 3], False, 5000, caps)
  seeds = torch.randperm(5000, device=DEV)[:256].contiguous()
  arena.sample(gg.graph_handler, seeds, None, 3, 0, False, False, False)
  c = arena.counters.cpu().tolist()
  cum = c[:5]
  assert cum[1] == 256
  for h in range(1, 4):
    assert cum[h + 1] - cum[h] <= arena.cap_rows[h], (h, cum, arena.cap_rows)
  assert cum[4] <= arena.cap_nodes
  assert c[12] > 0                                           # something was dropped
  for h in range(3):
    rows = cum[h + 1] - cum[h]
    ell = arena.ell[h][:rows * [10, 5, 3][h]]
    assert int(ell.max()) < cum[h + 2] and int(ell.min()) >= -1
  node, row, col, _, nn, ne = arena.to_coo()
  assert node.numel() == cum[4] and int(row.max()) < node.numel() and int(row.min()) >= -1


def test_hetero_and_link_sampling_gpu_matches_cpu(native):
  """Hetero multi-hop + link sampling with negatives on the GPU (generic IdTable path)."""
  from graphlearn_for_pytorch_b200.sampler import EdgeSamplerInput, NegativeSampling
  g = torch.Generator().manual_seed(0)
  u2i = torch.stack([torch.randint(0, 300, (3000,), generator=g), torch.randint(0, 200, (3000,), generator=g)])
  i2i = torch.stack([torch.randint(0, 200, (2000,), generator=g), torch.randint(0, 200, (2000,), generator=g)])
  outs = {}
  for mode in ('CPU', 'CUDA'):
    ds = glt.data.Dataset(edge_dir='out')
    ds.init_graph({('user', 'u2i', 'item'): u2i, ('item', 'i2i', 'item'): i2i}, graph_mode=mode, device=0,
                  num_nodes={'user': 300, 'item': 200})
    s = NeighborSampler(ds.graph, [3, 2], with_edge=True, seed=5, device=DEV if mode == 'CUDA' else None)
    outs[mode] = s.sample_from_nodes(NodeSamplerInput(torch.arange(0, 300, 7), 'user'))
  a, b = outs['CPU'], outs['CUDA']
  assert set(a.row.keys()) == set(b.row.keys())
  for nt in a.node:
    assert set(a.node[nt].tolist()) == set(b.node[nt].cpu().tolist())
  for et in a.row:
    st, dt = et[0], et[2]
    ea = set(zip(a.node[st][a.row[et]].tolist(), a.node[dt][a.col[et]].tolist(), a.edge[et].tolist()))
    eb = set(zip(b.node[st][b.row[et]].cpu().tolist(), b.node[dt][b.col[et]].cpu().tolist(), b.edge[et].cpu().tolist()))
    assert ea == eb
  assert {k: v.tolist() for k, v in a.num_sampled_nodes.items()} == \
      {k: v.tolist() for k, v in b.num_sampled_nodes.items()}        # per-type int64 tensors (reference convention)
  # homogeneous link sampling with strict binary negatives on the GPU
  ds = ring_dataset(40, graph_mode='CUDA', with_gpu=True, device=0, split_ratio=1.0)
  s = NeighborSampler(ds.graph, [2], with_neg=True, seed=3, device=DEV)
  row, col = torch.tensor([0, 1, 2], device=DEV), torch.tensor([1, 3, 3], device=DEV)
  out = s.sample_from_edges(EdgeSamplerInput(row, col, neg_sampling=NegativeSampling('binary', 2)))
  eli, lab = out.metadata['edge_label_index'], out.metadata['edge_label']
  assert eli.shape == (2, 9) and lab.tolist() == [1, 1, 1] + [0] * 6
  ns, nd = out.node[eli[0, 3:]], out.node[eli[1, 3:]]
  assert torch.all(((nd - ns) % 40 != 1) & ((nd - ns) % 40 != 2))


def test_hetero_arena_igbh_shape_matches_cpu_sampler(native):
  """Native grouped hetero sampler/inducer (HeteroArena) on an IGBH-shaped schema (4 node types, 7 relations,
  3 hops, edge_dir='in'): the sampled edge SET of every relation and the node set of every type must equal the
  CPU sampler's (same Philox streams), local ids must be hop-contiguous, and the generic per-relation hop loop on
  the device must agree as well."""
  import os
  sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
  from common import synthetic_igbh
  edges, feats, labels, sizes = synthetic_igbh(3000, 1500, 60, 40, feat_dim=16, seed=1)
  seeds = torch.arange(5, 3000, 11)[:200]
  outs = {}
  for mode in ('CPU', 'CUDA', 'CUDA-generic'):
    ds = glt.data.Dataset(edge_dir='in')
    ds.init_graph(edges, graph_mode='CPU' if mode == 'CPU' else 'CUDA', device=0, num_nodes=sizes)
    s = NeighborSampler(ds.graph, [4, 3, 2], seed=9, device=None if mode == 'CPU' else DEV, edge_dir='in')
    if mode == 'CUDA-generic':
      outs[mode] = [s._drive(s._hetero_loop({'paper': seeds.to(DEV)})) for _ in range(2)]
    else:
      outs[mode] = [s.sample_from_nodes(NodeSamplerInput(seeds, 'paper')) for _ in range(2)]
  for it in range(2):
    a = outs['CPU'][it]
    for other in ('CUDA', 'CUDA-generic'):
      b = outs[other][it]
      assert set(a.row.keys()) == set(b.row.keys()), (other, a.row.keys(), b.row.keys())
      for nt in a.node:
        assert set(a.node[nt].tolist()) == set(b.node[nt].cpu().tolist()), (other, nt)
      for et in a.row:
        st, dt = et[0], et[2]
        ea = set(zip(a.node[st][a.row[et]].tolist(), a.node[dt][a.col[et]].tolist()))
        eb = set(zip(b.node[st][b.row[et]].cpu().tolist(), b.node[dt][b.col[et]].cpu().tolist()))
        assert ea == eb, (other, et, len(ea), len(eb))
        assert a.row[et].numel() == b.row[et].numel()
      for nt in a.node:
        assert sum(a.num_sampled_nodes[nt]) == sum(b.num_sampled_nodes[nt]) == a.node[nt].numel()
      assert torch.equal(a.batch['paper'], b.batch['paper'].cpu())
  # hop-contiguity of the arena's local ids: edges of hop h only reference nodes known after hop h
  b = outs['CUDA'][0]
  for et, r in b.row.items():
    st, dt = et[0], et[2]
    ne, off = b.num_sampled_edges[et], 0
    for h, n_e in enumerate(ne):
      if n_e == 0:
        continue
      seg_r, seg_c = r[off:off + n_e], b.col[et][off:off + n_e]
      assert int(seg_c.max()) < sum(b.num_sampled_nodes[dt][:h + 1])       # targets: frontier of hop h
      assert int(seg_r.max()) < sum(b.num_sampled_nodes[st][:h + 2])       # sources: known after hop h
      off += n_e


def test_deterministic_local_id_order(native):
  """deterministic=True: the local ids of every hop's new nodes are assigned in ascending global-id order, so two
  independent samplers with the same seed return IDENTICAL tensors (node order, COO), and every hop's slice of
  `node` is sorted; the sampled structure still equals the CPU sampler's."""
  ei, topo = rmat_csr(20000, 400000, seed=7)
  seeds = torch.randperm(20000)[:700]
  outs = []
  for _ in range(2):
    g = glt.data.Graph(topo, 'CUDA', 0)
    s = NeighborSampler(g, [7, 5, 3], device=DEV, seed=11, deterministic=True)
    outs.append([s.sample_from_nodes(NodeSamplerInput(seeds)) for _ in range(2)])
  for a, b in zip(outs[0], outs[1]):
    assert torch.equal(a.node, b.node) and torch.equal(a.row, b.row) and torch.equal(a.col, b.col)
    off = a.num_sampled_nodes[0]
    for n in a.num_sampled_nodes[1:]:
      seg = a.node[off:off + n]
      assert bool((seg[1:] > seg[:-1]).all())
      off += n
  cpu = NeighborSampler(glt.data.Graph(topo, 'CPU'), [7, 5, 3], seed=11).sample_from_nodes(NodeSamplerInput(seeds))
  a = outs[0][0]
  assert canonical_edges(cpu) == canonical_edges(a)
