import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.loader import NeighborLoader
from graphlearn_for_pytorch_b200.models import DGCNN, HGT, RGNN, GraphSAGE, drnl_node_labeling
from helpers import ring_dataset


def test_graphsage_eager_trains_on_loader_batches():
  torch.manual_seed(0)
  ds = ring_dataset(40, dim=8)
  ds.init_node_labels((torch.arange(40) >= 20).long())
  loader = NeighborLoader(ds, [2, 2], torch.arange(40), batch_size=20, shuffle=True, seed=1)
  model = GraphSAGE(8, 16, 2, num_layers=2)
  opt = torch.optim.Adam(model.parameters(), lr=0.01)
  first = last = None
  for epoch in range(30):
    for b in loader:
      x = b.x / 40.0
      out = model(x, b.edge_index, b.num_sampled_nodes, b.num_sampled_edges)
      assert out.shape[0] == b.batch_size
      loss = torch.nn.functional.cross_entropy(out, b.y[:b.batch_size])
      opt.zero_grad(); loss.backward(); opt.step()
      first = first if first is not None else loss.item()
      last = loss.item()
  assert last < first


def test_trimmed_equals_untrimmed_for_seeds():
  ds = ring_dataset(40, dim=8)
  loader = NeighborLoader(ds, [2, 2], torch.arange(8), batch_size=8)
  b = next(iter(loader))
  model = GraphSAGE(8, 16, 3, num_layers=2).eval()
  full = model(b.x, b.edge_index)[:b.batch_size]
  trimmed = model(b.x, b.edge_index, b.num_sampled_nodes, b.num_sampled_edges)
  assert torch.allclose(full, trimmed, atol=1e-5)


def test_rgnn_variants_on_hetero_batches():
  u2i = torch.tensor([[0, 0, 1, 2, 3, 3], [0, 1, 1, 2, 3, 0]])
  i2i = torch.tensor([[0, 1, 2, 3], [1, 2, 3, 0]])
  ds = glt.data.Dataset(edge_dir='out')
  ds.init_graph({('user', 'u2i', 'item'): u2i, ('item', 'i2i', 'item'): i2i}, graph_mode='CPU')
  ds.init_node_features({'user': torch.randn(4, 8), 'item': torch.randn(4, 8)}, with_gpu=False)
  ds.init_node_labels({'user': torch.tensor([0, 1, 0, 1])})
  loader = NeighborLoader(ds, [2, 2], ('user', torch.arange(4)), batch_size=4)
  b = next(iter(loader))
  etypes = list(b.edge_index_dict.keys())
  for kind in ('rsage', 'rgcn', 'rgat'):
    model = RGNN(etypes, 8, 16, 2, num_layers=2, node_type='user', model=kind)
    out = model(b.x_dict, b.edge_index_dict)
    assert out.shape == (b['user'].node.numel(), 2)
    out.sum().backward()
    out_t = model(b.x_dict, b.edge_index_dict, b.num_sampled_nodes, b.num_sampled_edges)
    assert out_t.shape[1] == 2 and out_t.shape[0] >= b['user'].batch_size
    # bf16 autocast (the --precision bf16 recipe of the IGBH trainers): attention softmax / weighted sums and the
    # degree counts stay in fp32 inside the layers, results agree with the fp32 forward to bf16 accuracy
    model.eval()
    with torch.no_grad():
      ref = model(b.x_dict, b.edge_index_dict)
      with torch.autocast('cpu', dtype=torch.bfloat16):
        low = model(b.x_dict, b.edge_index_dict)
    assert torch.allclose(low.float(), ref, atol=0.1, rtol=0.1), (kind, (low.float() - ref).abs().max())
  hgt = HGT(['user', 'item'], etypes, 8, 16, 2, num_layers=2, heads=2, node_type='user').eval()
  with torch.no_grad():
    ref = hgt(b.x_dict, b.edge_index_dict)
    with torch.autocast('cpu', dtype=torch.bfloat16):
      low = hgt(b.x_dict, b.edge_index_dict)
  assert torch.allclose(low.float(), ref, atol=0.1, rtol=0.1)
  # degree counts beyond bf16's exact-integer range (256): a 600-neighbour mean of bf16 rows still divides by 600
  from graphlearn_for_pytorch_b200.models.rgnn import _segment_mean
  rows = torch.zeros(600, 4, dtype=torch.bfloat16)
  rows[0] = 600.0
  m = _segment_mean(rows, torch.zeros(600, dtype=torch.int64), 1)
  assert m.dtype == torch.bfloat16 and abs(float(m[0, 0]) - 1.0) < 0.02


def test_drnl_and_dgcnn():
  # path 0-1-2-3, link (0, 3)
  ei = torch.tensor([[0, 1, 2], [1, 2, 3]])
  z = drnl_node_labeling(ei, 0, 3, 4)
  assert z[0] == 1 and z[3] == 1 and z[1] == z[2] and z[1] > 1
  model = DGCNN(num_labels=50, hidden=8, num_layers=2, k=10)
  zz = torch.cat([z, z])
  e2 = torch.cat([ei, ei + 4], 1)
  batch = torch.tensor([0, 0, 0, 0, 1, 1, 1, 1])
  out = model(zz, e2, batch, 2)
  assert out.shape == (2,)
  out.sum().backward()


def test_hgt_trains_on_hetero_batches():
  torch.manual_seed(0)
  g = torch.Generator().manual_seed(0)
  u2i = torch.stack([torch.randint(0, 60, (400,), generator=g), torch.randint(0, 40, (400,), generator=g)])
  ds = glt.data.Dataset(edge_dir='out')
  ds.init_graph({('user', 'u2i', 'item'): u2i, ('item', 'rev_u2i', 'user'): u2i.flip(0)}, graph_mode='CPU',
                num_nodes={'user': 60, 'item': 40})
  xu, xi = torch.randn(60, 8, generator=g), torch.randn(40, 12, generator=g)
  ds.init_node_features({'user': xu, 'item': xi}, with_gpu=False)
  ds.init_node_labels({'user': (xu[:, 0] > 0).long()})
  loader = NeighborLoader(ds, [4, 4], ('user', torch.arange(60)), batch_size=30, shuffle=True, seed=0)
  b0 = next(iter(loader))
  model = HGT(['user', 'item'], list(b0.edge_index_dict.keys()), {'user': 8, 'item': 12}, 16, 2, num_layers=2,
              heads=4, node_type='user')
  opt = torch.optim.Adam(model.parameters(), lr=0.02)
  first = last = None
  for epoch in range(25):
    for b in loader:
      out = model(b.x_dict, b.edge_index_dict)[:b['user'].batch_size]
      loss = torch.nn.functional.cross_entropy(out, b['user'].y[:b['user'].batch_size])
      opt.zero_grad(); loss.backward(); opt.step()
      first = first if first is not None else loss.item()
      last = loss.item()
  assert last < 0.7 * first, (first, last)


def test_transposed_gather_backward_equals_scatter_backward():
  """Algorithm behind csrc/cuda/transpose.cu: the backward of the ELL mean aggregation
  computed as an atomics-free GATHER over a transposed adjacency (sources -> targets, hop-ordered segments)
  equals the scatter formulation the engine uses today, for every layer's hop prefix."""
  torch.manual_seed(0)
  cum = [0, 40, 150, 380]                       # local node ids before hop 0 / 1 / 2's new nodes
  k = [5, 4]
  d = 16
  ell, deg = [], torch.zeros(cum[2], dtype=torch.int64)
  for h in range(2):
    rows = cum[h + 1] - cum[h]
    e = torch.randint(-1, cum[h + 2], (rows, k[h]))
    dg = torch.randint(0, k[h] + 1, (rows,))
    ell.append(e); deg[cum[h]:cum[h + 1]] = dg
  # transposed adjacency, hop 0 entries first inside every segment
  n_src = cum[3]
  cnt = torch.zeros(2, n_src, dtype=torch.int64)
  for h in range(2):
    for r in range(cum[h + 1] - cum[h]):
      for j in range(int(deg[cum[h] + r])):
        s = int(ell[h][r, j])
        if s >= 0:
          cnt[h, s] += 1
  upto = cnt.cumsum(0)
  off = torch.cat([torch.zeros(1, dtype=torch.int64), upto[1].cumsum(0)])
  tgt = torch.full((int(off[-1]),), -1)
  cur = torch.zeros(2, n_src, dtype=torch.int64)
  for h in range(2):
    before = upto[h - 1] if h > 0 else torch.zeros(n_src, dtype=torch.int64)
    for r in range(cum[h + 1] - cum[h]):
      for j in range(int(deg[cum[h] + r])):
        s = int(ell[h][r, j])
        if s >= 0:
          tgt[off[s] + before[s] + cur[h, s]] = cum[h] + r
          cur[h, s] += 1
  for nh in (1, 2):                              # layer that aggregates over hops 0..nh-1
    T, S = cum[nh], cum[nh + 1]
    dA = torch.randn(T, 2 * d)                   # gradient of [mean | self]
    # scatter formulation
    dH = torch.zeros(S, d)
    dH[:T] += dA[:, d:]
    for h in range(nh):
      for r in range(cum[h + 1] - cum[h]):
        t = cum[h] + r
        dg = int(deg[t])
        for j in range(dg):
          s = int(ell[h][r, j])
          if s >= 0:
            dH[s] += dA[t, :d] / dg
    # gather formulation
    out = torch.zeros(S, d)
    for s in range(S):
      acc = dA[s, d:].clone() if s < T else torch.zeros(d)
      for e in range(int(upto[nh - 1, s])):
        t = int(tgt[off[s] + e])
        acc += dA[t, :d] / int(deg[t])
      out[s] = acc
    assert torch.allclose(out, dH, atol=1e-5), nh


def test_rel_sage_project_first_is_exact():
  """RelSAGEConv projects before aggregating when in > out (mean is linear): same result as aggregate-first,
  including isolated destination nodes (which must still receive the bias)."""
  from graphlearn_for_pytorch_b200.models.rgnn import RelSAGEConv, _segment_mean
  torch.manual_seed(0)
  conv = RelSAGEConv(64, 16, 8)                       # in_src 64 > out 8 -> project-first path
  x_src, x_dst = torch.randn(50, 64), torch.randn(30, 16)
  ei = torch.stack([torch.randint(0, 50, (200,)), torch.randint(0, 25, (200,))])   # dst 25..29 isolated
  ref = conv.lin_l(_segment_mean(x_src[ei[0]], ei[1], 30)) + conv.lin_r(x_dst)
  assert torch.allclose(conv(x_src, x_dst, ei), ref, atol=1e-5)
  conv2 = RelSAGEConv(8, 16, 32)                      # in < out -> aggregate-first path, same contract
  x2 = torch.randn(50, 8)
  ref2 = conv2.lin_l(_segment_mean(x2[ei[0]], ei[1], 30)) + conv2.lin_r(x_dst)
  assert torch.allclose(conv2(x2, x_dst, ei), ref2, atol=1e-5)


def test_graph_sage_trainer_learns_and_resumes(tmp_path):
  """GraphSageTrainer = the engine's step API on any device: it learns a learnable labelling, evaluates, and a
  restored state_dict continues with the same sampler stream (identical next loss)."""
  from graphlearn_for_pytorch_b200.models import GraphSageTrainer
  from graphlearn_for_pytorch_b200.utils.synthetic import rmat_edges
  torch.manual_seed(1)
  n, d, c = 3000, 16, 5
  ei = rmat_edges(n, 15000, seed=2)
  ei = torch.cat([ei, ei.flip(0)], 1)
  x = torch.randn(n, d)
  y = (x @ torch.randn(d, c)).argmax(1)
  ds = glt.data.Dataset()
  ds.init_graph(ei, graph_mode='CPU', num_nodes=n)
  ds.init_node_features(x, with_gpu=False)

  def make():
    return GraphSageTrainer(ds.graph, ds.node_features, y, in_dim=d, fanouts=[5, 5], hidden=32, num_classes=c,
                            lr=1e-2, seed=3)
  tr = make()
  first = None
  for i in range(40):
    loss = float(tr.train_step(torch.randperm(n)[:256]))
    first = first if first is not None else loss
  ev_loss, correct, cnt = tr.evaluate_batch(torch.arange(512))
  assert loss < 0.8 * first and cnt == 512 and correct / cnt > 1.5 / c
  import copy
  state = copy.deepcopy(tr.state_dict())        # state_dict() returns live references, like nn.Module
  seeds = torch.arange(300, 556)
  expect = float(tr.train_step(seeds))
  tr2 = make()
  tr2.load_state_dict(state)
  assert abs(float(tr2.train_step(seeds)) - expect) < 1e-5
