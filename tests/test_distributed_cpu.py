"""Worker-mode and server-client-mode distributed tests on CPU: 2 spawned processes talking over
localhost RPC (the reference's strategy, test/python/test_dist_neighbor_loader.py:297-594), with
child exit codes asserted."""
import os
import tempfile

import pytest
import torch

from dist_utils import N, build_partition, check_batch, run_workers


def _w_rpc_basics(rank, world, port):
  import graphlearn_for_pytorch_b200.distributed as d
  d.init_worker_group(world, rank)
  d.init_rpc('127.0.0.1', port)
  got = d.all_gather(rank * 10)
  assert sorted(got.values()) == [0, 10]
  d.barrier()
  table = d.rpc_sync_data_partitions(world, rank)
  assert [len(t) for t in table] == [1, 1]

  class Echo(d.RpcCalleeBase):
    def call(self, x):
      return x + rank
  cid = d.rpc_register(Echo())
  other = table[1 - rank][0]
  assert d.rpc_request(other, cid, args=(torch.tensor([5]),)).item() == 5 + (1 - rank)
  d.barrier()
  d.shutdown_rpc()


def test_rpc_basics():
  run_workers(_w_rpc_basics)


def _w_dist_feature(rank, world, port):
  import graphlearn_for_pytorch_b200.distributed as d
  d.init_worker_group(world, rank)
  d.init_rpc('127.0.0.1', port)
  ds = build_partition(rank, world)
  router = d.RpcDataPartitionRouter(d.rpc_sync_data_partitions(world, rank))
  df = d.DistFeature(world, rank, ds.node_features, ds.node_feat_pb, rpc_router=router)
  ids = torch.tensor([0, 1, 2, 3, 39, 38, 7, 7])
  out = df[ids]
  assert torch.equal(out[:, 0].long(), ids)
  d.barrier()
  d.shutdown_rpc()


def test_dist_feature():
  run_workers(_w_dist_feature)


def _w_neighbor_loader(rank, world, port, scheme, mode, edge_dir):
  import graphlearn_for_pytorch_b200.distributed as d
  d.init_worker_group(world, rank)
  ds = build_partition(rank, world, scheme, edge_dir)
  seeds = torch.nonzero(ds.node_pb[torch.arange(N)] == rank).view(-1)
  if mode == 'collocated':
    opts = d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1', master_port=port)
  else:
    opts = d.MpDistSamplingWorkerOptions(num_workers=2, worker_concurrency=2, master_addr='127.0.0.1',
                                         master_port=port, channel_size='16MB')
  loader = d.DistNeighborLoader(ds, [2, 2], seeds, batch_size=5, shuffle=True, with_edge=True, edge_dir=edge_dir,
                                collect_features=True, to_device=torch.device('cpu'), worker_options=opts,
                                random_seed=3)
  for epoch in range(2):
    seen = []
    for b in loader:
      if edge_dir == 'out':
        check_batch(b)
      else:
        assert torch.equal(b.x[:, 0].long(), b.node)
        src, dst = b.node[b.edge_index[0]], b.node[b.edge_index[1]]
        assert torch.all(((dst - src) % N == 1) | ((dst - src) % N == 2))
      assert len(b.num_sampled_nodes) == 3 and b.batch_size == b.batch.numel()
      seen += b.batch.tolist()
    assert sorted(seen) == sorted(seeds.tolist()), (epoch, sorted(seen))
  loader.shutdown()
  if mode == 'collocated':
    d.barrier()
    d.shutdown_rpc()


@pytest.mark.parametrize('scheme,mode,edge_dir', [('hash', 'collocated', 'out'), ('range', 'collocated', 'out'),
                                                  ('hash', 'collocated', 'in'), ('hash', 'mp', 'out')])
def test_dist_neighbor_loader(scheme, mode, edge_dir):
  run_workers(_w_neighbor_loader, args=(scheme, mode, edge_dir), timeout=300)


def _w_link_and_subgraph(rank, world, port):
  import graphlearn_for_pytorch_b200.distributed as d
  from graphlearn_for_pytorch_b200.sampler import NegativeSampling
  d.init_worker_group(world, rank)
  ds = build_partition(rank, world)
  opts = d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1', master_port=port)
  ei = torch.stack(ds.graph.topo.to_coo()[:2])
  loader = d.DistLinkNeighborLoader(ds, [2], batch_size=8, edge_label_index=ei,
                                    neg_sampling=NegativeSampling('binary', 1), collect_features=True,
                                    to_device=torch.device('cpu'), worker_options=opts)
  n_pos = 0
  for b in loader:
    eli, lab = b.edge_label_index, b.edge_label
    pos = lab == 1
    src, dst = b.node[eli[1]], b.node[eli[0]]
    assert torch.all(((dst[pos] - src[pos]) % N == 1) | ((dst[pos] - src[pos]) % N == 2))
    assert torch.equal(b.x[:, 0].long(), b.node)
    n_pos += int(pos.sum())
  assert n_pos == ei.shape[1]
  sub = d.DistSubGraphLoader(ds, torch.arange(rank, N, 8), num_neighbors=[-1], batch_size=2, with_edge=True,
                             collect_features=True, to_device=torch.device('cpu'), worker_options=opts)
  for b in sub:
    nodes = set(b.node.tolist())
    src, dst = b.node[b.edge_index[0]], b.node[b.edge_index[1]]
    got = set(zip(src.tolist(), dst.tolist()))
    want = {(c, a) for a in nodes for c in nodes if (c - a) % N in (1, 2)}       # (neighbour, source), as sampled batches
    assert got == want                                    # induced edges from *both* partitions
    assert torch.equal(b.node[b.mapping], b.batch)
  loader.shutdown(); sub.shutdown()
  d.barrier()
  d.shutdown_rpc()


def test_dist_link_and_subgraph_loaders():
  run_workers(_w_link_and_subgraph, timeout=300)


def _w_server_client(rank, world, port):
  """ranks 0,1 = servers (one partition each); ranks 2,3 = clients."""
  import graphlearn_for_pytorch_b200.distributed as d
  from graphlearn_for_pytorch_b200.typing import Split
  if rank < 2:
    ds = build_partition(rank, 2)
    own = torch.nonzero(ds.node_pb[torch.arange(N)] == rank).view(-1)
    ds.init_node_split((own, own[:2], own[:2]))
    d.init_server(2, rank, ds, '127.0.0.1', port, num_clients=2)
    d.wait_and_shutdown_server()
    return
  crank = rank - 2
  d.init_client(2, 2, crank, '127.0.0.1', port)
  n_parts, _, ntypes, etypes = d.request_server(0, d.DistServer.get_dataset_meta)
  assert n_parts == 2 and ntypes is None
  feat = d.request_server(1, d.DistServer.get_node_feature, None, torch.tensor([1, 3]))
  assert feat[:, 0].tolist() == [1.0, 3.0]
  assert d.request_server(0, d.DistServer.get_node_partition_id, None, torch.tensor([4, 5])).tolist() == [0, 1]
  # the rest of the PyG remote-backend surface (reference test_pyg_remote_backend.py:145-281)
  assert d.request_server(0, d.DistServer.get_node_label, None, torch.tensor([7, 30])).tolist() == [7, 30]
  assert tuple(d.request_server(1, d.DistServer.get_tensor_size, None)) == (N // 2, 8)
  for srv in (0, 1):
    row, col = d.request_server(srv, d.DistServer.get_edge_index, None)
    assert row.numel() == N and torch.all(row % 2 == srv)               # hash partition: edges keyed by source
    assert torch.all(((col - row) % N == 1) | ((col - row) % N == 2))
    rows, cols = d.request_server(srv, d.DistServer.get_edge_size, None)
    assert rows == N and cols == N
  opts = d.RemoteDistSamplingWorkerOptions(server_rank=[0, 1], num_workers=1, worker_concurrency=2,
                                           master_addr='127.0.0.1', master_port=port + 1 + crank,
                                           buffer_size='16MB', prefetch_size=2)
  loader = d.DistNeighborLoader(None, [2, 2], Split.train, batch_size=4, with_edge=True, collect_features=True,
                                to_device=torch.device('cpu'), worker_options=opts)
  for epoch in range(2):
    seen = []
    for b in loader:
      check_batch(b)
      seen += b.batch.tolist()
    assert sorted(seen) == list(range(N)), sorted(seen)
  loader.shutdown()
  d.shutdown_client()


def test_server_client_mode():
  run_workers(_w_server_client, world=4, timeout=400)


def _w_dist_partitioner(rank, world, port, out):
  import graphlearn_for_pytorch_b200.distributed as d
  from graphlearn_for_pytorch_b200.utils.synthetic import id_features, ring_graph
  d.init_worker_group(world, rank)
  d.init_rpc('127.0.0.1', port)
  ei = ring_graph(N)
  half = ei.shape[1] // 2
  sl = slice(rank * half, (rank + 1) * half)
  nsl = slice(rank * N // 2, (rank + 1) * N // 2)
  d.DistRandomPartitioner(out, N, ei[:, sl], torch.arange(ei.shape[1])[sl], id_features(N, 4)[nsl],
                          torch.arange(N)[nsl], id_features(ei.shape[1], 2)[sl],
                          torch.arange(ei.shape[1])[sl], chunk_size=7).partition()   # many small chunks per slice
  d.barrier()
  d.shutdown_rpc()


def test_dist_random_partitioner():
  from graphlearn_for_pytorch_b200.partition import load_partition
  from graphlearn_for_pytorch_b200.utils.synthetic import ring_graph
  with tempfile.TemporaryDirectory() as out:
    run_workers(_w_dist_partitioner, args=(out,))
    ei = ring_graph(N)
    nodes, edges = [], []
    for p in range(2):
      num, idx, g, nf, ef, npb, epb = load_partition(out, p)
      assert torch.all(npb[g.edge_index[0]] == p) and torch.all(epb[g.eids] == p)
      assert torch.equal(ei[0][g.eids], g.edge_index[0]) and torch.equal(ei[1][g.eids], g.edge_index[1])
      assert torch.equal(nf.feats[:, 0].long(), nf.ids) and torch.all(npb[nf.ids] == p)
      assert torch.equal(ef.feats[:, 0].long(), ef.ids) and sorted(ef.ids.tolist()) == sorted(g.eids.tolist())
      nodes += nf.ids.tolist(); edges += g.eids.tolist()
    assert sorted(nodes) == list(range(N)) and sorted(edges) == list(range(ei.shape[1]))


def _w_hetero_loader(rank, world, port, edge_dir):
  import graphlearn_for_pytorch_b200.distributed as d
  from dist_utils import build_hetero_partition
  d.init_worker_group(world, rank)
  ds, edges = build_hetero_partition(rank, world, edge_dir)
  opts = d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1', master_port=port)
  seed_t = 'user' if edge_dir == 'out' else 'item'
  seeds = torch.arange(rank, 20, world)
  loader = d.DistNeighborLoader(ds, [2, 2], (seed_t, seeds), batch_size=4, shuffle=True, with_edge=True,
                                edge_dir=edge_dir, collect_features=True, to_device=torch.device('cpu'),
                                worker_options=opts)
  true_u2i = set(zip(edges[('user', 'u2i', 'item')][0].tolist(), edges[('user', 'u2i', 'item')][1].tolist()))
  true_i2i = set(zip(edges[('item', 'i2i', 'item')][0].tolist(), edges[('item', 'i2i', 'item')][1].tolist()))
  seen = []
  for b in loader:
    assert torch.equal(b['user'].x[:, 0].long(), b['user'].node) if b['user'].x is not None else True
    if b['item'].x is not None:
      assert torch.equal(b['item'].x[:, 0].long() - 1000, b['item'].node)
    for et, ei in b.edge_index_dict.items():
      s_nodes, d_nodes = b[et[0]].node[ei[0]], b[et[2]].node[ei[1]]
      if edge_dir == 'out':   # reversed relations: messages flow neighbour -> seed
        if et == ('item', 'rev_u2i', 'user'):
          assert all((u, i) in true_u2i for i, u in zip(s_nodes.tolist(), d_nodes.tolist()))
        else:
          assert et == ('item', 'i2i', 'item')
          assert all((a, c) in true_i2i for c, a in zip(s_nodes.tolist(), d_nodes.tolist()))
      else:
        truth = true_u2i if et == ('user', 'u2i', 'item') else true_i2i
        assert all((a, c) in truth for a, c in zip(s_nodes.tolist(), d_nodes.tolist()))
    seen += b[seed_t].batch.tolist()
    if seed_t == 'user':
      assert torch.equal(b['user'].y[:b['user'].batch_size], b['user'].batch)
  assert sorted(seen) == seeds.tolist()
  loader.shutdown()
  d.barrier()
  d.shutdown_rpc()


@pytest.mark.parametrize('edge_dir', ['out', 'in'])
def test_dist_hetero_neighbor_loader(edge_dir):
  run_workers(_w_hetero_loader, args=(edge_dir,), timeout=300)


def _w_rpc_sample_matches_single_process(rank, world, port):
  import graphlearn_for_pytorch_b200 as glt
  import graphlearn_for_pytorch_b200.distributed as d
  from dist_utils import build_hetero_partition
  from graphlearn_for_pytorch_b200.sampler import (EdgeSamplerInput, NegativeSampling, NeighborSampler,
                                                    NodeSamplerInput)
  from graphlearn_for_pytorch_b200.typing import as_str
  d.init_worker_group(world, rank)
  d.init_rpc('127.0.0.1', port)
  ds, edges = build_hetero_partition(rank, world, 'out')
  # full neighbourhoods: the sample depends neither on the Philox streams nor on the order of a shard's rows
  s = d.DistNeighborSampler(ds, [-1, -1], with_edge=True, edge_dir='out', seed=5)
  s.start_loop()
  seeds = torch.arange(rank, 20, 3)
  msg = s.sample_from_nodes(NodeSamplerInput(seeds, 'user'))
  whole = glt.data.Dataset(edge_dir='out')
  whole.init_graph(edges, graph_mode='CPU', num_nodes={'user': 20, 'item': 20})
  ref = NeighborSampler(whole.graph, [-1, -1], with_edge=True, seed=5).sample_from_nodes(NodeSamplerInput(seeds, 'user'))
  assert {k[:-len('.ids')] for k in msg if k.endswith('.ids')} == {as_str(nt) for nt in ref.node}
  for nt in ref.node:
    assert set(msg[f'{as_str(nt)}.ids'].tolist()) == set(ref.node[nt].tolist()), nt
    # 'user' only appears at hop 0: no trailing zero hops
    assert msg[f'{as_str(nt)}.num_sampled_nodes'].tolist() == ref.num_sampled_nodes[nt].tolist(), nt
  assert {k[:-len('.rows')] for k in msg if k.endswith('.rows')} == {as_str(et) for et in ref.row}
  for et in ref.row:
    k = as_str(et)
    got = zip(msg[f'{as_str(et[0])}.ids'][msg[f'{k}.rows']].tolist(),
              msg[f'{as_str(et[2])}.ids'][msg[f'{k}.cols']].tolist(), msg[f'{k}.eids'].tolist())
    want = zip(ref.node[et[0]][ref.row[et]].tolist(), ref.node[et[2]][ref.col[et]].tolist(), ref.edge[et].tolist())
    assert set(got) == set(want), et
    assert msg[f'{k}.num_sampled_edges'].tolist() == ref.num_sampled_edges[et].tolist(), et
  # triplet link sampling takes no edge labels, as on one process
  with pytest.raises(AssertionError, match='triplet mode does not take edge labels'):
    s.sample_from_edges(EdgeSamplerInput(torch.tensor([0, 1]), torch.tensor([0, 1]), label=torch.ones(2),
                                         input_type=('user', 'u2i', 'item'),
                                         neg_sampling=NegativeSampling('triplet', 1)))
  s.shutdown_loop()
  d.barrier()
  d.shutdown_rpc()


def test_rpc_hetero_sample_matches_single_process():
  """The rpc data plane returns the sample of a NeighborSampler over the whole graph: the same node and edge sets
  and the same per-hop counts."""
  run_workers(_w_rpc_sample_matches_single_process, timeout=300)


def _w_dist_table(rank, world, port, out):
  import numpy as np
  import graphlearn_for_pytorch_b200.distributed as d
  from graphlearn_for_pytorch_b200.utils.synthetic import ring_graph
  d.init_worker_group(world, rank)
  d.init_rpc('127.0.0.1', port)
  ei = ring_graph(N)
  half = ei.shape[1] // 2
  sl = slice(rank * half, (rank + 1) * half)
  ids = np.arange(rank * N // 2, (rank + 1) * N // 2)
  edges = {'src_id': ei[0, sl].numpy(), 'dst_id': ei[1, sl].numpy()}
  nodes = {'id': ids, 'feature': np.array([f'{i}:{i}' for i in ids], dtype=object), 'label': ids % 3}
  ds = d.DistTableDataset()
  ds.load(N, {None: edges}, {None: nodes}, graph_mode='CPU', output_dir=out)
  assert ds.num_partitions == 2 and ds.partition_idx == rank
  own = torch.nonzero(ds.node_pb == rank).view(-1)
  assert torch.equal(ds.node_features.cpu_get(own)[:, 0].long(), own)
  assert torch.equal(ds.node_labels, torch.arange(N) % 3)
  opts = d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1', master_port=port)
  loader = d.DistNeighborLoader(ds, [2, 2], own, batch_size=6, collect_features=True, to_device=torch.device('cpu'),
                                worker_options=opts)
  for b in loader:
    assert torch.equal(b.x[:, 0].long(), b.node) and torch.equal(b.y, b.node % 3)
    src, dst = b.node[b.edge_index[0]], b.node[b.edge_index[1]]
    assert torch.all(((src - dst) % N == 1) | ((src - dst) % N == 2))
  loader.shutdown()
  d.barrier()
  d.shutdown_rpc()


def test_dist_table_dataset():
  with tempfile.TemporaryDirectory() as out:
    run_workers(_w_dist_table, args=(out,), timeout=300)


def _w_vineyard_fragments(rank, world, port, root):
  """Each worker loads ITS fragment of an Arrow fragment store (the GraphScope / vineyard path of
  the reference: dist_dataset.py:215-243) and runs the RPC neighbor loader over it."""
  import graphlearn_for_pytorch_b200.distributed as d
  d.init_worker_group(world, rank)
  ds = d.DistDataset(edge_dir='out')
  ds.load_vineyard(f'ring_{rank}', root, [('v', 'e', 'v')], node_features={'v': ['feat']}, node_labels={'v': 'label'})
  assert (ds.num_partitions, ds.partition_idx) == (world, rank)
  ds.random_node_split(0.0, 0.0)
  seeds = ds.train_idx
  per = N // world
  assert sorted(seeds.tolist()) == list(range(rank * per, (rank + 1) * per))
  loader = d.DistNeighborLoader(ds, [2, 2], seeds, batch_size=5, shuffle=True, collect_features=True,
                                to_device=torch.device('cpu'), random_seed=5,
                                worker_options=d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1',
                                                                                     master_port=port))
  seen, foreign = [], 0
  for b in loader:
    assert torch.equal(b.x[:, 0].long(), b.node)
    src, dst = b.node[b.edge_index[0]], b.node[b.edge_index[1]]
    assert torch.all(((src - dst) % N == 1) | ((src - dst) % N == 2))
    assert torch.equal(b.y[:b.batch_size], b.batch)     # labels of the (locally owned) seeds
    foreign += int((b.node // per != rank).sum())
    seen += b.batch.tolist()
  assert sorted(seen) == sorted(seeds.tolist())
  assert foreign > 0      # neighbourhoods cross into the other worker's fragment (served over RPC)
  loader.shutdown()
  d.barrier()
  d.shutdown_rpc()


def test_dist_loader_on_vineyard_fragments(tmp_path):
  from graphlearn_for_pytorch_b200.data.vineyard_utils import write_arrow_fragments
  from graphlearn_for_pytorch_b200.utils.synthetic import id_features, ring_graph
  write_arrow_fragments(str(tmp_path), 'ring', 2, {'v': {'feat': id_features(N, 8), 'label': torch.arange(N)}},
                        {'e': ('v', 'v', ring_graph(N), {})})
  run_workers(_w_vineyard_fragments, args=(str(tmp_path),), timeout=300)


def _w_fault_and_replay(rank, world, port):
  """SURVEY 5.3: (a) an exception inside a sampling SUB-PROCESS must reach the consumer as an error (the
  reference only logs it and the epoch hangs); (b) sampling is replayable from (seed, epoch, batch) counters."""
  import graphlearn_for_pytorch_b200.distributed as d
  d.init_worker_group(world, rank)
  ds = build_partition(0, 1)
  bad = torch.tensor([0, 1, 2, 3, 4, 5, 10 ** 6, 7, 8, 9])     # one id far outside the graph / feature table
  opts = d.MpDistSamplingWorkerOptions(num_workers=1, worker_concurrency=1, master_addr='127.0.0.1', master_port=port,
                                       channel_size='8MB')
  loader = d.DistNeighborLoader(ds, [2, 2], bad, batch_size=5, collect_features=True, to_device=torch.device('cpu'),
                                worker_options=opts)
  try:
    for _ in loader:
      pass
    raise AssertionError('the worker failure was swallowed')
  except RuntimeError as e:
    assert 'sampling worker' in str(e) and 'IndexError' in str(e)
  loader.shutdown()

  def epoch_of(seed, port_):
    ld = d.DistNeighborLoader(ds, [2, 2], torch.arange(N), batch_size=8, shuffle=True, collect_features=True,
                              to_device=torch.device('cpu'), random_seed=seed,
                              worker_options=d.CollocatedDistSamplingWorkerOptions(master_addr='127.0.0.1',
                                                                                   master_port=port_))
    out = [(b.batch.tolist(), b.node.tolist(), b.edge_index.tolist()) for b in ld]
    ld.shutdown()
    return out
  a, b, c = epoch_of(11, port + 1), epoch_of(11, port + 1), epoch_of(12, port + 1)
  assert a == b, 'same seed must replay the same batches, nodes and edges'
  assert a != c
  d.shutdown_rpc()


def test_worker_failure_reaches_consumer_and_sampling_replays():
  run_workers(_w_fault_and_replay, world=1, timeout=300)


def _w_server_client_auto(rank, world, port, seed_files, dynamic):
  """2 servers + 2 clients: servers are assigned to clients automatically (client c <- server c), the seeds are
  read BY THE SERVER from a file path (RemoteNodePathSamplerInput); optionally with dynamic RPC membership."""
  import graphlearn_for_pytorch_b200.distributed as d
  from graphlearn_for_pytorch_b200.sampler import RemoteNodePathSamplerInput
  if rank < 2:
    ds = build_partition(rank, 2)
    # dynamic: a non-default server group name, which the clients must discover by rank (they are not told)
    d.init_server(2, rank, ds, '127.0.0.1', port, num_clients=2, is_dynamic=dynamic,
                  server_group_name='custom_named_servers' if dynamic else None)
    d.wait_and_shutdown_server()
    return
  crank = rank - 2
  d.init_client(2, 2, crank, '127.0.0.1', port, is_dynamic=dynamic)
  # one producer per server: the sampling workers of ALL servers form one RPC group (they serve each other's
  # cross-partition hops), so both clients name the same rendezvous port
  opts = d.RemoteDistSamplingWorkerOptions(num_workers=1, worker_concurrency=2, master_addr='127.0.0.1',
                                           master_port=port + 1, buffer_size='16MB', prefetch_size=2)
  assert opts.server_rank in (crank, [crank])                       # assignment by order
  loader = d.DistNeighborLoader(None, [2, 2], RemoteNodePathSamplerInput(seed_files[crank]), batch_size=4,
                                collect_features=True, with_edge=True, to_device=torch.device('cpu'),
                                worker_options=opts)
  expect = sorted(torch.load(seed_files[crank]).tolist())
  for epoch in range(2):
    seen = []
    for b in loader:
      check_batch(b)
      seen += b.batch.tolist()
    assert sorted(seen) == expect
  loader.shutdown()
  d.shutdown_client()


@pytest.mark.parametrize('dynamic', [False, True])
def test_server_client_auto_assignment_and_path_seeds(tmp_path, dynamic):
  files = []
  for c in range(2):
    f = str(tmp_path / f'seeds_{c}.pt')
    torch.save(torch.arange(c, N, 2)[:12], f)
    files.append(f)
  if not dynamic:
    run_workers(_w_server_client_auto, world=4, args=(files, dynamic), timeout=400)
    return
  # torch's dynamic RPC groups (join/leave tokens in the store) stalled once in ~30 local runs of this scenario:
  # bound the wait and retry once instead of letting a rendezvous stall fail the whole suite
  try:
    run_workers(_w_server_client_auto, world=4, args=(files, dynamic), timeout=100)
  except AssertionError:
    run_workers(_w_server_client_auto, world=4, args=(files, dynamic), timeout=200)
