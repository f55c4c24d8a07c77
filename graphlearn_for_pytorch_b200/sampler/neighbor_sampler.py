"""NeighborSampler: one-hop / multi-hop / link / subgraph / random-walk sampling on a
single process (CPU or one GPU, possibly reading peer-GPU shards).

API parity: reference python/sampler/neighbor_sampler.py:38-692.  Structural differences:
  * homogeneous multi-hop sampling with positive fanouts runs in a static-shape
    device arena (native SamplerArena): 2 kernels per hop, no host sync until the
    PyG-shaped output is materialised (the reference syncs >= 2x per hop);
  * sampling is without replacement on CPU *and* GPU and both draw from the same
    Philox streams, so (seed, batch counter) fully determines a batch;
  * weighted sampling and random walks exist on the GPU.
"""
import math
import threading
from typing import Dict, List, Optional, Tuple, Union

import torch

from ..data.graph import Graph
from ..ops import require_native
from ..ops.tables import IdTable
from ..typing import EdgeType, NodeType, NumNeighbors, reverse_edge_type
from ..utils.common import count_dict, merge_dict
from .base import (BaseSampler, EdgeIndex, EdgeSamplerInput, HeteroSamplerOutput, NegativeSampling,
                   NeighborOutput, NodeSamplerInput, SamplerOutput)
from .negative_sampler import RandomNegativeSampler

_MAX_ARENA_NODES = 1 << 27


def _count_tensors(counts: dict) -> dict:
  """Per-hop counts of a heterogeneous sample as int64 tensors keyed by type, like the reference
  (neighbor_sampler.py:310-314; they stay on the host: every consumer reads them as Python ints)."""
  out = {}
  for k, v in counts.items():
    t = torch.as_tensor(v, dtype=torch.int64)
    nz = torch.nonzero(t).view(-1)
    # the reference appends a hop's count only while the type still shows up (count_dict): no trailing zero hops
    out[k] = t[:max(int(nz[-1]) + 1 if nz.numel() else 1, 1)]
  return out


class NeighborSampler(BaseSampler):
  """Args:
    graph: `Graph` (homo) or Dict[EdgeType, Graph] (hetero).
    num_neighbors: fanout per hop ([15,10,5]) or per edge type; -1 = all neighbours.
    device: sampling device (defaults to the graph's placement).
    with_edge: also return global edge ids.
    with_neg: create negative samplers for link sampling.
    with_weight: draw neighbours in proportion to the edge weights instead of uniformly.
    strategy: 'random' (only strategy, as in the reference).
    edge_dir: 'out' samples out-neighbours from CSR, 'in' samples in-neighbours from CSC.
    seed: Philox seed; together with the internal batch counter it determines every draw.
    replace: sample with replacement (the reference's CPU behaviour) instead of without.

  What a row of degree d > k draws, on CPU and GPU alike (a row with d <= k returns all its neighbours):
    uniform, no replacement    a uniform k-subset (Floyd);
    uniform, replacement       k independent uniform draws;
    weighted, no replacement   a weighted k-subset: successive draws in proportion to the weights of the neighbours
                               not yet drawn (exponential race); zero-weight neighbours only fill the places that
                               positive weights cannot, in position order;
    weighted, replacement      k independent draws, each neighbour with probability w / sum(w); a row whose weights
                               are all 0 returns no neighbours.
  Without replacement the picks of a row are a set: their order within the row is not random.
  """

  def __init__(self, graph: Union[Graph, Dict[EdgeType, Graph]], num_neighbors: Optional[NumNeighbors] = None,
               device: Optional[torch.device] = None, with_edge: bool = False, with_neg: bool = False,
               with_weight: bool = False, strategy: str = 'random', edge_dir: str = 'out',
               seed: Optional[int] = None, replace: bool = False, deterministic: bool = False):
    self.graph = graph
    # deterministic=True: the GPU arena re-assigns the local ids of every hop's new nodes in ascending global-id
    # order (one device sort per hop), so two runs with the same seed return identical tensors, not just identical
    # sets (default: arrival order of the sampling warps)
    self.deterministic = bool(deterministic)
    self.num_neighbors = num_neighbors
    self.with_edge = with_edge
    self.with_neg = with_neg
    self.with_weight = with_weight
    self.strategy = strategy
    self.edge_dir = edge_dir
    self.replace = replace
    self._nat = require_native()
    self._lock = threading.RLock()
    self._arena = None
    self._arena_key = None
    self._neg_sampler = None
    self._batch = 0
    from ..utils.common import RandomSeedManager
    self.seed = int(seed) if seed is not None else RandomSeedManager.next_seed()

    if isinstance(graph, Graph):
      self._g_cls = 'homo'
      mode = graph.mode
      gdev = graph.device
    else:
      self._g_cls = 'hetero'
      first = next(iter(graph.values()))
      mode, gdev = first.mode, first.device
      self.edge_types = list(graph.keys())
      self._set_num_neighbors_and_num_hops(num_neighbors)
    if mode == 'CPU' or not torch.cuda.is_available():
      self.device = torch.device('cpu')
    elif device is not None and torch.device(device).type == 'cuda':
      d = torch.device(device)
      self.device = torch.device('cuda', d.index if d.index is not None else torch.cuda.current_device())
    else:
      self.device = torch.device('cuda', gdev if gdev is not None else torch.cuda.current_device())
    self.is_cuda = self.device.type == 'cuda'

  # ------------------------------------------------------------------ helpers
  def _set_num_neighbors_and_num_hops(self, num_neighbors):
    if isinstance(num_neighbors, (list, tuple)):
      num_neighbors = {et: list(num_neighbors) for et in self.edge_types}
    self.num_neighbors = num_neighbors
    if num_neighbors is not None:
      hops = {len(v) for v in num_neighbors.values()}
      assert len(hops) == 1, 'every edge type needs the same number of hops'
      self.num_hops = hops.pop()
    else:
      self.num_hops = 0

  @property
  def hops(self) -> int:
    if self._g_cls == 'hetero':
      return self.num_hops
    return len(self.num_neighbors) if self.num_neighbors is not None else 0

  def _graph_of(self, etype: Optional[EdgeType]) -> Graph:
    return self.graph if self._g_cls == 'homo' else self.graph[etype]

  def _next_stream(self, n: int = 8) -> int:
    with self._lock:
      s = (self._batch * 8) & 0x3FFFFFFF
      self._batch += max(1, (n + 7) // 8)
    return s

  def state_dict(self):
    """Checkpointable sampler position (absent in the reference, SURVEY.md 5.4)."""
    return {'seed': self.seed, 'batch': self._batch}

  def load_state_dict(self, state):
    self.seed, self._batch = int(state['seed']), int(state['batch'])

  def lazy_init_sampler(self):
    if self._g_cls == 'homo':
      self.graph.lazy_init()
    else:
      for g in self.graph.values():
        g.lazy_init()

  def lazy_init_neg_sampler(self):
    if self._neg_sampler is None and self.with_neg:
      with self._lock:
        if self._g_cls == 'homo':
          self._neg_sampler = RandomNegativeSampler(self.graph, 'CUDA' if self.is_cuda else 'CPU',
                                                    self.edge_dir, seed=self.seed + 17)
        else:
          self._neg_sampler = {et: RandomNegativeSampler(g, 'CUDA' if self.is_cuda else 'CPU',
                                                         self.edge_dir, seed=self.seed + 17)
                               for et, g in self.graph.items()}

  # accessors the reference exposes next to the lazy initialisers (neighbor_sampler.py:86-90,137-144,629-646)
  def lazy_init_subgraph_op(self):
    """The induced-subgraph operator needs no separate object here: `subgraph()` runs the native count / fill
    kernels (CUDA) or `cpu_node_subgraph` on the graph handle; this only makes sure the graph is placed."""
    self.lazy_init_sampler()

  @property
  def subgraph_op(self):
    self.lazy_init_subgraph_op()
    return self.subgraph

  def create_inducer(self, input_batch_size: int):
    """A fresh id table (global id -> dense local id, first-seen order) sized for a batch of `input_batch_size`
    seeds; one table per node type on heterogeneous graphs."""
    cap = self._max_sampled_nodes(int(input_batch_size))
    if self._g_cls == 'homo':
      return IdTable(self.device, cap)
    ntypes = sorted({et[0] for et in self.graph} | {et[2] for et in self.graph})
    return {nt: IdTable(self.device, cap) for nt in ntypes}

  def get_inducer(self, input_batch_size: int):
    if getattr(self, '_inducer', None) is None:
      self._inducer = self.create_inducer(input_batch_size)
    return self._inducer

  # ------------------------------------------------------------------ one hop
  def sample_one_hop(self, input_seeds: torch.Tensor, req_num: int,
                     etype: Optional[EdgeType] = None, stream: Optional[int] = None) -> NeighborOutput:
    """Sample up to `req_num` neighbours of every seed (-1: all)."""
    g = self._graph_of(etype)
    if stream is None:
      stream = self._next_stream(1)
    seeds = input_seeds.to(self.device, dtype=torch.int64).contiguous()
    if seeds.numel() == 0:
      e = torch.empty(0, dtype=torch.int64, device=self.device)
      return NeighborOutput(e, e.clone(), e.clone() if self.with_edge else None)
    if not self.is_cuda:
      topo = g.topo
      if self.with_weight and topo.edge_weights is not None and req_num >= 0:
        nbr, num, eid = self._nat.cpu_sample_neighbors_weighted(
          topo.indptr, topo.indices, topo.edge_ids, topo.edge_weights, seeds, int(req_num),
          self.with_edge, self.seed, stream, self.replace)
      else:
        nbr, num, eid = self._nat.cpu_sample_neighbors(
          topo.indptr, topo.indices, topo.edge_ids, seeds, int(req_num), self.with_edge,
          self.replace, self.seed, stream)
      return NeighborOutput(nbr, num, eid if self.with_edge else None)
    h = g.graph_handler
    if req_num < 0:
      nbr, num, eid = h.full_neighbors(seeds, self.with_edge)
      return NeighborOutput(nbr, num, eid if self.with_edge else None)
    weighted = bool(self.with_weight and h.has_weights)
    nbr2d, cnt, eid2d = h.sample_one_hop(seeds, int(req_num), self.with_edge, weighted, self.replace,
                                         self.seed, stream)
    mask = nbr2d >= 0
    nbr = nbr2d[mask]
    eid = eid2d[mask] if self.with_edge else None
    return NeighborOutput(nbr, cnt.to(torch.int64), eid)

  # ------------------------------------------------------------------ from nodes
  def sample_from_nodes(self, inputs: NodeSamplerInput, **kwargs):
    inputs = NodeSamplerInput.cast(inputs)
    seeds = inputs.node.to(self.device, dtype=torch.int64)
    self.lazy_init_sampler()
    if self._g_cls == 'hetero':
      assert inputs.input_type is not None, 'hetero sampling needs input_type'
      out = self._hetero_sample_from_nodes({inputs.input_type: seeds})
      out.input_type = inputs.input_type
      return out
    return self._sample_from_nodes(seeds)

  def _arena_ok(self, n_seeds: int) -> bool:
    if not self.is_cuda or self.num_neighbors is None:
      return False
    if any(k <= 0 or k > 512 for k in self.num_neighbors) or len(self.num_neighbors) > 4:
      return False
    worst = n_seeds
    total = n_seeds
    n_nodes = max(self.graph.row_count, self.graph.col_count)
    for k in self.num_neighbors:
      worst = min(worst * k, n_nodes)
      total += worst
    return total < _MAX_ARENA_NODES

  def _get_arena(self, n_seeds: int):
    cap = 1 << max(4, (max(n_seeds, 1) - 1).bit_length())
    key = (cap, tuple(self.num_neighbors), self.with_edge)
    if self._arena is None or self._arena_key != key:
      n_nodes = max(self.graph.row_count, self.graph.col_count)
      self._arena = self._nat.SamplerArena(self.device.index, cap, list(self.num_neighbors),
                                           self.with_edge, int(n_nodes))
      self._arena.deterministic = self.deterministic
      self._arena_key = key
    return self._arena

  def _sample_from_nodes(self, seeds: torch.Tensor) -> SamplerOutput:
    if self._arena_ok(seeds.numel()):
      with self._lock:
        arena = self._get_arena(seeds.numel())
        h = self.graph.graph_handler
        stream = self._next_stream(len(self.num_neighbors))
        weighted = bool(self.with_weight and h.has_weights)
        arena.sample(h, seeds.contiguous(), None, self.seed, stream, weighted, self.replace, False)
        node, nbr_local, tgt_local, eids, nn, ne = arena.to_coo()
      # messages flow neighbour -> seed: row = neighbour, col = target
      while len(nn) > 1 and nn[-1] == 0 and ne[-1] == 0:
        nn.pop(); ne.pop()
      return SamplerOutput(node=node, row=nbr_local, col=tgt_local, edge=eids if self.with_edge else None,
                           batch=node[:nn[0]], num_sampled_nodes=nn, num_sampled_edges=ne,
                           device=self.device)
    return self._drive(self._homo_loop(seeds))

  # ------------------------------------------------------------------ hop loops
  # A hop loop is a generator: it yields the one-hop requests of a hop as a list of (ids, k, etype, stream), is sent
  # back their NeighborOutputs in the same order and finally returns its result.  `_drive` serves the requests here;
  # DistNeighborSampler serves them over the graph's partitions.
  def _drive(self, loop):
    outs = None
    while True:
      try:
        reqs = loop.send(outs)
      except StopIteration as done:
        return done.value
      outs = [self.sample_one_hop(*r) for r in reqs]

  def _homo_loop(self, seeds: torch.Tensor):
    """Hop-by-hop sample of a homogeneous graph (CPU, -1 fanouts, partitioned graphs): one-hop sampler + IdTable."""
    table = IdTable(self.device, self._max_sampled_nodes(seeds.numel()))
    table.init(seeds)
    n0 = table.size()
    frontier = table.keys(0)
    frontier_local = torch.arange(n0, dtype=torch.int64, device=self.device)
    rows, cols, eids = [], [], []
    nn, ne = [n0], []
    stream = self._next_stream(len(self.num_neighbors))
    for h, k in enumerate(self.num_neighbors):
      out, = yield [(frontier, k, None, stream + h)]
      if out.nbr.numel() == 0:
        break
      before = table.size()
      nbr_local = table.insert(out.nbr)
      src_local = torch.repeat_interleave(frontier_local, out.nbr_num)
      rows.append(nbr_local)
      cols.append(src_local)
      if out.edge is not None:
        eids.append(out.edge)
      after = table.size()
      nn.append(after - before)
      ne.append(int(out.nbr.numel()))
      frontier = table.keys(before)
      frontier_local = torch.arange(before, after, dtype=torch.int64, device=self.device)
      if frontier.numel() == 0:
        break
    e = torch.empty(0, dtype=torch.int64, device=self.device)
    node = table.keys(0)
    return SamplerOutput(node=node, row=torch.cat(rows) if rows else e, col=torch.cat(cols) if cols else e.clone(),
                         edge=(torch.cat(eids) if eids else e.clone()) if self.with_edge else None,
                         batch=node[:n0], num_sampled_nodes=nn, num_sampled_edges=ne, device=self.device)

  def _max_sampled_nodes(self, n_seeds: int) -> int:
    n_nodes = max(self.graph.row_count, self.graph.col_count) if self._g_cls == 'homo' else None
    total, cur = n_seeds, n_seeds
    for k in (self.num_neighbors or []):
      if k < 0:
        return (n_nodes or 1 << 24) + n_seeds
      cur = cur * k
      if n_nodes is not None:
        cur = min(cur, n_nodes)
      total += cur
    if n_nodes is not None:
      total = min(total, n_nodes + n_seeds)
    return total

  # ------------------------------------------------------------------ hetero
  def _etype_ends(self, etype: EdgeType) -> Tuple[NodeType, NodeType]:
    """(type we sample *from*, type of the sampled neighbours)."""
    return (etype[0], etype[2]) if self.edge_dir == 'out' else (etype[2], etype[0])

  def _hetero_table_cap(self, n_seeds: int) -> int:
    total, cur = n_seeds, n_seeds
    for h in range(self.num_hops):
      kmax = max(max(v[h], 0) if v[h] >= 0 else 64 for v in self.num_neighbors.values())
      cur = cur * max(kmax, 1) * max(1, len(self.edge_types))
      total += cur
      if total > (1 << 26):
        return 1 << 26
    return total

  def _hetero_type_bound(self, nt: NodeType, n_seeds: int, total_hint: Optional[int] = None) -> Optional[int]:
    """A table of node type `nt` can never hold more distinct ids than the type has nodes: without
    this bound the worst-case fan-out product sizes (and initialises) 2^26-slot tables per type."""
    if total_hint is not None:
      return int(total_hint) + n_seeds
    if not hasattr(self, '_type_bounds'):
      self._type_bounds = {}
    if nt not in self._type_bounds:
      bound = 0
      for et in self.edge_types:
        frm, to = self._etype_ends(et)
        g = self.graph[et]
        if frm == nt:
          bound = max(bound, int(g.row_count))
        if to == nt:
          bound = max(bound, int(g.col_count))
      self._type_bounds[nt] = bound
    return self._type_bounds[nt] + n_seeds if self._type_bounds[nt] > 0 else None

  # ------------------------------------------------------------------ native hetero arena
  def _hetero_arena_ok(self) -> bool:
    if not self.is_cuda or self.num_hops > 4 or self.num_hops < 1:
      return False
    return all(0 <= int(k) <= 512 for v in self.num_neighbors.values() for k in v)

  def _get_hetero_arena(self, seed_counts: Dict[NodeType, int]):
    """Native device-resident hetero sampler + inducer (csrc/bindings.cc HeteroArena): node types and relations
    are integer coded (sorted node types; relations in `self.edge_types` order so the Philox stream ids equal the
    per-relation one-hop path), one grouped launch per hop over all relations, no host sync until to_coo()."""
    ntypes = sorted({t for et in self.edge_types for t in self._etype_ends(et)} | set(seed_counts))
    caps = tuple(1 << max(4, (max(int(seed_counts.get(nt, 0)), 1) - 1).bit_length()) if nt in seed_counts else 0
                 for nt in ntypes)
    limit = getattr(self, '_hetero_cap_limit', 1 << 22)
    key = (caps, limit, self.with_edge)
    if getattr(self, '_harena_key', None) != key:
      tid = {nt: i for i, nt in enumerate(ntypes)}
      graphs, kt, nt_, fan = [], [], [], []
      for et in self.edge_types:
        frm, to = self._etype_ends(et)
        g = self.graph[et]
        g.lazy_init()
        graphs.append(g.graph_handler)
        kt.append(tid[frm]); nt_.append(tid[to])
        fan.append([int(k) for k in self.num_neighbors[et]])
      num_nodes = [int(self._hetero_type_bound(nt, 0) or 0) for nt in ntypes]
      weighted = bool(self.with_weight and all(h.has_weights for h in graphs))
      self._harena = self._nat.HeteroArena(self.device.index, len(ntypes), graphs, kt, nt_, fan, num_nodes,
                                           list(caps), self.with_edge, self.seed, weighted, bool(self.replace),
                                           int(limit), [])
      self._harena_key, self._harena_types, self._harena_overflow = key, ntypes, 0
    return self._harena, self._harena_types

  def _hetero_arena_sample(self, seeds_dict: Dict[NodeType, torch.Tensor]) -> HeteroSamplerOutput:
    arena, ntypes = self._get_hetero_arena({nt: int(v.numel()) for nt, v in seeds_dict.items()})
    tid = {nt: i for i, nt in enumerate(ntypes)}
    stream = self._next_stream(self.num_hops * max(1, len(self.edge_types)))
    arena.step.fill_(int(stream))
    order = [nt for nt in seeds_dict]
    arena.sample([tid[nt] for nt in order], [seeds_dict[nt].contiguous() for nt in order], 0)
    nodes, rows, cols, eids, nn, ne = arena.to_coo()                  # the only host sync of the batch
    ovf = int(arena.counters[arena.overflow_index()].item())
    if ovf > self._harena_overflow:
      import warnings
      warnings.warn(f'hetero sampling arena dropped {ovf - self._harena_overflow} neighbours (frontier capacity '
                    f'{self._hetero_cap_limit if hasattr(self, "_hetero_cap_limit") else 1 << 22} rows); '
                    'doubling the capacity for the following batches')
      self._hetero_cap_limit = 2 * getattr(self, '_hetero_cap_limit', 1 << 22)
    node = {nt: nodes[i] for i, nt in enumerate(ntypes) if nodes[i].numel() > 0}
    num_nodes = {nt: [int(x) for x in nn[i]] for i, nt in enumerate(ntypes) if nodes[i].numel() > 0}
    row, col, edge, num_edges, out_types = {}, {}, {}, {}, []
    for r, et in enumerate(self.edge_types):
      key = reverse_edge_type(et) if self.edge_dir == 'out' else et
      out_types.append(key)
      if rows[r].numel() == 0:
        continue
      row[key], col[key] = rows[r], cols[r]
      if self.with_edge:
        edge[key] = eids[r]
      num_edges[key] = [int(x) for x in ne[r]]
    batch = {nt: node[nt][:num_nodes[nt][0]].clone() for nt in seeds_dict if nt in node}
    return HeteroSamplerOutput(node=node, row=row, col=col, edge=edge if self.with_edge else None, batch=batch,
                               num_sampled_nodes=_count_tensors(num_nodes),
                               num_sampled_edges=_count_tensors(num_edges), edge_types=out_types,
                               device=self.device)

  def _hetero_sample_from_nodes(self, seeds_dict: Dict[NodeType, torch.Tensor]) -> HeteroSamplerOutput:
    if self._hetero_arena_ok():
      return self._hetero_arena_sample({nt: v.to(self.device, dtype=torch.int64) for nt, v in seeds_dict.items()})
    return self._drive(self._hetero_loop(seeds_dict))

  def _hetero_loop(self, seeds_dict: Dict[NodeType, torch.Tensor],
                   type_totals: Optional[Dict[NodeType, int]] = None):
    """Hop-by-hop sample of a heterogeneous graph: per-type IdTables, one request per relation with a frontier.
    `type_totals` (node count of each type, for graphs this process holds only a shard of) bounds the tables in
    place of the local graph sizes; a type it leaves out gets the fan-out bound alone."""
    n_seed_total = sum(v.numel() for v in seeds_dict.values())
    cap = self._hetero_table_cap(n_seed_total)
    tables: Dict[NodeType, IdTable] = {}

    def table_of(nt):
      if nt not in tables:
        if type_totals is None:
          bound = self._hetero_type_bound(nt, n_seed_total)
        else:
          bound = self._hetero_type_bound(nt, n_seed_total, type_totals[nt]) if nt in type_totals else None
        tables[nt] = IdTable(self.device, min(cap, bound) if bound else cap)
      return tables[nt]

    src_dict, src_local = {}, {}
    num_nodes: Dict[NodeType, List[int]] = {}
    num_edges: Dict[EdgeType, List[int]] = {}
    for nt, s in seeds_dict.items():
      t = table_of(nt)
      t.init(s)
      src_dict[nt] = t.keys(0)
      src_local[nt] = torch.arange(t.size(), dtype=torch.int64, device=self.device)
    count_dict(src_dict, num_nodes, 1)
    batch = {nt: v.clone() for nt, v in src_dict.items()}
    rows, cols, eids = {}, {}, {}
    n_et = max(1, len(self.edge_types))
    stream = self._next_stream(self.num_hops * n_et)
    for h in range(self.num_hops):
      before = {nt: t.size() for nt, t in tables.items()}
      reqs = []
      for ei, etype in enumerate(self.edge_types):
        src = src_dict.get(self._etype_ends(etype)[0])
        if src is not None and src.numel() > 0:
          reqs.append((src, self.num_neighbors[etype][h], etype, stream + h * n_et + ei))
      outs = yield reqs
      hop_edges: Dict[EdgeType, torch.Tensor] = {}
      for (_, _, etype, _), out in zip(reqs, outs):
        if out.nbr.numel() == 0:
          continue
        src_t, nbr_t = self._etype_ends(etype)
        nbr_local = table_of(nbr_t).insert(out.nbr)
        s_local = torch.repeat_interleave(src_local[src_t], out.nbr_num)
        key = reverse_edge_type(etype) if self.edge_dir == 'out' else etype
        rows.setdefault(key, []).append(nbr_local)
        cols.setdefault(key, []).append(s_local)
        if out.edge is not None:
          eids.setdefault(key, []).append(out.edge)
        hop_edges[key] = out.nbr
      new_src, new_local = {}, {}
      for nt, t in tables.items():
        b = before.get(nt, 0)
        if t.size() > b:
          new_src[nt] = t.keys(b)
          new_local[nt] = torch.arange(b, t.size(), dtype=torch.int64, device=self.device)
      count_dict(new_src, num_nodes, h + 2)
      count_dict(hop_edges, num_edges, h + 1)
      src_dict, src_local = new_src, new_local
      if not new_src:
        break
    node = {nt: t.keys(0) for nt, t in tables.items()}
    out_types = [reverse_edge_type(et) if self.edge_dir == 'out' else et for et in self.edge_types]
    return HeteroSamplerOutput(
      node=node,
      row={k: torch.cat(v) for k, v in rows.items()},
      col={k: torch.cat(v) for k, v in cols.items()},
      edge={k: torch.cat(v) for k, v in eids.items()} if self.with_edge else None,
      batch=batch, num_sampled_nodes=_count_tensors(num_nodes), num_sampled_edges=_count_tensors(num_edges),
      edge_types=out_types, device=self.device)

  # ------------------------------------------------------------------ from edges
  def sample_from_edges(self, inputs: EdgeSamplerInput, **kwargs):
    """Link sampling with optional binary / triplet negatives (PyG semantics;
    reference neighbor_sampler.py:319-446)."""
    inputs = EdgeSamplerInput.cast(inputs)
    seeds, metadata = self._link_seeds(inputs)
    if self._g_cls == 'homo':
      out = self._sample_from_nodes(seeds)
    else:
      out = self._hetero_sample_from_nodes(seeds)
      out.input_type = inputs.input_type
    out.metadata = metadata
    return out

  def _link_seeds(self, inputs: EdgeSamplerInput):
    """Negatives, seed dedup and metadata of a link batch -> (seeds: a tensor, or a dict by node type on
    heterogeneous graphs, the output's metadata)."""
    src = inputs.row.to(self.device, dtype=torch.int64)
    dst = inputs.col.to(self.device, dtype=torch.int64)
    edge_label = inputs.label.to(self.device) if inputs.label is not None else None
    input_type = inputs.input_type
    neg = inputs.neg_sampling
    num_pos = src.numel()
    self.lazy_init_sampler()
    if neg is not None:
      self.with_neg = True
      self.lazy_init_neg_sampler()
      num_neg = math.ceil(num_pos * neg.amount)
      ns = self._neg_sampler if self._g_cls == 'homo' else self._neg_sampler[input_type]
      if neg.is_binary():
        neg_pair = ns.sample(num_neg, padding=True)
        src = torch.cat([src, neg_pair[0].to(self.device)])
        dst = torch.cat([dst, neg_pair[1].to(self.device)])
        if edge_label is None:
          edge_label = torch.ones(num_pos, device=self.device)
        neg_label = edge_label.new_zeros((neg_pair.shape[1],) + tuple(edge_label.shape[1:]))
        edge_label = torch.cat([edge_label, neg_label])
      else:
        assert num_neg % max(num_pos, 1) == 0
        neg_pair = ns.sample(num_neg, padding=True)
        dst = torch.cat([dst, neg_pair[1].to(self.device)])
        assert edge_label is None, 'triplet mode does not take edge labels'

    if self._g_cls == 'homo' or input_type[0] == input_type[-1]:
      seed, inverse = torch.unique(torch.cat([src, dst]), return_inverse=True)
      seeds = seed if self._g_cls == 'homo' else {input_type[0]: seed}
      inv_src, inv_dst = inverse[:src.numel()], inverse[src.numel():]
    else:
      s_seed, inv_src = torch.unique(src, return_inverse=True)
      d_seed, inv_dst = torch.unique(dst, return_inverse=True)
      seeds = {input_type[0]: s_seed, input_type[-1]: d_seed}
    if neg is None or neg.is_binary():
      return seeds, {'edge_label_index': torch.stack([inv_src, inv_dst]), 'edge_label': edge_label}
    return seeds, {'src_index': inv_src[:num_pos], 'dst_pos_index': inv_dst[:num_pos],
                   'dst_neg_index': inv_dst[num_pos:].view(num_pos, -1)}

  # ------------------------------------------------------------------ PyG v1
  def sample_pyg_v1(self, ids: torch.Tensor):
    """(batch_size, n_id, adjs) of the legacy PyG NeighborSampler: one bipartite
    EdgeIndex per hop, outermost hop first (reference :448-472)."""
    out = self._sample_from_nodes(ids.to(self.device, dtype=torch.int64))
    nn, ne = out.num_sampled_nodes, out.num_sampled_edges
    adjs, e0, n_src = [], 0, nn[0]
    for h in range(len(ne)):
      n_dst = n_src
      n_src = n_dst + nn[h + 1]
      e1 = e0 + ne[h]
      # layer h uses every edge sampled up to hop h (targets are the first n_dst nodes)
      ei = torch.stack([out.row[:e1], out.col[:e1]])
      eid = out.edge[:e1] if out.edge is not None else None
      adjs.append(EdgeIndex(ei, eid, (n_src, n_dst)))
      e0 = e1
    return nn[0], out.node, adjs[::-1]

  # ------------------------------------------------------------------ subgraph
  def subgraph(self, inputs: NodeSamplerInput) -> SamplerOutput:
    """Induced subgraph on the seeds plus (optionally) their k-hop neighbourhoods;
    metadata['mapping'] gives node[mapping] == inputs (reference :474-498)."""
    inputs = NodeSamplerInput.cast(inputs)
    seeds = inputs.node.to(self.device, dtype=torch.int64)
    assert self._g_cls == 'homo', 'subgraph sampling supports homogeneous graphs'
    self.lazy_init_sampler()
    all_nodes = self._drive(self._subgraph_loop(seeds))
    node, rows, cols, eids, mapping = self.node_subgraph(all_nodes, seeds.numel())
    return SamplerOutput(node=node, row=rows, col=cols, edge=eids if self.with_edge else None,
                         device=self.device, metadata=mapping)

  def _subgraph_loop(self, seeds: torch.Tensor):
    """k-hop node expansion of a subgraph sample, as a hop loop: returns the seeds followed by the unique
    neighbours of every hop."""
    nodes = [seeds]
    if self.num_neighbors is not None:
      frontier = torch.unique(seeds)
      stream = self._next_stream(len(self.num_neighbors))
      for h, k in enumerate(self.num_neighbors):
        out, = yield [(frontier, k, None, stream + h)]
        if out.nbr.numel() == 0:
          break
        frontier = torch.unique(out.nbr)
        nodes.append(frontier)
    return torch.cat(nodes)

  def node_subgraph(self, all_nodes: torch.Tensor, num_seeds: int = 0):
    """Induced subgraph on exactly `all_nodes` (no neighbourhood expansion).
    -> (unique nodes in ASCENDING id order, rows, cols, eids, local ids of the first `num_seeds` inputs).

    Conventions of the reference (neighbor_sampler.py:474-498, test/python/test_subgraph.py): the node list is the
    sorted unique id set; edges come out ordered by (source-side row, position in the row); and the edge index is
    REVERSED with respect to the stored adjacency -- `row` holds the adjacency's column side, `col` its row side --
    the same message-flow orientation `sample_from_nodes` uses."""
    all_nodes = all_nodes.to(self.device, dtype=torch.int64).contiguous()
    self.lazy_init_sampler()
    uniq = torch.unique(all_nodes)                       # sorted
    if self.is_cuda:
      table = IdTable(self.device, uniq.numel())
      table.init(uniq)                                   # ordered insert: local id == rank in `uniq`
      n = table.size()
      rows, cols, eids = table.native.subgraph(self.graph.graph_handler, n, self.with_edge)
      node = table.keys(0)
    else:
      topo = self.graph.topo
      node, rows, cols, eids = self._nat.cpu_node_subgraph(topo.indptr, topo.indices, topo.edge_ids,
                                                           uniq, self.with_edge)
    mapping = torch.searchsorted(node, all_nodes[:num_seeds].contiguous())
    return node, cols, rows, (eids if self.with_edge else None), mapping

  # ------------------------------------------------------------------ random walk
  def random_walk(self, starts: torch.Tensor, walk_length: int, p: float = 1.0, q: float = 1.0,
                  etype: Optional[EdgeType] = None) -> torch.Tensor:
    """[n, walk_length + 1] node ids; uniform (p=q=1) or node2vec-biased walks.
    New functionality: the reference only declares SamplingType.RANDOM_WALK.

    A step of a biased walk weighs the previous node 1/p, its neighbours 1 and every other node 1/q, and samples
    by rejection: p and q must be finite and > 0 with max(1, 1/p, 1/q) / min(1, 1/p, 1/q) <= 64."""
    p, q, walk_length = float(p), float(q), int(walk_length)
    if walk_length < 0:
      raise ValueError(f'random_walk: walk_length must be >= 0, got {walk_length}')
    if not (math.isfinite(p) and math.isfinite(q) and p > 0 and q > 0):
      raise ValueError(f'random_walk: p and q must be finite and > 0, got p={p}, q={q}')
    w = (1.0, 1.0 / p, 1.0 / q)
    if max(w) / min(w) > 64.0:
      raise ValueError(f'random_walk: max(1, 1/p, 1/q) / min(1, 1/p, 1/q) must be <= 64, got p={p}, q={q}')
    g = self._graph_of(etype)
    self.lazy_init_sampler()
    starts = starts.to(self.device, dtype=torch.int64).contiguous()
    stream = self._next_stream(1)
    if self.is_cuda:
      return g.graph_handler.random_walk(starts, int(walk_length), float(p), float(q), self.seed, stream)
    topo = g.topo
    return self._nat.cpu_random_walk(topo.indptr, topo.indices, starts, int(walk_length), float(p),
                                     float(q), self.seed, stream)

  # ------------------------------------------------------------------ hotness
  def sample_prob(self, inputs: NodeSamplerInput, node_cnt):
    """Probability of each node being touched when sampling from `inputs`
    (drives FrequencyPartitioner / cache admission; reference :500-627)."""
    inputs = NodeSamplerInput.cast(inputs)
    self.lazy_init_sampler()
    seeds = inputs.node.to(self.device, dtype=torch.int64)
    if self._g_cls == 'hetero':
      return self._hetero_sample_prob({inputs.input_type: seeds}, node_cnt)
    last = torch.full((int(node_cnt),), 0.01, dtype=torch.float32, device=self.device)
    last[seeds] = 1.0
    for k in self.num_neighbors:
      last = self._nbr_prob(self.graph, self.graph, last, last, k)
    return last

  def _nbr_prob(self, g: Graph, nbr_g: Graph, last, nbr_last, k):
    if self.is_cuda:
      return g.graph_handler.nbr_prob(nbr_g.graph_handler, last.contiguous(), nbr_last.contiguous(), int(k))
    return self._nat.cpu_nbr_prob(g.topo.indptr, g.topo.indices, nbr_g.topo.indptr, last.contiguous(),
                                  nbr_last.contiguous(), int(k))

  def _hetero_sample_prob(self, seeds_dict, node_cnt: Dict[NodeType, int]):
    """Per-type hotness.  For hop h, a node v of type A gets, through every relation
    whose CSR rows are of type A, the chance that one of its row-neighbours (type B)
    was hot in the previous hop and picked v; contributions of different relations
    are combined as independent events (1 - prod(1 - p))."""
    def _cnt(v):
      return int(v.size(0)) if isinstance(v, torch.Tensor) else int(v)
    probs = {nt: torch.full((_cnt(c),), 0.005, dtype=torch.float32, device=self.device)
             for nt, c in node_cnt.items()}
    for nt, s in seeds_dict.items():
      probs[nt][s] = 1.0
    for h in range(self.num_hops):
      nxt = {nt: [] for nt in probs}
      for etype in self.edge_types:
        row_t, col_t = (etype[0], etype[2]) if self.edge_dir == 'out' else (etype[2], etype[0])
        if row_t not in probs or col_t not in probs:
          continue
        # the relation whose rows are of type col_t and point back at row_t gives deg(u)
        back = None
        for other in self.edge_types:
          o_row, o_col = (other[0], other[2]) if self.edge_dir == 'out' else (other[2], other[0])
          if o_row == col_t and o_col == row_t:
            back = other
            break
        if back is None:
          continue
        k = self.num_neighbors[back][h]
        cur = self._nbr_prob(self.graph[etype], self.graph[back], probs[row_t], probs[col_t], k)
        nxt[row_t].append(cur)
      for nt, lst in nxt.items():
        if lst:
          acc = torch.ones_like(probs[nt])
          for c in lst:
            acc = acc * (1 - c[:acc.numel()])
          probs[nt] = torch.maximum(probs[nt], 1 - acc)
    return probs
