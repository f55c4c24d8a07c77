"""DistNeighborSampler: multi-hop sampling over a partitioned graph.

Parity: reference python/distributed/dist_neighbor_sampler.py:96-807 (async hop loop,
partition scatter / remote one-hop / stitch, link + subgraph sampling, message collation
with labels and features).  Data planes:
  * p2p : the dataset's Graph already spans every rank's shard over NVLink; the whole
          multi-hop sample is the single-process arena sampler (no RPC, no stitch);
  * rpc : seeds are split by the node partition book, remote partitions are sampled by
          their owners through RPC, partial results are stitched back in seed order.
"""
import asyncio
from typing import Dict, List, Optional, Tuple, Union

import torch

from ..channel import ChannelBase, SampleMessage
from ..ops import require_native
from ..sampler import (EdgeSamplerInput, HeteroSamplerOutput, NegativeSampling, NeighborOutput, NeighborSampler,
                       NodeSamplerInput, SamplerOutput, SamplingConfig, SamplingType)
from ..typing import EdgeType, NodeType, as_str, reverse_edge_type
from .dist_dataset import DistDataset
from .dist_feature import DistFeature
from .dist_graph import DistGraph
from .event_loop import ConcurrentEventLoop, wrap_torch_future
from .rpc import (RpcCalleeBase, RpcDataPartitionRouter, rpc_is_initialized, rpc_register, rpc_request_async,
                  rpc_sync_data_partitions)


class RpcSamplingCallee(RpcCalleeBase):
  """Serves one-hop sampling requests for the ids this partition owns."""

  def __init__(self, sampler: NeighborSampler, device: torch.device):
    self.sampler, self.device = sampler, device

  def call(self, ids: torch.Tensor, req_num: int, etype=None, stream: int = 0):
    out = self.sampler.sample_one_hop(ids.to(self.device), req_num, etype, stream=stream)
    return out.nbr.cpu(), out.nbr_num.cpu(), (out.edge.cpu() if out.edge is not None else None)


class RpcSubGraphCallee(RpcCalleeBase):
  """Returns the induced edges among `nodes` that live in this partition (global ids)."""

  def __init__(self, sampler: NeighborSampler, device: torch.device):
    self.sampler, self.device = sampler, device

  def call(self, nodes: torch.Tensor, with_edge: bool):
    node, rows, cols, eids, _ = self.sampler.node_subgraph(nodes.to(self.device))
    return node[rows].cpu(), node[cols].cpu(), (eids.cpu() if eids is not None else None)


def stitch_one_hop(n_seeds: int, parts: List[Tuple[torch.Tensor, NeighborOutput]], device, with_edge: bool):
  """Merge per-partition one-hop results back into seed order (torch ops on `device`;
  the native CPU variant is csrc/cpu/cpu_ops.cc::cpu_stitch)."""
  if device.type == 'cpu':
    nat = require_native()
    idx = [p[0].cpu().contiguous() for p in parts]
    nbr, num, eid = nat.cpu_stitch(n_seeds, idx, [p[1].nbr.cpu().contiguous() for p in parts],
                                   [p[1].nbr_num.cpu().contiguous() for p in parts],
                                   [p[1].edge.cpu().contiguous() for p in parts] if with_edge else [])
    return NeighborOutput(nbr, num, eid if with_edge else None)
  counts = torch.zeros(n_seeds, dtype=torch.int64, device=device)
  for idx, out in parts:
    counts[idx.to(device)] = out.nbr_num.to(device)
  offs = torch.cumsum(counts, 0) - counts
  total = int(counts.sum())
  nbr = torch.empty(total, dtype=torch.int64, device=device)
  eid = torch.empty(total, dtype=torch.int64, device=device) if with_edge else None
  for idx, out in parts:
    num = out.nbr_num.to(device)
    if num.numel() == 0 or int(num.sum()) == 0:
      continue
    start = torch.repeat_interleave(offs[idx.to(device)], num)
    within = torch.arange(int(num.sum()), device=device) - torch.repeat_interleave(torch.cumsum(num, 0) - num, num)
    nbr[start + within] = out.nbr.to(device)
    if with_edge:
      eid[start + within] = out.edge.to(device)
  return NeighborOutput(nbr, counts, eid)


class DistNeighborSampler(ConcurrentEventLoop):
  """Args follow the reference: data, num_neighbors, with_edge, with_neg, with_weight,
  edge_dir, collect_features, channel (None = return results to the caller), use_all2all,
  concurrency, device, seed."""

  def __init__(self, data: DistDataset, num_neighbors=None, with_edge: bool = False, with_neg: bool = False,
               with_weight: bool = False, edge_dir: str = 'out', collect_features: bool = False,
               channel: Optional[ChannelBase] = None, use_all2all: bool = False, concurrency: int = 1,
               device: Optional[torch.device] = None, seed: Optional[int] = None):
    super().__init__(concurrency)
    self.data = data
    self.num_neighbors = num_neighbors
    self.with_edge, self.with_neg, self.with_weight = with_edge, with_neg, with_weight
    self.edge_dir = edge_dir
    self.collect_features = collect_features
    self.channel = channel
    self.use_all2all = use_all2all
    self.data_plane = getattr(data, 'data_plane', 'rpc')
    self.sampler = NeighborSampler(data.graph, num_neighbors, device, with_edge, with_neg, with_weight,
                                   edge_dir=edge_dir, seed=seed)
    self.device = self.sampler.device
    self.data_cls = 'hetero' if isinstance(data.graph, dict) else 'homo'
    self.num_partitions, self.partition_idx = data.num_partitions, data.partition_idx
    self.dist_graph = DistGraph(self.num_partitions, self.partition_idx, data.graph, data.node_pb, data.edge_pb)
    self.rpc_router = None
    self.rpc_sample_callee_id = self.rpc_subgraph_callee_id = None
    self.dist_node_feature = self.dist_edge_feature = None
    remote = self.data_plane == 'rpc' and self.num_partitions > 1
    if remote:
      assert rpc_is_initialized(), 'rpc plane with several partitions needs init_rpc()'
      self.rpc_router = RpcDataPartitionRouter(rpc_sync_data_partitions(self.num_partitions, self.partition_idx))
    if data.node_features is not None and self.data_plane == 'rpc':
      self.dist_node_feature = DistFeature(self.num_partitions, self.partition_idx, data.node_features,
                                           data.node_feat_pb, local_only=not remote,
                                           rpc_router=self.rpc_router, device=self.device)
    if data.edge_features is not None and self.data_plane == 'rpc':
      self.dist_edge_feature = DistFeature(self.num_partitions, self.partition_idx, data.edge_features,
                                           data.edge_feat_pb, local_only=not remote,
                                           rpc_router=self.rpc_router, device=self.device)
    if remote:
      self.rpc_sample_callee_id = rpc_register(RpcSamplingCallee(self.sampler, self.device))
      self.rpc_subgraph_callee_id = rpc_register(RpcSubGraphCallee(self.sampler, self.device))
    self._remote = remote

  # ------------------------------------------------------------------ public entry points
  def sample_from_nodes(self, inputs: NodeSamplerInput) -> Optional[SampleMessage]:
    inputs = NodeSamplerInput.cast(inputs)
    return self._dispatch(self._send_adapter(self._sample_from_nodes, inputs))

  def sample_from_edges(self, inputs: EdgeSamplerInput) -> Optional[SampleMessage]:
    inputs = EdgeSamplerInput.cast(inputs)
    return self._dispatch(self._send_adapter(self._sample_from_edges, inputs))

  def subgraph(self, inputs: NodeSamplerInput) -> Optional[SampleMessage]:
    inputs = NodeSamplerInput.cast(inputs)
    return self._dispatch(self._send_adapter(self._subgraph, inputs))

  def _dispatch(self, coro):
    if self.channel is None:
      return self.run_task(coro)
    self.add_task(coro)
    return None

  async def _send_adapter(self, fn, *args, **kwargs):
    out = await fn(*args, **kwargs)
    msg = await self._colloate_fn(out)
    if self.channel is None:
      return msg
    self.channel.send(msg)
    return None

  # ------------------------------------------------------------------ one hop
  async def _sample_one_hop(self, srcs: torch.Tensor, num_nbr: int, etype: Optional[EdgeType], stream: int
                            ) -> NeighborOutput:
    if not self._remote:
      return self.sampler.sample_one_hop(srcs, num_nbr, etype, stream=stream)
    src_t = None
    if etype is not None:
      src_t = etype[0] if self.edge_dir == 'out' else etype[-1]
    owners = self.dist_graph.get_node_partitions(srcs, src_t).to(srcs.device)
    parts, futs = [], []
    order = [self.partition_idx] + [p for p in range(self.num_partitions) if p != self.partition_idx]
    for p in order:
      idx = torch.nonzero(owners == p, as_tuple=False).view(-1)
      if idx.numel() == 0:
        continue
      ids = srcs[idx]
      if p == self.partition_idx:
        parts.append((idx, self.sampler.sample_one_hop(ids, num_nbr, etype, stream=stream)))
      else:
        to = self.rpc_router.get_to_worker(p)
        f = rpc_request_async(to, self.rpc_sample_callee_id, args=(ids.cpu(), num_nbr, etype, stream))
        futs.append((idx, wrap_torch_future(f)))
    for idx, f in futs:
      nbr, num, eid = await f
      parts.append((idx, NeighborOutput(nbr, num, eid)))
    return stitch_one_hop(srcs.numel(), parts, self.device, self.with_edge)

  # ------------------------------------------------------------------ from nodes
  async def _sample_from_nodes(self, inputs: NodeSamplerInput):
    seeds = inputs.node.to(self.device, dtype=torch.int64)
    if self.data_cls == 'hetero':
      out = await self._hetero_from_seeds({inputs.input_type: seeds})
      out.input_type = inputs.input_type
      return out
    return await self._homo_from_seeds(seeds)

  async def _drive(self, loop):
    """Serve a NeighborSampler hop loop over the partitions: every request of a hop starts at once, then they are
    awaited in order."""
    outs = None
    while True:
      try:
        reqs = loop.send(outs)
      except StopIteration as done:
        return done.value
      tasks = [asyncio.ensure_future(self._sample_one_hop(*r)) for r in reqs]
      outs = [await t for t in tasks]

  async def _homo_from_seeds(self, seeds: torch.Tensor) -> SamplerOutput:
    if not self._remote:
      return self.sampler._sample_from_nodes(seeds)
    return await self._drive(self.sampler._homo_loop(seeds))

  async def _hetero_from_seeds(self, seeds_dict: Dict[NodeType, torch.Tensor]) -> HeteroSamplerOutput:
    if not self._remote:
      return self.sampler._hetero_sample_from_nodes(seeds_dict)
    # global node count of each type the partition book can tell (the local shard cannot)
    totals = {}
    for nt, pb in (self.data.node_pb.items() if isinstance(self.data.node_pb, dict) else ()):
      if isinstance(pb, torch.Tensor):
        totals[nt] = pb.numel()
      elif hasattr(pb, 'partition_bounds'):
        totals[nt] = int(pb.partition_bounds[-1])
      elif hasattr(pb, '_ranges'):
        totals[nt] = int(pb._ranges[-1])
    return await self._drive(self.sampler._hetero_loop(seeds_dict, totals))

  # ------------------------------------------------------------------ from edges
  async def _sample_from_edges(self, inputs: EdgeSamplerInput):
    """Negatives are drawn against the *local* graph view: strict on the p2p plane (the
    view spans every shard), local-partition-only on the rpc plane like the reference
    (dist_neighbor_sampler.py:411-413)."""
    seeds, metadata = self.sampler._link_seeds(inputs)
    if self.data_cls == 'homo':
      out = await self._homo_from_seeds(seeds)
    else:
      out = await self._hetero_from_seeds(seeds)
      out.input_type = inputs.input_type
    out.metadata = metadata
    return out

  # ------------------------------------------------------------------ subgraph
  async def _subgraph(self, inputs: NodeSamplerInput) -> SamplerOutput:
    if self.data_cls != 'homo':
      raise NotImplementedError('distributed subgraph sampling supports homogeneous graphs')
    seeds = inputs.node.to(self.device, dtype=torch.int64)
    if not self._remote:
      out = self.sampler.subgraph(NodeSamplerInput(seeds))
      out.batch = seeds
      return out
    node = torch.unique(await self._drive(self.sampler._subgraph_loop(seeds)))   # ascending ids, like subgraph()
    owners = self.dist_graph.get_node_partitions(node, None)
    futs, rows_g, cols_g, eids_g = [], [], [], []
    for p in range(self.num_partitions):
      if not bool((owners == p).any()):
        continue
      if p == self.partition_idx:
        n2, r2, c2, e2, _ = self.sampler.node_subgraph(node)
        rows_g.append(n2[r2]); cols_g.append(n2[c2])
        if e2 is not None:
          eids_g.append(e2)
      else:
        to = self.rpc_router.get_to_worker(p)
        futs.append(wrap_torch_future(rpc_request_async(to, self.rpc_subgraph_callee_id,
                                                        args=(node.cpu(), self.with_edge))))
    for f in futs:
      r, c, e = await f
      rows_g.append(r.to(self.device)); cols_g.append(c.to(self.device))
      if e is not None:
        eids_g.append(e.to(self.device))
    empty = torch.empty(0, dtype=torch.int64, device=self.device)
    rg = torch.cat(rows_g) if rows_g else empty
    cg = torch.cat(cols_g) if cols_g else empty
    return SamplerOutput(node=node, row=torch.searchsorted(node, rg), col=torch.searchsorted(node, cg),
                         edge=(torch.cat(eids_g) if eids_g else empty) if self.with_edge else None,
                         batch=seeds, device=self.device, metadata=torch.searchsorted(node, seeds))

  # ------------------------------------------------------------------ message collation
  async def _get_node_feats(self, ids: torch.Tensor, ntype=None):
    if self.data_plane == 'p2p':
      feat = self.data.node_features
      feat = feat[ntype] if isinstance(feat, dict) else feat
      return feat[ids] if feat is not None else None
    if self.dist_node_feature is None:
      return None
    if self.use_all2all:
      return self.dist_node_feature.get_all2all(ids, ntype)
    return await wrap_torch_future(self.dist_node_feature.async_get(ids, ntype))

  async def _get_edge_feats(self, eids: torch.Tensor, etype=None):
    if self.dist_edge_feature is None:
      return None
    return await wrap_torch_future(self.dist_edge_feature.async_get(eids, etype))

  async def _colloate_fn(self, output: Union[SamplerOutput, HeteroSamplerOutput]) -> SampleMessage:
    """-> flat Dict[str, Tensor] (wire keys: SURVEY.md Appendix B)."""
    msg: SampleMessage = {}
    is_hetero = isinstance(output, HeteroSamplerOutput)
    msg['#IS_HETERO'] = torch.tensor([int(is_hetero)])
    md = output.metadata
    if isinstance(md, dict):
      for k, v in md.items():
        if v is not None:
          msg[f'#META.{k}'] = v
    elif md is not None:
      msg['#META.mapping'] = md
    labels = self.data.node_labels
    if is_hetero:
      for nt, ids in output.node.items():
        msg[f'{as_str(nt)}.ids'] = ids
        msg[f'{as_str(nt)}.num_sampled_nodes'] = torch.as_tensor(output.num_sampled_nodes.get(nt, []))
        if output.batch is not None and nt in output.batch:
          msg[f'{as_str(nt)}.batch'] = output.batch[nt]
        lab = labels.get(nt) if isinstance(labels, dict) else None
        if lab is not None:
          msg[f'{as_str(nt)}.nlabels'] = lab[ids.to(lab.device)]
        if self.collect_features:
          x = await self._get_node_feats(ids, nt)
          if x is not None:
            msg[f'{as_str(nt)}.nfeats'] = x
      for et, rows in output.row.items():
        k = as_str(et)
        msg[f'{k}.rows'], msg[f'{k}.cols'] = rows, output.col[et]
        msg[f'{k}.num_sampled_edges'] = torch.as_tensor(output.num_sampled_edges.get(et, []))
        if output.edge is not None and et in output.edge:
          msg[f'{k}.eids'] = output.edge[et]
          if self.collect_features:
            orig = reverse_edge_type(et) if self.edge_dir == 'out' else et
            ef = await self._get_edge_feats(output.edge[et], orig)
            if ef is not None:
              msg[f'{k}.efeats'] = ef
      if output.input_type is not None:
        t = output.input_type
        msg['#META.input_type'] = torch.tensor(list(as_str(t).encode()), dtype=torch.uint8)
      return msg
    msg['ids'], msg['rows'], msg['cols'] = output.node, output.row, output.col
    if output.num_sampled_nodes is not None:
      msg['num_sampled_nodes'] = torch.as_tensor(output.num_sampled_nodes)
      msg['num_sampled_edges'] = torch.as_tensor(output.num_sampled_edges)
    if output.batch is not None:
      msg['batch'] = output.batch
    if output.edge is not None:
      msg['eids'] = output.edge
    if isinstance(labels, torch.Tensor):
      msg['nlabels'] = labels[output.node.to(labels.device)]
    if self.collect_features:
      x = await self._get_node_feats(output.node)
      if x is not None:
        msg['nfeats'] = x
      if output.edge is not None:
        ef = await self._get_edge_feats(output.edge)
        if ef is not None:
          msg['efeats'] = ef
    return msg
