"""`HeteroSageEngine`: device-resident relational GraphSAGE (R-SAGE) training step for heterogeneous graphs.

The reference trains IGBH with a PyG `HeteroConv({etype: SAGEConv})` fed by its hetero `NeighborLoader`
(examples/igbh/rgnn.py:22-81, examples/igbh/train_rgnn_multi_gpu.py:80-142): per hop and per edge type a sampling
call, a D2H size read, an inducer call, then per-relation scatter/linear autograd ops.  Here the whole step is a
fixed launch sequence over static buffers, captured into ONE CUDA graph:

  sample   native `HeteroArena`: one grouped launch per hop over all relations, per-type id tables, no host sync
  layer l  for every destination type t that can hold targets at this depth:
             A_t = [ mean_{r -> t} x_src(r)  ...  | x_t ]   one ELL aggregation kernel per incoming relation,
                                                           writing its column block (layer 1 reads the feature
                                                           tables -- local or peer HBM -- in place)
             Z_t = act(A_t . W_t^T + b_t)                  TMA-fed wgmma GEMM, rows from the device counter
  loss     fused log-softmax / NLL on the seed type (labels looked up through the batch's node list)
  backward per (layer, type): dW (split-K, fp32 red-add) + dA in one wgmma launch, then per relation the ELL
           scatter of its dA column block into the source type's fp32 gradient rows, ReLU mask + bf16 cast
  update   fused flat Adam (fp32 master weights, bf16 shadow copy)

`W_t = [W_r1 | W_r2 | ... | W_self]` concatenates the relation weights of a destination type, so summing the
per-relation SAGEConv outputs (HeteroConv aggr='sum') is a single GEMM.  Activation is ReLU (the reference example
uses leaky_relu + dropout; see docs).  Node types are integer coded in sorted order, relations in the order of
`graphs`.
"""
import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch

from ..data.quantize import mxfp8_row_bytes
from ..ops import require_native
from .sage import infer_chunk_rows, infer_chunks, infer_gemm

EdgeType = Tuple[str, str, str]


def _round_up(x, m):
  return (x + m - 1) // m * m


def resolve_feature_formats(feature_format, dim_in: Dict[str, int], feature_tables: Dict[str, object]) -> Dict[str, str]:
  """{node type: 'bf16' | 'mxfp8'} from the engines' `feature_format` argument (one format for every type, or a dict
  whose missing types are bf16), checked against each type's width and table: an MXFP8 type needs a width that is a
  multiple of 32 and a uint8 table of `mxfp8_row_bytes(width)`-byte rows (`data.quantize_mxfp8`); a bf16 type must not
  be handed a uint8 table.  Raises ValueError."""
  fmt = {}
  for t, d in dim_in.items():
    f = feature_format.get(t, 'bf16') if isinstance(feature_format, dict) else feature_format
    if f not in ('bf16', 'mxfp8'):
      raise ValueError(f"feature_format of node type {t!r} must be 'bf16' or 'mxfp8' (got {f!r})")
    tbl = feature_tables[t]
    if f == 'mxfp8':
      if d % 32 != 0:
        raise ValueError(f'MXFP8 features of node type {t!r}: in_dim must be a multiple of 32 (got {d})')
      if not tbl.is_uint8 or tbl.width != mxfp8_row_bytes(d):
        raise ValueError(f'MXFP8 features of node type {t!r}: the table must hold uint8 rows of '
                         f'mxfp8_row_bytes({d}) = {mxfp8_row_bytes(d)} bytes (data.quantize_mxfp8)')
    elif tbl.is_uint8:
      raise ValueError(f"node type {t!r} has a uint8 feature table but feature_format 'bf16'; pass "
                       f"feature_format='mxfp8' (or a dict naming this type) for data.quantize_mxfp8 rows")
    fmt[t] = f
  return fmt


class HeteroSageEngine(object):
  """Args:
    graphs: {(src, rel, dst): data.Graph} device graphs (single- or multi-shard), CSC by dst for edge_dir='in',
      CSR by src for edge_dir='out'.
    feature_tables: {node type: native RowTableHandle of rows indexed by global id} (`UnifiedTensor._table()`,
      `PartitionedFeature.table`): bf16 rows, or `data.quantize_mxfp8` rows for the types `feature_format` names.
    feature_format: 'bf16', 'mxfp8', or {node type: format} (types left out are bf16; small tables rarely justify
      quantising).  MXFP8 rows are de-quantised inside the layer-1 aggregation, the gathers and the inference
      aggregation; every buffer downstream is bf16 as before.  An MXFP8 type needs an in_dim that is a multiple of 32.
    labels: int64 [num_nodes[seed_type]].
    in_dim: feature width (int or {type: int}), a multiple of 8 up to 1024.  The layer-1 operand of each destination
      type (its incoming relations' source widths plus its own) must be a multiple of 64 wide.
    num_nodes: {type: node count}.
    hidden: a multiple of 64 up to 1024.

  Widths outside these limits raise ValueError at construction.
    fanouts: [k per hop] (all relations) or {etype: [k per hop]}.

  Parameters are named ('W', l, t) and ('b', l, t) per layer and destination type; `param(name, grad=False)`.
  """

  def __init__(self, graphs: Dict[EdgeType, object], feature_tables: Dict[str, object], labels: torch.Tensor,
               in_dim: Union[int, Dict[str, int]], num_nodes: Dict[str, int], seed_type: str,
               fanouts: Union[Sequence[int], Dict[EdgeType, Sequence[int]]] = (15, 10, 5), batch_size: int = 1024,
               hidden: int = 512, num_classes: int = 19, edge_dir: str = 'in', lr: float = 1e-3,
               weight_decay: float = 0.0, seed: int = 0, device: Optional[torch.device] = None,
               use_cuda_graph: bool = True, cap_limit: int = 1 << 21, group=None,
               feature_format: Union[str, Dict[str, str]] = 'bf16'):
    self.nat = require_native()
    self.edge_types = [tuple(e) for e in graphs]
    self.graphs = graphs
    self.edge_dir = edge_dir
    first = next(iter(graphs.values()))
    first.lazy_init()
    self.device = torch.device(device) if device is not None else torch.device('cuda', first.device)
    dev = self.device
    self.seed_type = seed_type
    self.bs = int(batch_size)
    self.hidden, self.C = int(hidden), int(num_classes)
    self.n_out_pad = _round_up(self.C, 64)
    self.lr, self.wd, self.seed = lr, weight_decay, int(seed)
    self.use_cuda_graph = use_cuda_graph
    import torch.distributed as dist
    self.group = group
    self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
    self.peer_group = None
    # ---- integer-coded schema -------------------------------------------------------------------------
    ends = [(et[0], et[2]) if edge_dir == 'out' else (et[2], et[0]) for et in self.edge_types]   # (key, nbr)
    self.ntypes = sorted({t for e in ends for t in e} | {seed_type})
    self.tid = {t: i for i, t in enumerate(self.ntypes)}
    self.kt = [self.tid[k] for k, _ in ends]          # type a relation is sampled FROM (its messages' destination)
    self.nt = [self.tid[n] for _, n in ends]          # neighbour type (message source)
    if isinstance(fanouts, dict):
      self.fan = [[int(k) for k in fanouts[et]] for et in self.edge_types]
    else:
      self.fan = [[int(k) for k in fanouts] for _ in self.edge_types]
    self.L = len(self.fan[0])
    assert 1 <= self.L <= 4 and all(len(f) == self.L for f in self.fan)
    NT, NR = len(self.ntypes), len(self.edge_types)
    self.dim_in = {t: int(in_dim[t] if isinstance(in_dim, dict) else in_dim) for t in self.ntypes}
    # the aggregation / scatter kernels cover rows of up to 1024 columns; the wgmma GEMMs need 64-column multiples
    for t, d in self.dim_in.items():
      if d % 8 != 0 or not 8 <= d <= 1024:
        raise ValueError(f'in_dim of node type {t!r} must be a multiple of 8 in [8, 1024] (got {d})')
    if self.hidden % 64 != 0 or not 64 <= self.hidden <= 1024:
      raise ValueError(f'hidden must be a multiple of 64 in [64, 1024] (got {self.hidden})')
    if self.C < 1:
      raise ValueError(f'num_classes must be >= 1 (got {self.C})')
    self.feat = feature_tables
    self.feature_format = resolve_feature_formats(feature_format, self.dim_in, feature_tables)
    self.labels = labels.to(dev)
    # types that can appear at hop h (static reachability over the schema)
    hop_types = [{self.tid[seed_type]}]
    for h in range(self.L):
      hop_types.append({self.nt[r] for r in range(NR) if self.kt[r] in hop_types[h] and self.fan[r][h] > 0})
    self.hop_types = hop_types
    # layer l (1-based) has targets of the types reachable within hops 0..L-l
    self.targets = [None] + [sorted(set().union(*hop_types[:self.L - l + 1])) for l in range(1, self.L + 1)]
    with torch.cuda.device(dev):
      handles = []
      for et in self.edge_types:
        graphs[et].lazy_init()
        handles.append(graphs[et].graph_handler)
      nn_list = [int(num_nodes[t]) for t in self.ntypes]
      self._n_nodes = nn_list
      max_seeds = [self.bs if t == seed_type else 0 for t in self.ntypes]
      self.arena = self.nat.HeteroArena(dev.index, NT, handles, self.kt, self.nt, self.fan, nn_list, max_seeds,
                                        False, self.seed, False, False, int(cap_limit), [])
      self.cap_rows = [list(v) for v in self.arena.cap_rows]
      self.cap_nodes = list(self.arena.cap_nodes)
      self._ctr = [self.arena.counters[t * 8:t * 8 + 8] for t in range(NT)]       # per-type hop counters (views)
      self._ovf_idx = self.arena.overflow_index()
      # relations feeding type t at layer l: every relation sampled from t with a positive fan-out in a used hop
      self.in_rel = [None]
      for l in range(1, self.L + 1):
        nh = self.L - l + 1
        # (a relation only counts for the hops at which its key type can actually be in the frontier)
        self.in_rel.append({t: [r for r in range(NR) if self.kt[r] == t and
                                any(self.fan[r][h] > 0 and t in hop_types[h] for h in range(nh))]
                            for t in self.targets[l]})
      self._alloc()
      self._init_params()
      self._seeds = torch.zeros(self.bs, dtype=torch.int64, device=dev)
      self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
      self.correct = torch.zeros(1, dtype=torch.int32, device=dev)
      self.step_dev = torch.zeros(2, dtype=torch.int32, device=dev)
    self._plans = {}
    self._graph = None
    self.step_idx = 0
    self.kernels_per_step = 0

  # ------------------------------------------------------------------ buffers / parameters
  def _rows(self, l: int, t: int) -> int:
    """Rows of type t's layer-l buffers (l = 0: the input layer, every sampled node)."""
    return max(int(min(self.cap_nodes[t], sum(self.cap_rows[t][:self.L - l + 1]))), 128)

  def _width_in(self, l: int, t: int) -> int:
    return self.dim_in[self.ntypes[t]] if l == 1 else self.hidden

  def _zeros(self, *shape, dt=torch.bfloat16) -> torch.Tensor:
    return torch.zeros(*shape, dtype=dt, device=self.device)

  @staticmethod
  def _check_heads(heads: int, hidden: int) -> int:
    """The attention engines' head count, which must split hidden into head widths that are multiples of 8."""
    heads = int(heads)
    if heads < 1 or int(hidden) % heads != 0 or (int(hidden) // heads) % 8 != 0:
      raise ValueError(f'heads must divide hidden into head widths that are multiples of 8 (hidden {hidden}, '
                       f'heads {heads})')
    return heads

  def _check_attention_schema(self):
    """The attention engines take in_dim multiples of 64 in [64, 1024] and need an incoming relation into every
    destination type at every layer."""
    for t, d in self.dim_in.items():
      if d % 64 != 0 or not 64 <= d <= 1024:
        raise ValueError(f'in_dim of node type {t!r} must be a multiple of 64 in [64, 1024] (got {d})')
    for l in range(1, self.L + 1):
      for t in self.targets[l]:
        if not self.in_rel[l][t]:
          raise ValueError(f'node type {self.ntypes[t]!r} has no incoming relation at layer {l}')

  def _alloc_head(self):
    """Output and gradient of the attention engines' Linear head on the seed type."""
    rows = self._rows(self.L, self.tid[self.seed_type])
    self.logits = self._zeros(rows, self.n_out_pad)
    self.dlogits = self._zeros(rows, self.n_out_pad)

  def _alloc(self):
    z, f32 = self._zeros, torch.float32
    self.A, self.Z, self.dPre, self.dA, self.dH, self.col = [None], [None], [None], [None], [None], [None]
    for l in range(1, self.L + 1):
      n_out = self.hidden if l < self.L else self.n_out_pad
      A, Z, dP, dA, dH, col = {}, {}, {}, {}, {}, {}
      for t in self.targets[l]:
        cap = self._rows(l, t)
        offs, c = [], 0
        for r in self.in_rel[l][t]:
          offs.append(c)
          c += self._width_in(l, self.nt[r])
        col[t] = (offs, c)                       # mean-block offsets, self-block offset
        K = c + self._width_in(l, t)
        if K % 64 != 0:                          # weight-gradient GEMM: N = K
          raise ValueError(f'layer {l} operand of node type {self.ntypes[t]!r} is {K} columns wide (the widths of its '
                           f'incoming relations\' source types plus its own); it must be a multiple of 64')
        A[t] = z(cap, K)
        Z[t] = z(cap, n_out)
        dP[t] = z(cap, n_out)
        if l > 1:
          dA[t] = z(cap, K)
        if l < self.L:
          dH[t] = z(cap, n_out, dt=f32)         # gradient wrt Z[l][t], filled by layer l+1
      self.A.append(A); self.Z.append(Z); self.dPre.append(dP); self.dA.append(dA); self.dH.append(dH)
      self.col.append(col)

  def _param_layout(self):
    """(name, shape) of every parameter in layout and initialisation order: ('W', l, t) [n_out, K] and ('b', l, t)
    [n_out] per layer and destination type."""
    for l in range(1, self.L + 1):
      for t in self.targets[l]:
        yield ('W', l, t), (self.Z[l][t].shape[1], self.A[l][t].shape[1])
        yield ('b', l, t), (self.Z[l][t].shape[1],)

  def _param_init(self, name, shape, g: torch.Generator) -> torch.Tensor:
    """Initial fp32 value of a parameter (weights drawn from g; zero biases and zero padding class rows)."""
    kind, l, t = name
    if kind == 'b':
      return torch.zeros(shape)
    w = (torch.rand(*shape, generator=g) * 2 - 1) / math.sqrt(max(shape[1] // (len(self.in_rel[l][t]) + 1), 1))
    if l == self.L:
      w[self.C:] = 0
    return w

  def _init_params(self):
    """Flat fp32 parameters `p32`, laid out by `_param_layout()`: `param_index[name] = (offset, shape)`, every
    parameter starting at a multiple of 8 floats (16-byte aligned bf16 shadow).  Checkpoints, the peer all-reduce and
    Adam rely on this layout.  Initial values are drawn in layout order from one generator seeded with `seed`.  Then the
    bf16 shadow, gradient and Adam buffers (and the peer group when world > 1)."""
    dev = self.device
    self.param_index, off = {}, 0
    for name, shape in self._param_layout():
      off = _round_up(off, 8)
      self.param_index[name] = (off, shape)
      off += math.prod(shape)
    self.p32 = torch.zeros(_round_up(off, 8), dtype=torch.float32, device=dev)
    g = torch.Generator(device='cpu')
    g.manual_seed(self.seed)
    for name, (o, shape) in self.param_index.items():
      self.p32[o:o + math.prod(shape)].copy_(self._param_init(name, shape, g).flatten())
    pad = (-self.p32.numel()) % 4
    self.p16 = self.p32.to(torch.bfloat16)
    self.g32 = torch.zeros_like(self.p32)
    if self.world > 1:
      # data parallel over the GPUs of the box: the gradient all-reduce is a peer-HBM read fused into the Adam
      # kernel (csrc/cuda/peer.cu), one NVLink barrier per step, no NCCL call inside the captured step
      import torch.distributed as dist
      from ..parallel.peer import exchange_peer_tensors
      assert pad == 0, 'flat parameter buffer must be a multiple of 4 floats'
      rank = dist.get_rank(self.group)
      peers_g = exchange_peer_tensors(torch.zeros_like(self.p32), self.group)
      flags = exchange_peer_tensors(torch.zeros(2 * self.world, dtype=torch.int32, device=dev), self.group)
      self.g32 = peers_g[rank]
      self.peer_group = self.nat.PeerGroup(dev.index, rank, peers_g, flags)
    self.m = torch.zeros_like(self.p32)
    self.v = torch.zeros_like(self.p32)

  def param(self, name, grad: bool = False) -> torch.Tensor:
    """bf16 view of a parameter (grad=True: its fp32 gradient slot)."""
    o, shape = self.param_index[name]
    buf = self.g32 if grad else self.p16
    return buf[o:o + math.prod(shape)].view(*shape)

  def _p32(self, name, grad: bool = False) -> torch.Tensor:
    o, shape = self.param_index[name]
    return (self.g32 if grad else self.p32)[o:o + math.prod(shape)]

  def _rel_params(self, kind, l: int, t: int, grad: bool = False) -> torch.Tensor:
    """Flat bf16 view (grad=True: fp32 gradient) of the parameters (kind, l, r) of the relations r into (l, t), which
    the layout places back to back."""
    rels = self.in_rel[l][t]
    o, shape = self.param_index[(kind, l, rels[0])]
    n = math.prod(shape)
    assert all(self.param_index[(kind, l, r)][0] == o + i * n for i, r in enumerate(rels))
    return (self.g32 if grad else self.p16)[o:o + n * len(rels)]

  def state_dict(self):
    return {'p32': self.p32.clone(), 'm': self.m.clone(), 'v': self.v.clone(), 'step': int(self.step_dev[0].item()),
            'sample_step': int(self.arena.step.item()), 'step_idx': self.step_idx, 'seed': self.seed}

  def load_state_dict(self, s):
    self.p32.copy_(s['p32']); self.m.copy_(s['m']); self.v.copy_(s['v'])
    self.p16.copy_(self.p32)
    self.step_dev.zero_()
    self.step_dev[0] = int(s['step'])
    self.arena.step.fill_(int(s['sample_step']))
    self.step_idx, self.seed = s['step_idx'], s['seed']

  # ------------------------------------------------------------------ step pieces
  def _rel_ell(self, r: int, nh: int):
    return [self.arena.ell_of(r, h) for h in range(nh)], [max(self.fan[r][h], 1) for h in range(nh)]

  def _sample(self):
    self.arena.sample([self.tid[self.seed_type]], [self._seeds], self.L * len(self.edge_types))

  def _plan(self, kind: str, l: int, t: int):
    key = (kind, l, t)
    pl = self._plans.get(key)
    if pl is None:
      nh = self.L - l + 1
      pl = self.nat.TcGemm(self.device.index)
      W = self.param(('W', l, t))
      if kind == 'fwd':
        pl.add_forward(self.A[l][t], W, self.param(('b', l, t)), l < self.L, self.Z[l][t], self._ctr[t], nh)
      else:
        pl.add_wgrad(self.dPre[l][t], self.A[l][t], self.param(('W', l, t), True), self._ctr[t], nh)
        if l > 1:
          pl.add_dgrad(self.dPre[l][t], W, self.dA[l][t], self._ctr[t], nh)
      self._plans[key] = pl
    return pl

  def _head_plan(self, dZ: Optional[torch.Tensor] = None):
    """TcGemm of the Linear head of the attention engines over the seed type's batch rows: the forward into `logits`,
    or (dZ given) the weight gradient and the dgrad into dZ."""
    key = ('head', dZ is None)
    pl = self._plans.get(key)
    if pl is None:
      st = self.tid[self.seed_type]
      Z, c = self.Z[self.L][st], self._ctr[st]
      pl = self.nat.TcGemm(self.device.index)
      if dZ is None:
        pl.add_forward(Z, self.param(('head_W',)), self.param(('head_b',)), False, self.logits, c, 1)
      else:
        pl.add_wgrad(self.dlogits, Z, self.param(('head_W',), True), c, 1)
        pl.add_dgrad(self.dlogits, self.param(('head_W',)), dZ, c, 1)
      self._plans[key] = pl
    return pl

  def _gather_feat(self, t: int, ids: torch.Tensor, n_dev: Optional[torch.Tensor], out: torch.Tensor):
    """out[i, :in_dim] = bf16 feature row ids[i] of type t (MXFP8 tables are de-quantised); rows past the device count
    `n_dev` are zeros.  One launch."""
    name = self.ntypes[t]
    if self.feature_format[name] == 'mxfp8':
      self.feat[name].gather_mxfp8_into(ids, None, n_dev, out, self.dim_in[name])
    else:
      self.feat[name].gather_into(ids, None, n_dev, out)

  def _gather_input(self, u: int):
    """Layer-1 input of the attention engines: the feature rows of every sampled node of type u into X0[u]."""
    n = min(self.X0[u].shape[0], self.cap_nodes[u])
    self._gather_feat(u, self.arena.nodes_of(u)[:n], self._ctr[u][self.L + 1:self.L + 2], self.X0[u][:n])

  def _loss(self, logits: torch.Tensor, dlogits: torch.Tensor, bias_grad: torch.Tensor):
    """Forward tail: clear the gradients, then the fused log-softmax / NLL of the seed rows of `logits`, writing
    `dlogits` and the last layer's bias gradient."""
    nat, st = self.nat, self.tid[self.seed_type]
    if self.peer_group is not None:
      self.peer_group.barrier(1)            # peers finished reading last step's gradients
    nat.zero_grads(self.g32, self.loss, self.correct)
    nat.softmax_nll(logits, self.C, None, self.labels, self.arena.nodes_of(st), self._ctr[st], self.loss, dlogits,
                    self.correct, bias_grad, True)

  def _forward(self):
    nat, ar = self.nat, self.arena
    for l in range(1, self.L + 1):
      nh = self.L - l + 1
      for t in self.targets[l]:
        offs, self_col = self.col[l][t]
        A = self.A[l][t]
        for j, r in enumerate(self.in_rel[l][t]):
          s = self.nt[r]
          d = self._width_in(l, s)
          ell, ks = self._rel_ell(r, nh)
          if l == 1:
            nat.sage_aggregate_block(self.feat[self.ntypes[s]], ar.nodes_of(s), None, d, self._ctr[t], nh, ell, ks,
                                     ar.deg_of(r), A, offs[j])
          else:
            nat.sage_aggregate_block(None, None, self.Z[l - 1][s], d, self._ctr[t], nh, ell, ks, ar.deg_of(r), A,
                                     offs[j])
        d = self._width_in(l, t)
        blk = A[:, self_col:self_col + d]
        if l == 1:
          n = min(A.shape[0], self.cap_nodes[t])
          self._gather_feat(t, ar.nodes_of(t)[:n], self._ctr[t][nh:nh + 1], blk)
        else:
          blk.copy_(self.Z[l - 1][t][:A.shape[0]])
        self._plan('fwd', l, t).run()
    st = self.tid[self.seed_type]
    self._loss(self.Z[self.L][st], self.dPre[self.L][st], self.param(('b', self.L, st), True))

  def _backward(self):
    nat, ar = self.nat, self.arena
    for l in range(self.L, 0, -1):
      nh = self.L - l + 1
      for t in self.targets[l]:
        self._plan('bwd', l, t).run()
      if l == 1:
        break
      H = self.hidden
      for s in self.targets[l - 1]:
        nat.zero_rows(self.dH[l - 1][s], self._ctr[s], nh + 1)
      for t in self.targets[l]:
        offs, self_col = self.col[l][t]
        for j, r in enumerate(self.in_rel[l][t]):
          ell, ks = self._rel_ell(r, nh)
          nat.sage_scatter_block(self.dA[l][t], H, offs[j], self._ctr[t], nh, ell, ks, ar.deg_of(r),
                                 self.dH[l - 1][self.nt[r]])
        nat.add_block_f32(self.dA[l][t], self_col, H, self._ctr[t], nh, self.dH[l - 1][t])
      for s in self.targets[l - 1]:
        nat.relu_bwd_cast(self.dH[l - 1][s], self.Z[l - 1][s], self._ctr[s], nh + 1, self.dPre[l - 1][s],
                          self.param(('b', l - 1, s), True), True)

  def _optimizer(self):
    if self.peer_group is not None:
      self.peer_group.barrier(0)            # every rank finished writing its gradients
      self.peer_group.adam(self.p32, self.m, self.v, self.p16, self.lr, 0.9, 0.999, 1e-8, self.wd, self.step_dev,
                           1.0 / self.world)
      return
    self.nat.adam_step(self.p32, self.g32, self.m, self.v, self.p16, self.lr, 0.9, 0.999, 1e-8, self.wd,
                       self.step_dev, 1.0)

  def _step_eager(self):
    self._sample()
    self._forward()
    self._backward()
    self._optimizer()

  # ------------------------------------------------------------------ public API
  def warmup_and_capture(self, n_eager: int = 2):
    """Run a few eager steps (lazy inits, GEMM plans), then capture the step into one CUDA graph and set
    `kernels_per_step` to its kernel, memset and memcpy nodes.  Engines built with use_cuda_graph=False capture the
    step only to count it, and keep running eagerly."""
    with torch.cuda.device(self.device):
      saved = self.state_dict()
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        for _ in range(n_eager):
          self._step_eager()
      torch.cuda.current_stream().wait_stream(side)
      torch.cuda.synchronize()
      self.load_state_dict(saved)
      g = torch.cuda.CUDAGraph(keep_graph=True)
      with torch.cuda.graph(g):
        self._step_eager()
      self.kernels_per_step = sum(self.nat.graph_node_counts(g.raw_cuda_graph()))
      if self.use_cuda_graph:
        g.instantiate()
      torch.cuda.synchronize()
      self.load_state_dict(saved)
      self._graph = g if self.use_cuda_graph else None

  def train_step(self, seeds: torch.Tensor) -> torch.Tensor:
    """One training step on a batch of seed ids of `seed_type` (host-pinned or device tensor); returns the device
    scalar holding the mean NLL loss."""
    n = seeds.numel()
    assert n <= self.bs
    if n < self.bs:
      self._seeds.fill_(-1)
    self._seeds[:n].copy_(seeds, non_blocking=True)
    if self._graph is not None:
      self._graph.replay()
    else:
      self._step_eager()
    self.step_idx += 1
    return self.loss

  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    n = seeds.numel()
    self._seeds.fill_(-1)
    self._seeds[:n].copy_(seeds)
    assert self.peer_group is None, 'evaluate_batch runs the gradient protocol of the multi-GPU step; use a single-GPU replica'
    self._sample()
    self._forward()
    st = self.tid[self.seed_type]
    return float(self.loss.item()), int(self.correct.item()), int(self._ctr[st][1].item())

  # ------------------------------------------------------------------ full-neighbourhood inference
  @torch.no_grad()
  def inference(self, chunk_rows: Optional[int] = None) -> torch.Tensor:
    """Exact layer-wise full-neighbourhood inference: bf16 logits [num_nodes[seed_type], num_classes] of every node of
    the seed type.

    Every layer uses each node's complete CSR row in every relation (the `fanout >= degree` limit of the training
    forward), with the bf16 parameters of the training forward, no dropout and the same activations (R-SAGE: ReLU;
    R-GAT: leaky_relu(0.01); HGT: GELU, the skip gate, and ReLU on the input layer).  Layer l computes every node of
    every type in `targets[l]` from exactly the relations `in_rel[l][t]`, and the last layer only the seed type, so the
    model is the sampled one: `inference()[seeds]` equals the sampled forward when every relation's fan-out is at least
    every in-degree and is positive at every hop.

    Runs on the current stream, so it sees every step queued before it.  The per-type activation tables (one or two
    per type: ping-pong between layers), the per-relation projection / score / attention buffers of the layer being
    computed and one chunk of `chunk_rows` rows for the aggregation operands are allocated for the call only;
    parameters, optimizer state, gradients, arenas, `step_dev`, the sampler step and captured graphs are not touched,
    and training can continue afterwards.  No reduction uses floating-point atomics, so the result is bitwise identical
    from call to call and for any `chunk_rows` (None sizes the chunk from free device memory).

    Not collective: with several GPUs a rank reads peer graph shards and feature rows in place."""
    dev, L = self.device, self.L
    st = self.tid[self.seed_type]
    with torch.cuda.device(dev):
      chunk_rows = infer_chunk_rows(chunk_rows, max(self._n_nodes), self._infer_chunk_row_bytes(), dev)
      # TcGemm / elementwise row counts read on the device: [0] one chunk, [1 + t] every node of type t
      self._rows_dev = torch.tensor([chunk_rows] + self._n_nodes, dtype=torch.int32, device=dev)
      self._ids = torch.arange(max(self._n_nodes), dtype=torch.int64, device=dev)
      X = self._infer_input(chunk_rows)
      for l in range(1, L + 1):
        Z = {t: torch.empty(self._n_nodes[t], self.Z[l][t].shape[1], dtype=torch.bfloat16, device=dev)
             for t in self.targets[l]}
        self._infer_layer(l, X, Z, chunk_rows)
        X = Z
      out = self._infer_head(X[st])
      self._rows_dev = self._ids = None
      return out[:, :self.C].contiguous()

  def _gh(self, r: int):
    return self.graphs[self.edge_types[r]].graph_handler

  def _infer_chunk_row_bytes(self) -> int:
    """Bytes per chunk row of the call's chunk buffers (sizes the default chunk)."""
    return 2 * max(A.shape[1] for l in range(1, self.L + 1) for A in self.A[l].values())

  def _infer_input(self, chunk_rows: int):
    """Input tables of layer 1 (None: layer 1 reads the feature tables)."""
    return None

  def _infer_head(self, X: torch.Tensor) -> torch.Tensor:
    """Logits from the last layer's output (R-SAGE: the last layer is the classifier)."""
    return X

  def _infer_linear_head(self, X: torch.Tensor) -> torch.Tensor:
    """The attention engines' `_infer_head`: their Linear head over every seed-type node."""
    out = torch.empty(X.shape[0], self.n_out_pad, dtype=torch.bfloat16, device=self.device)
    self._gemm(X, self.param(('head_W',)), self.param(('head_b',)), False, out, 1 + self.tid[self.seed_type])
    return out

  def _gather_chunk(self, t: int, r0: int, r1: int, buf: torch.Tensor) -> torch.Tensor:
    """bf16 feature rows [r0, r1) of type t, gathered from its feature table (any memory tier) into buf."""
    d = self.dim_in[self.ntypes[t]]
    x = buf[:(r1 - r0) * d].view(r1 - r0, d)
    self._gather_feat(t, self._ids[r0:r1], None, x)
    return x

  def _gemm(self, A, W, b, relu, out, idx):
    infer_gemm(self.nat, A, W, b, relu, out, self._rows_dev, idx)

  def _infer_layer(self, l: int, X, Z, chunk_rows: int):
    """R-SAGE layer l: A_t = [mean_r1 | ... | mean_rk | self] per chunk (sage_full_aggregate, mean-only blocks), then
    one TcGemm against W_t with the bias and, below the top layer, ReLU."""
    nat, dev = self.nat, self.device
    K_max = max(self.A[l][t].shape[1] for t in self.targets[l])
    buf = torch.empty(chunk_rows * K_max, dtype=torch.bfloat16, device=dev)
    for t in self.targets[l]:
      offs, self_col = self.col[l][t]
      d_t = self._width_in(l, t)
      K = self_col + d_t
      for r0, r1 in infer_chunks(self._n_nodes[t], chunk_rows):
        a = buf[:(r1 - r0) * K].view(r1 - r0, K)
        for j, r in enumerate(self.in_rel[l][t]):
          s = self.nt[r]
          d = self._width_in(l, s)
          blk = a[:, offs[j]:offs[j] + d]
          if l == 1:
            nat.sage_full_aggregate(self._gh(r), self.feat[self.ntypes[s]], None, 0, 0, d, r0, r1, False, None, False,
                                    blk, mean_only=True)
          else:
            nat.sage_full_aggregate(self._gh(r), None, X[s], 0, 0, d, r0, r1, False, None, False, blk,
                                    mean_only=True)
        blk = a[:, self_col:K]
        if l == 1:
          self._gather_feat(t, self._ids[r0:r1], None, blk)
        else:
          blk.copy_(X[t][r0:r1])
        self._gemm(a, self.param(('W', l, t)), self.param(('b', l, t)), l < self.L, Z[t][r0:r1], 0)

  def overflow_count(self) -> int:
    return int(self.arena.counters[self._ovf_idx].item())

  def batch_sizes(self):
    """{type: nodes per hop} and {etype: edges per hop} of the last batch (host sync; diagnostics)."""
    c = self.arena.counters.cpu().tolist()
    NT = len(self.ntypes)
    nodes = {t: [c[i * 8 + h + 1] - c[i * 8 + h] for h in range(self.L + 1)] for i, t in enumerate(self.ntypes)}
    edges = {et: c[NT * 8 + r * 4:NT * 8 + r * 4 + self.L] for r, et in enumerate(self.edge_types)}
    return nodes, edges

  def close(self):
    """Drop the captured graph (call before destroying the process group)."""
    torch.cuda.synchronize(self.device)
    self._graph = None
