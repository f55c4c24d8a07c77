"""GraphSAGE: a generic PyG-style module and the fused, CUDA-graphed training engine.

The reference ships no model code; its examples use PyG's SAGEConv
(examples/train_sage_ogbn_products.py:30-59: 3 x SAGEConv, hidden 256, mean aggregation,
fanout [15,10,5], batch 1024).  `GraphSAGE` below is the drop-in eager module for the
`NeighborLoader` path.  `GraphSageEngine` is the H100-first path:

  sample (static-shape arena, no host sync)
    -> layer 1: ONE wgmma kernel = peer/local HBM row gather + neighbour mean +
       [mean | self] x W1 + bias + ReLU (csrc/cuda/sage_tc.cu)
    -> layers 2..L: ELL aggregation kernel + wgmma GEMM (csrc/cuda/tc_gemm.cu)
    -> fused log-softmax/NLL fwd+bwd -> hand-written backward -> Adam (multi-GPU: fused with a peer-HBM all-reduce)

with every extent read from device counters, so the whole step is a fixed launch sequence
replayed from a CUDA graph.
"""
import math
from typing import List, Optional

import torch

from ..utils.tracing import nvtx_range
import torch.nn as nn
import torch.nn.functional as F

from ..data.quantize import mxfp8_row_bytes
from ..ops import require_native


# ----------------------------------------------------------------------------- eager modules
class SAGEConv(nn.Module):
  """out_i = W_l . mean_{j in N(i)} x_j + W_r . x_i + b   (PyG SAGEConv semantics)."""

  def __init__(self, in_channels: int, out_channels: int, bias: bool = True):
    super().__init__()
    self.lin_l = nn.Linear(in_channels, out_channels, bias=bias)
    self.lin_r = nn.Linear(in_channels, out_channels, bias=False)

  def forward(self, x, edge_index, num_dst: Optional[int] = None):
    x_src, x_dst = (x, x) if not isinstance(x, tuple) else x
    n_dst = num_dst if num_dst is not None else x_dst.shape[0]
    x_dst = x_dst[:n_dst]
    src, dst = edge_index[0], edge_index[1]
    agg = torch.zeros(n_dst, x_src.shape[1], dtype=x_src.dtype, device=x_src.device)
    agg.index_add_(0, dst, x_src[src])
    deg = torch.zeros(n_dst, dtype=torch.float32, device=x_src.device)       # fp32: bf16 counts exactly only to 256
    deg.index_add_(0, dst, torch.ones_like(dst, dtype=torch.float32))
    agg = agg * (1.0 / deg.clamp(min=1)).to(agg.dtype).unsqueeze(1)
    return self.lin_l(agg) + self.lin_r(x_dst)


class GraphSAGE(nn.Module):
  """Eager GraphSAGE for `NeighborLoader` batches; trims targets layer by layer using
  `num_sampled_nodes/edges` when given (the reference relies on PyG trim_to_layer,
  examples/train_sage_prod_with_trim.py:60-65)."""

  def __init__(self, in_channels: int, hidden_channels: int, out_channels: int, num_layers: int = 3,
               dropout: float = 0.0):
    super().__init__()
    dims = [in_channels] + [hidden_channels] * (num_layers - 1) + [out_channels]
    self.convs = nn.ModuleList([SAGEConv(dims[i], dims[i + 1]) for i in range(num_layers)])
    self.dropout = dropout

  def forward(self, x, edge_index, num_sampled_nodes=None, num_sampled_edges=None):
    L = len(self.convs)
    for i, conv in enumerate(self.convs):
      n_dst = None
      ei = edge_index
      if num_sampled_nodes is not None and num_sampled_edges is not None:
        keep_hops = L - i                       # hops whose edges are still needed
        n_e = int(sum(num_sampled_edges[:keep_hops]))
        n_dst = int(sum(num_sampled_nodes[:keep_hops]))
        ei = edge_index[:, :n_e]
      x = conv(x, ei, n_dst)
      if i < L - 1:
        x = F.relu(x)
        if self.dropout > 0:
          x = F.dropout(x, self.dropout, self.training)
    return x


# ----------------------------------------------------------------------------- engine
def _round_up(x, m):
  return (x + m - 1) // m * m


# The chunking of the engines' exact layer-wise inference (GraphSageEngine, HeteroSageEngine and its subclasses).
def infer_chunk_rows(chunk_rows: Optional[int], n: int, row_bytes: int, device) -> int:
  """Target rows per chunk, clamped to [1, n]; None: a quarter of the free device memory at row_bytes per row, at
  least 4096 and at most 512 k rows."""
  if chunk_rows is None:
    free, _ = torch.cuda.mem_get_info(device)
    chunk_rows = max(4096, min(1 << 19, free // 4 // row_bytes))
  return max(1, min(int(chunk_rows), n))


def infer_chunks(n: int, chunk_rows: int):
  """[r0, r1) of n rows, chunk_rows at a time."""
  for r0 in range(0, n, chunk_rows):
    yield r0, min(n, r0 + chunk_rows)


def infer_gemm(nat, A, W, b, relu, out, rows_dev, idx):
  """out = act(A W^T + b) by a single-use TcGemm forward over rows_dev[idx] rows."""
  g = nat.TcGemm(A.device.index)
  g.add_forward(A, W, b, relu, out, rows_dev, idx)
  g.run()


class GraphSageEngine(object):
  """Static-shape, CUDA-graph-captured GraphSAGE training step.

  Args:
    graph: `data.Graph` in a device mode (single shard or multi-GPU shards).
    feature_table: native RowTableHandle of bf16 rows indexed by global node id
      (`UnifiedTensor._table()` / `PartitionedFeature.table`); width = in_dim.
    labels: int64 [num_nodes] on the device.
    in_dim: feature width, a multiple of 8 up to 1024 (64 or 128 for the fused layer-1 kernel, a multiple of 32
      for the wgmma weight-gradient GEMM).
    num_nodes: number of graph nodes (arena sizing).
    fanouts / batch_size / hidden / num_classes: model + sampling config.  `hidden` is a multiple of 8 up to 1024
      (a multiple of 64 unless every hidden layer runs the fused kernel); see `_check_widths`.  Widths that no
      kernel supports raise ValueError here.
    group: torch.distributed group of the data-parallel ranks (None = single process).  Every rank reads the
      others' gradients and feature rows in place, so the GPUs of the group need peer access.
    use_fused: True = use the wgmma gather+GEMM kernel where the shape allows; 'auto' = time the
      fused and the unfused (aggregate kernel + wgmma GEMM) layer on real batches during warm-up and
      keep the faster one (remote-heavy multi-GPU runs can favour the unfused pair).
    use_cuda_graph: capture sample+forward+backward(+adam) into CUDA graphs.
    preaggregate_layer1: pipelined engines whose layer 1 runs unfused aggregate layer 1 of the next batch on the
      sampling stream, right after sampling it (the aggregation depends on the batch and the feature table only, not
      on the weights), so the training chain starts with the layer-1 GEMM.  Each arena then has its own layer-1 A
      buffer.  None = on where it applies; False = aggregate inside the forward as usual.
  """
  # read by bench.py: the backward of the aggregation is always the atomics-free gather (csrc/cuda/transpose.cu)
  use_gather_bwd = True
  # read by bench.py and benchmarks/bench_link.py: every contraction runs on this project's kernels, none on cuBLAS
  library_gemms_per_step = 0

  def __init__(self, graph, feature_table, labels: torch.Tensor, in_dim: int, num_nodes: int,
               fanouts: List[int] = (15, 10, 5), batch_size: int = 1024, hidden: int = 256,
               num_classes: int = 47, lr: float = 3e-3, weight_decay: float = 0.0, seed: int = 0,
               device: Optional[torch.device] = None, group=None, use_fused: bool = True,
               use_cuda_graph: bool = True, calibration_seeds: Optional[torch.Tensor] = None,
               calibration_margin: float = 1.3, calibration_batches: int = 16, pipeline: bool = False,
               check_every: int = 64, auto_regrow: bool = True, feature_format: str = 'bf16',
               deterministic_sampling: bool = False,
               dropout: float = 0.0, preaggregate_layer1: Optional[bool] = None):
    self.nat = require_native()
    # dropout on the hidden activations (the reference example trains with p = 0.5,
    # examples/train_sage_ogbn_products.py:58): one in-place Philox kernel per hidden layer in training steps,
    # mask keyed by (seed, layer, optimizer step, element); backward rescales inside sage_gather_bwd.
    assert 0.0 <= float(dropout) < 1.0
    self.dropout = float(dropout)
    # 'mxfp8': `feature_table` holds data.quantize_mxfp8 rows (uint8, mxfp8_row_bytes(in_dim) bytes, in_dim a multiple
    # of 32), de-quantised inside whichever kernel reads them (half the gather bytes).  Layer 1 runs the fused kernel
    # where its MXFP8 loader applies (in_dim 128 and a fused-capable shape and table), otherwise sage_aggregate + GEMM.
    assert feature_format in ('bf16', 'mxfp8')
    self.feature_format = feature_format
    if feature_format == 'mxfp8':
      if int(in_dim) % 32 != 0:
        raise ValueError(f'MXFP8 features: in_dim must be a multiple of 32 (got {in_dim})')
      if not feature_table.is_uint8 or feature_table.width != mxfp8_row_bytes(int(in_dim)):
        raise ValueError(f'MXFP8 features: the table must hold uint8 rows of mxfp8_row_bytes({in_dim}) = '
                         f'{mxfp8_row_bytes(int(in_dim))} bytes (data.quantize_mxfp8)')
      use_fused = True
    self.pipeline = bool(pipeline)
    self.deterministic_sampling = bool(deterministic_sampling)
    self._preagg_opt = preaggregate_layer1 is None or bool(preaggregate_layer1)
    self.preaggregate = False         # resolved once the layer-1 variant is known (_resolve_preagg)
    self._tc_plans = {}
    self.peer_group = None
    self.graph = graph
    graph.lazy_init()
    self.gh = graph.graph_handler
    self.feat = feature_table
    self.device = torch.device(device) if device is not None else torch.device('cuda', graph.device)
    self.labels = labels.to(self.device)
    self.fanouts = [int(k) for k in fanouts]
    self.L = len(self.fanouts)
    assert 1 <= self.L <= 4
    self.bs = int(batch_size)
    self.in_dim, self.hidden, self.C = int(in_dim), int(hidden), int(num_classes)
    self.n_out_pad = _round_up(self.C, 64)
    self._check_widths(use_fused)
    self.lr, self.wd = lr, weight_decay
    self.seed = int(seed)
    self.group = group
    import torch.distributed as dist
    self.world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
    self.use_cuda_graph = use_cuda_graph
    self.step_idx = 0
    self.kernels_per_step = 0

    dev = self.device
    self._num_nodes = int(num_nodes)
    # ---- health monitoring (peer-barrier timeouts, arena overflow) without stalling the step: every
    # `check_every` steps a tiny probe is copied to pinned memory and read one period later
    self.check_every = int(check_every)
    self.auto_regrow = bool(auto_regrow)
    self.regrow_count = 0
    self._overflow_seen = 0
    self._probe_event = None
    with torch.cuda.device(dev):
      cap_override = []
      if calibration_seeds is not None and calibration_seeds.numel() >= self.bs:
        cap_override = self._calibrate(calibration_seeds, int(num_nodes), calibration_margin, calibration_batches)
      self.calibrated = bool(cap_override)
      self.dims_in = [self.in_dim] + [self.hidden] * (self.L - 1)
      self.dims_out = [self.hidden] * (self.L - 1) + [self.n_out_pad]
      self._build_buffers(cap_override)
      self._init_params()
      n_arenas = len(self._arenas)
      self._seeds = [torch.zeros(self.bs, dtype=torch.int64, device=dev) for _ in range(n_arenas)]
      self._side = torch.cuda.Stream(device=dev) if self.pipeline else None
      self._primed = False
      self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
      self.correct = torch.zeros(1, dtype=torch.int32, device=dev)
      self.step_dev = torch.zeros(2, dtype=torch.int32, device=dev)   # {steps taken, block ticket}
      self._health_dev = torch.zeros(2, dtype=torch.int32, device=dev)
      self._health_host = torch.zeros(2, dtype=torch.int32).pin_memory()
      self._autotune_fused = (use_fused == 'auto')
      # layer 1 also needs a feature table that the fused kernel's 32-bit row handles can address
      self.fused_ok = [False] + [bool(use_fused and self._fused_shape(l, self.dims_in[l - 1], self.dims_out[l - 1]))
                                 for l in range(1, self.L + 1)]
      bf = torch.bfloat16
      self.w_packed = [None] + [torch.zeros(self.dims_out[l - 1] * 2 * self.dims_in[l - 1], dtype=bf, device=dev)
                                if self.fused_ok[l] else None for l in range(1, self.L + 1)]
      self._repack()
      self._resolve_preagg()
    self._graph_fb = None

  def _fused_shape(self, l: int, d: int, n_out: int) -> bool:
    """Can the fused layer kernel run layer l (input width d, output width n_out)?  Its MXFP8 loader is written for
    128-wide rows."""
    if l == 1 and self.feature_format == 'mxfp8' and d != 128:
      return False
    return bool(self.nat.sage_fused_supported(d, n_out, self.feat if l == 1 else None))

  def _check_widths(self, use_fused):
    """Rejects, at construction, widths that a kernel of the step cannot run (instead of failing at the first step or
    silently computing on truncated rows).  `in_dim` and `hidden` are multiples of 8 up to 1024, the widest row of
    the aggregation and gather-backward kernels.  The wgmma weight-gradient GEMM needs every layer's A operand
    [mean | self] to be a multiple of 64 wide, so `in_dim` and `hidden` are multiples of 32; and the wgmma forward
    GEMM needs `hidden` to be a multiple of 64 when a hidden layer runs unfused, i.e. unless each hidden layer fits
    the fused layer kernel (input width 64 or 128, `hidden` <= 256)."""
    for name, d in (('in_dim', self.in_dim), ('hidden', self.hidden)):
      if d % 8 != 0 or not 8 <= d <= 1024:
        raise ValueError(f'{name} must be a multiple of 8 in [8, 1024] (got {d})')
    if self.C < 1:
      raise ValueError(f'num_classes must be >= 1 (got {self.C})')
    for name, d in (('in_dim', self.in_dim), ('hidden', self.hidden)):
      if name == 'hidden' and self.L == 1:
        continue
      if d % 32 != 0:
        raise ValueError(f'{name} = {d}: the weight-gradient GEMM needs the layer input [mean | self] '
                         f'(2 x {d} = {2 * d} columns) to be a multiple of 64 wide')
    if self.hidden % 64 != 0:
      dims_in = [self.in_dim] + [self.hidden] * (self.L - 1)
      for l in range(1, self.L):          # hidden layers (the last layer's output is padded to 64 columns)
        fused = use_fused != 'auto' and bool(use_fused) and self._fused_shape(l, dims_in[l - 1], self.hidden)
        if not fused:
          raise ValueError(f'hidden = {self.hidden}: layer {l} runs the unfused forward GEMM, whose output width must '
                           f'be a multiple of 64')

  def _build_buffers(self, cap_override):
    """(Re)creates everything whose size depends on the arena capacities: sampler arenas, activation /
    gradient buffers, cached GEMM launches.  Parameters and optimizer state are untouched."""
    dev = self.device
    bf = torch.bfloat16
    # pipelined mode double-buffers the sampler state: batch i+1 is sampled on a side stream
    # while batch i trains (the reference's sampler<->trainer producer/consumer pipeline,
    # distributed/dist_sampling_producer.py:54-163, collapsed onto CUDA streams of one GPU)
    n_arenas = 2 if self.pipeline else 1
    self._arenas = [self.nat.SamplerArena(dev.index, self.bs, self.fanouts, False, self._num_nodes,
                                          list(cap_override) if cap_override else [])
                    for _ in range(n_arenas)]
    self._cur = 0
    for p_, ar_ in enumerate(self._arenas):
      ar_.step.fill_(p_ - n_arenas)          # disjoint Philox stream ids per arena
      ar_.deterministic = self.deterministic_sampling   # local ids of a hop in ascending global-id order
      if self.L >= 2:
        # the sampler also builds the batch's transposed adjacency, which the gather backward of the aggregation
        # reads (csrc/cuda/transpose.cu); layer 2 uses hops 0..L-2, deeper layers a prefix of them
        ar_.enable_transpose(self.L - 1)
    self.cap_rows = list(self.arena.cap_rows)           # frontier capacity per hop (+ last-hop additions)
    # layer l (1-based) targets = nodes of hops 0..L-l
    self.cap_T = [0] + [int(sum(self.cap_rows[:self.L - l + 1])) for l in range(1, self.L + 1)]
    self.cap_T = [min(c, self.arena.cap_nodes) for c in self.cap_T]
    self.A = [None] + [torch.zeros(self.cap_T[l], 2 * self.dims_in[l - 1], dtype=bf, device=dev)
                       for l in range(1, self.L + 1)]
    # layer-1 A operand per arena (see _A): pre-aggregation writes arena b+1's while arena b's is read
    self._A1 = [self.A[1]] + [torch.zeros_like(self.A[1]) for _ in range(1, n_arenas) if self.preaggregate]
    self.Z = [None] + [torch.zeros(self.cap_T[l], self.dims_out[l - 1], dtype=bf, device=dev)
                       for l in range(1, self.L + 1)]
    self.dPre = [None] + [torch.zeros(self.cap_T[l], self.dims_out[l - 1], dtype=bf, device=dev)
                          for l in range(1, self.L + 1)]
    self.dA = [None, None] + [torch.zeros(self.cap_T[l], 2 * self.dims_in[l - 1], dtype=bf, device=dev)
                              for l in range(2, self.L + 1)]
    self._tc_plans = {}
    self._graphs = []
    self._graph_fb = None

  def regrow(self, factor: float = 1.5):
    """Enlarge the (calibrated) arena after neighbours were dropped by the capacity guard: new per-hop
    capacities = old x factor (bounded by the worst case), buffers and CUDA graphs are rebuilt, parameters,
    optimizer state and the sampling position are kept.  Collective when world > 1 (every rank calls it at the
    same step -- `_health_tick` guarantees that)."""
    with torch.cuda.device(self.device):
      torch.cuda.synchronize()
      steps = [int(a.step.item()) for a in self._arenas]
      tmp = self.nat.SamplerArena(self.device.index, self.bs, self.fanouts, False, self._num_nodes)
      worst = list(tmp.cap_rows)
      del tmp
      caps = [self.bs] + [min(worst[h], (int(self.cap_rows[h] * factor) + 255) // 128 * 128)
                          for h in range(1, self.L + 1)]
      had_graphs = bool(self._graphs)
      self._build_buffers(caps)
      for a, v in zip(self._arenas, steps):
        a.step.fill_(v)
      self._primed = False
      self.regrow_count += 1
      if had_graphs:
        self.warmup_and_capture(n_eager=1)

  def _health_tick(self):
    """Called once per train_step.  Every `check_every` steps: (1) read the probe enqueued one period ago --
    raise if a peer barrier timed out (the Adam kernels already skipped that update), regrow the arena if
    neighbours were dropped; (2) enqueue a new probe (max-reduced over ranks so that every rank takes the same
    decision at the same step)."""
    if self.check_every <= 0 or self.step_idx % self.check_every != 0:
      return
    if self._probe_event is not None:
      self._probe_event.synchronize()
      err, ovf = int(self._health_host[0]), int(self._health_host[1])
      self._probe_event = None
      if err != 0:
        raise RuntimeError(f'peer barrier timed out waiting for rank {err - 1}: a peer process died or stalled; '
                           'the optimizer updates since then were skipped')
      if ovf > self._overflow_seen:
        self._overflow_seen = ovf
        if self.auto_regrow:
          self.regrow()
    h = self._health_dev
    h.zero_()
    for pg in self._peer_groups:
      torch.maximum(h[0:1], pg.err, out=h[0:1])
    for a in self._arenas:
      h[1:2].add_(a.counters[12:13])
    if self.regrow_count:
      h[1:2].add_(self._overflow_seen)      # counters restart from zero in a rebuilt arena
    if self.world > 1:
      import torch.distributed as dist
      dist.all_reduce(h, op=dist.ReduceOp.MAX, group=self.group)
    self._health_host.copy_(h, non_blocking=True)
    self._probe_event = torch.cuda.Event()
    self._probe_event.record()

  @property
  def arena(self):
    return self._arenas[self._cur]

  @property
  def seeds_dev(self):
    return self._seeds[self._cur]

  @property
  def g32(self):
    """Flat fp32 gradient buffer of the batch being trained (per parity when double-buffered)."""
    return self._g[self._cur % len(self._g)]

  def _A(self, l: int, parity: Optional[int] = None):
    """A operand [mean | self] of layer l; layer 1 has one per arena when pre-aggregated."""
    if l == 1 and self.preaggregate:
      return self._A1[self._cur if parity is None else parity]
    return self.A[l]

  def _resolve_preagg(self):
    """Pre-aggregation of layer 1 (see `preaggregate_layer1`) applies to pipelined engines whose layer 1 runs
    unfused.  While `use_fused='auto'` has not decided, layer 1 aggregates inside the forward, so that the timed
    unfused variant includes its aggregation."""
    on = self._preagg_opt and self.pipeline and not self.fused_ok[1] and not self._autotune_fused
    if on == self.preaggregate:
      return
    self.preaggregate = on
    self._A1 = [self.A[1]] + [torch.zeros_like(self.A[1]) for _ in range(1, len(self._arenas)) if on]
    self._tc_plans = {}

  # ------------------------------------------------------------------ capacity calibration
  def _calibrate(self, pool: torch.Tensor, num_nodes: int, margin: float, n_batches: int):
    """Size the arena from observed frontier sizes instead of the worst case
    bs*prod(fanouts): sample a few batches of the seed pool with a worst-case arena, take the
    per-hop maxima (max over ranks), add a margin.  All buffers and every cap-proportional
    launch (GEMMs, fills) shrink accordingly.  The kernels stay safe past the caps
    (excess nodes are dropped and counted in `overflow_count()`)."""
    dev = self.device
    tmp = self.nat.SamplerArena(dev.index, self.bs, self.fanouts, False, num_nodes)
    worst = list(tmp.cap_rows)
    mx = torch.zeros(self.L + 1, dtype=torch.int64, device=dev)
    g = torch.Generator(device='cpu')
    g.manual_seed(self.seed + 991)
    for i in range(n_batches):
      idx = torch.randint(0, pool.numel(), (self.bs,), generator=g)
      seeds = pool[idx].to(dev)
      tmp.sample(self.gh, seeds.contiguous(), None, self.seed + 17, i * 8, False, False, False)
      c = tmp.counters[:self.L + 2].to(torch.int64)
      mx = torch.maximum(mx, c[1:] - c[:-1])
    if self.world > 1:
      import torch.distributed as dist
      dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=self.group)
    mx = mx.cpu().tolist()
    caps = []
    for h in range(self.L + 1):
      c = int(mx[h] * margin) + 128
      c = (c + 127) // 128 * 128
      caps.append(min(c, worst[h]) if h > 0 else self.bs)
    del tmp
    torch.cuda.empty_cache()
    return caps

  def overflow_count(self) -> int:
    """Neighbours dropped by the capacity guard since construction (0 in normal operation)."""
    return int(sum(int(a.counters[12].item()) for a in self._arenas))

  # ------------------------------------------------------------------ parameters
  def _init_params(self):
    dev = self.device
    sizes = []
    for l in range(self.L):
      sizes.append(self.dims_out[l] * 2 * self.dims_in[l])   # W [N, 2d] = [W_neigh | W_self]
      sizes.append(self.dims_out[l])                          # bias
    total = sum(sizes)
    self.p32 = torch.zeros(total, dtype=torch.float32, device=dev)
    g = torch.Generator(device='cpu')
    g.manual_seed(self.seed)
    off = 0
    self.W32, self.b32, self._w_off, self._b_off = [], [], [], []
    for l in range(self.L):
      n, k = self.dims_out[l], 2 * self.dims_in[l]
      bound = 1.0 / math.sqrt(self.dims_in[l])
      w = (torch.rand(n, k, generator=g) * 2 - 1) * bound
      if l == self.L - 1 and self.n_out_pad > self.C:
        w[self.C:] = 0
      self.p32[off:off + n * k].copy_(w.flatten())
      self._w_off.append((off, n, k)); off += n * k
      self._b_off.append((off, n)); off += n
    self.p16 = self.p32.to(torch.bfloat16)
    self._g = [torch.zeros_like(self.p32)]
    self._peer_groups = []
    if self.world > 1:
      # gradients live in a symmetric-heap segment: the optimizer kernel of every rank reads
      # all peers' gradients over NVLink (all-reduce fused into Adam, no NCCL in the step)
      import torch.distributed as dist
      from ..parallel.peer import exchange_peer_tensors
      rank = dist.get_rank(self.group)
      # pipelined engines run parity graphs, so each parity gets its own gradient segment and
      # flag set: one cross-GPU barrier per step is then enough (the buffer written at step k is
      # not touched again before step k+2, after everybody passed the barrier of step k+1)
      n_par = 2 if self.pipeline else 1
      self._g = []
      for _ in range(n_par):
        peers_g = exchange_peer_tensors(torch.zeros_like(self.p32), self.group)
        flags = exchange_peer_tensors(torch.zeros(2 * self.world, dtype=torch.int32, device=dev), self.group)
        self._g.append(peers_g[rank])
        self._peer_groups.append(self.nat.PeerGroup(dev.index, rank, peers_g, flags))
      self.peer_group = self._peer_groups[0]
    self.m = torch.zeros_like(self.p32)
    self.v = torch.zeros_like(self.p32)

  def W(self, l, buf=None):      # l is 1-based
    off, n, k = self._w_off[l - 1]
    return (buf if buf is not None else self.p16)[off:off + n * k].view(n, k)

  def b(self, l, buf=None):
    off, n = self._b_off[l - 1]
    return (buf if buf is not None else self.p16)[off:off + n]

  def _repack(self):
    for l in range(1, self.L + 1):
      if self.fused_ok[l]:
        self.nat.pack_weight_into(self.W(l), self.w_packed[l])

  def state_dict(self):
    return {'p32': self.p32.clone(), 'm': self.m.clone(), 'v': self.v.clone(),
            'step': int(self.step_dev[0].item()), 'sample_step': [int(a.step.item()) for a in self._arenas],
            'step_idx': self.step_idx, 'seed': self.seed}

  def load_state_dict(self, s):
    self.p32.copy_(s['p32']); self.m.copy_(s['m']); self.v.copy_(s['v'])
    self.p16.copy_(self.p32)
    self.step_dev.zero_()
    self.step_dev[0] = int(s['step'])
    ss = s.get('sample_step', None)
    if ss is not None:
      for a, v in zip(self._arenas, ss if isinstance(ss, (list, tuple)) else [ss]):
        a.step.fill_(v)
    self.step_idx, self.seed = s['step_idx'], s['seed']
    self._repack()

  # ------------------------------------------------------------------ step pieces
  def _ell(self, l):
    """ELL blocks + strides used by layer l: hops 0..L-l."""
    nh = self.L - l + 1
    return list(self.arena.ell[:nh]), self.fanouts[:nh], nh

  def _sample(self, which: Optional[int] = None):
    # the Philox stream advances from a device-side step counter (arena.step) so that a
    # CUDA-graph replay draws fresh samples every step
    which = self._cur if which is None else which
    ar = self._arenas[which]
    # (the increment itself is folded into the first sampling kernel: step_inc)
    ar.sample(self.gh, self._seeds[which], None, self.seed, 0, False, False, True, len(self._arenas))
    if self.preaggregate:
      self._aggregate_layer1(which)

  def _aggregate_layer1(self, which: int):
    """Layer-1 aggregation of the batch in arena `which` into its A buffer, on the current stream (the sampling
    stream of a pipelined step).  With several GPUs it reads the peers' feature rows in place."""
    ar = self._arenas[which]
    nh = self.L
    self.nat.sage_aggregate(self.feat, ar.nodes, None, self.in_dim, ar.counters, nh, list(ar.ell[:nh]),
                            self.fanouts[:nh], ar.deg, self._A1[which])

  def _forward(self, train: bool = True):
    nat, ar = self.nat, self.arena
    for l in range(1, self.L + 1):
      self._forward_layer(l, train)
    self._forward_loss(train)

  def _forward_layer(self, l: int, train: bool = True):
    self._forward_layer_nodrop(l)
    if train and self.dropout > 0.0 and l < self.L:
      self.nat.dropout_bf16(self.Z[l], self.arena.counters, self.L - l + 1, self.dropout, self.seed, l,
                            self.step_dev)

  def _forward_layer_nodrop(self, l: int):
    nat, ar = self.nat, self.arena
    ell, ks, nh = self._ell(l)
    d = self.dims_in[l - 1]
    relu = l < self.L
    feat = self.feat if l == 1 else None
    nodes = ar.nodes if l == 1 else None
    src_local = None if l == 1 else self.Z[l - 1]
    if self.fused_ok[l]:
      nat.sage_fused(feat, nodes, src_local, d, ar.counters, nh, ell, ks, ar.deg, self.w_packed[l],
                     self.b(l), relu, self.Z[l], self.A[l])
    else:
      if not (l == 1 and self.preaggregate):     # pre-aggregated: _sample already wrote A1 of this arena
        nat.sage_aggregate(feat, nodes, src_local, d, ar.counters, nh, ell, ks, ar.deg, self._A(l))
      # Z = act(A . W^T + b) on wgmma (TMA-fed, bias/ReLU in the register epilogue, rows from the device counter)
      self._plan('fwd', l).run()

  def _forward_loss(self, train: bool = True):
    # labels[nodes[r]] is looked up inside the loss kernel (no gather launch)
    nat, ar = self.nat, self.arena
    boff, n = self._b_off[self.L - 1]
    if train:                      # evaluation must not take part in the cross-rank gradient protocol
      self._begin_grads()
    # the bias gradient of the last layer (column sums of dlogits) is produced by the loss kernel
    nat.softmax_nll(self.Z[self.L], self.C, None, self.labels, ar.nodes, ar.counters, self.loss, self.dPre[self.L],
                    self.correct, self.g32[boff:boff + n], train)

  def _begin_grads(self):
    """Runs before the first kernel that writes into the flat gradient buffer (the loss kernel produces the
    last layer's bias gradient): peers must be done reading last step's gradients, and the split-K weight
    gradient kernels accumulate with red.add, so the buffer starts from zero."""
    if self.peer_group is not None and len(self._peer_groups) == 1:
      self.peer_group.barrier(1)          # peers finished reading last step's gradients
    # one launch zeroes the flat gradient buffer, the loss and the #correct counter; the kernels that accumulate
    # into them then skip their own memsets (memset nodes would cut the programmatic-launch chain of the step)
    self.nat.zero_grads(self.g32, self.loss, self.correct)

  def _plan(self, kind: str, l: int):
    """Cached TcGemm launch for layer l of the current arena / gradient parity (tensor maps are encoded once)."""
    key = (kind, l, self._cur)
    pl = self._tc_plans.get(key)
    if pl is not None:
      return pl
    nat, ar = self.nat, self.arena
    nh = self.L - l + 1                     # counters[nh] = number of target rows of layer l
    pl = nat.TcGemm(self.device.index)
    if kind == 'fwd':
      pl.add_forward(self._A(l), self.W(l), self.b(l), l < self.L, self.Z[l], ar.counters, nh)
    else:
      off, n, k = self._w_off[l - 1]
      gW = self.g32[off:off + n * k].view(n, k)
      # 'bwd': dW (split-K over the batch rows, fp32 red-add) and dA of the same layer share one launch
      pl.add_wgrad(self.dPre[l], self._A(l), gW, ar.counters, nh)
      if l > 1:
        pl.add_dgrad(self.dPre[l], self.W(l), self.dA[l], ar.counters, nh)
    self._tc_plans[key] = pl
    return pl

  def _backward(self):
    # bias gradients are fused into the kernels that produce dPre (loss / sage_gather_bwd)
    for l in range(self.L, 0, -1):
      self._plan('bwd', l).run()
      if l > 1:
        pboff, pn = self._b_off[l - 2]
        self.nat.sage_gather_bwd(self.dA[l], self.dims_in[l - 1], self.arena, self.L - l + 1, self.Z[l - 1],
                                 self.dPre[l - 1], self.g32[pboff:pboff + pn], True, 1.0 / (1.0 - self.dropout))

  def _optimizer(self):
    # Adam's step counter is advanced by the kernel itself (last block to finish)
    if self.peer_group is not None:
      pg = self._peer_groups[self._cur % len(self._peer_groups)]
      pg.barrier(0)                       # every rank finished writing its gradients
      pg.adam(self.p32, self.m, self.v, self.p16, self.lr, 0.9, 0.999, 1e-8, self.wd,
                           self.step_dev, 1.0 / self.world)
    else:
      self.nat.adam_step(self.p32, self.g32, self.m, self.v, self.p16, self.lr, 0.9, 0.999, 1e-8, self.wd,
                         self.step_dev, 1.0 / self.world)
    self._repack()

  def _train(self):
    """Forward, backward and optimizer update of the batch in the current arena."""
    self._forward()
    self._backward()
    self._optimizer()

  def _pipelined_body(self, cur: int):
    """train(batch in arena[cur])  ||  sample(next batch into arena[1-cur])."""
    self._cur = cur
    main = torch.cuda.current_stream()
    self._side.wait_stream(main)                       # fork
    with torch.cuda.stream(self._side):
      self._sample(1 - cur)
    self._train()
    main.wait_stream(self._side)                        # join

  def _step_eager(self):
    if self.pipeline:
      self._pipelined_body(self._cur)
    else:
      self._sample()
      self._train()

  def _autotune(self, iters: int = 5):
    """Pick fused vs unfused per layer from device timings on the current batch."""
    self.autotune_ms = {}
    ar = self.arena
    for l in range(1, self.L + 1):
      if not self.fused_ok[l]:
        continue
      res = {}
      for mode in (True, False):
        self.fused_ok[l] = mode
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        self._forward_layer_nodrop(l)
        e0.record()
        for _ in range(iters):
          self._forward_layer_nodrop(l)
        e1.record()
        e1.synchronize()
        res[mode] = e0.elapsed_time(e1) / iters
      t = torch.tensor([res[True], res[False]], device=self.device)
      if self.world > 1:
        import torch.distributed as dist
        dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)   # same choice on every rank
      self.fused_ok[l] = bool(t[0] <= t[1])
      self.autotune_ms[l] = {'fused': float(t[0]), 'unfused': float(t[1])}

  # ------------------------------------------------------------------ public API
  def warmup_and_capture(self, n_eager: int = 2):
    """Run a few eager steps (lazy inits, GEMM plans), then capture the step into a CUDA graph, one per buffer parity
    in pipelined engines, and set `kernels_per_step` to the kernel, memset and memcpy nodes of the parity-0 graph.
    Engines built with use_cuda_graph=False capture one step only to count it, and keep running eagerly."""
    with torch.cuda.device(self.device):
      saved = self.state_dict()
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        if self.pipeline:
          self._sample(0)
        for _ in range(n_eager):
          self._step_eager()
          if self.pipeline:
            self._cur ^= 1
      torch.cuda.current_stream().wait_stream(side)
      torch.cuda.synchronize()
      if self._autotune_fused:
        self._cur = 0
        self._autotune()
        self._autotune_fused = False
        self._resolve_preagg()
        if self.pipeline:
          self._sample(0)
        self._step_eager()                      # builds the GEMM plans of the chosen variants outside the capture
        torch.cuda.synchronize()
        self._cur = 0
      self.load_state_dict(saved)
      self._cur, self._primed = 0, False
      self._graphs = []
      # programmatic dependent launch helps single-stream chains and costs ~2 % when the sampling and training
      # streams interleave (measured, csrc/cuda/launch_utils.h): captured without it in pipelined mode
      prev_pdl = self.nat.set_pdl(not self.pipeline)
      for parity in range(2 if self.pipeline and self.use_cuda_graph else 1):
        g = torch.cuda.CUDAGraph(keep_graph=True)
        self._cur = parity
        with torch.cuda.graph(g):
          self._step_eager()
        if parity == 0:
          self.kernels_per_step = sum(self.nat.graph_node_counts(g.raw_cuda_graph()))
        if self.use_cuda_graph:
          g.instantiate()
          self._graphs.append(g)
      torch.cuda.synchronize()
      self.nat.set_pdl(prev_pdl)
      self.load_state_dict(saved)
      self._cur, self._primed = 0, False
      self._graph_fb = self._graphs[0] if self._graphs else None

  def close(self):
    """Drop the captured graphs (call before destroying the process group)."""
    torch.cuda.synchronize(self.device)
    self._graphs = []
    self._graph_fb = None

  def _run_captured_or_eager(self, parity: int):
    if self._graphs:
      self._graphs[parity].replay()
    else:
      self._cur = parity
      self._step_eager()

  def _stage_seeds(self, buf: torch.Tensor, seeds: torch.Tensor):
    n = seeds.numel()
    assert n <= self.bs
    if n < self.bs:
      buf.fill_(-1)
    buf[:n].copy_(seeds, non_blocking=True)

  def train_step(self, seeds: torch.Tensor) -> Optional[torch.Tensor]:
    """One training step on a batch of seed node ids.  `seeds` may be a (pinned) host
    tensor -- it is copied H2D asynchronously -- or a device tensor.  Returns the device
    scalar holding the mean NLL loss (read it with .item() / a D2H copy).

    Pipelined engines run *sample(this batch) || train(previous batch)*: the first call only
    samples (returns None), later calls return the loss of the batch passed one call earlier;
    `flush()` trains the last pending batch."""
    self._health_tick()
    if not self.pipeline:
      with nvtx_range('glt.engine.step'):
        self._stage_seeds(self._seeds[0], seeds)
        self._run_captured_or_eager(0)
      self.step_idx += 1
      return self.loss
    if not self._primed:
      self._cur = 0
      self._stage_seeds(self._seeds[0], seeds)
      self._sample(0)
      self._primed = True
      return None if self.step_idx == 0 and self.regrow_count == 0 else self.loss
    cur = self._cur
    with nvtx_range('glt.engine.step(sample b+1 || train b)'):
      self._stage_seeds(self._seeds[1 - cur], seeds)
      self._run_captured_or_eager(cur)
    self._cur = 1 - cur
    self.step_idx += 1
    return self.loss

  def flush(self) -> Optional[torch.Tensor]:
    """Pipelined mode: train the batch that was sampled by the last train_step() call."""
    if not self.pipeline or not self._primed:
      return None
    self._train()
    self._primed = False
    self.step_idx += 1
    return self.loss

  def profile_sections(self, seeds: torch.Tensor, iters: int = 10):
    """Device time (ms) of each stage of an *eager, unpipelined* step (CUDA events; the other
    ranks run the same sequence so the peer barriers inside are matched).  Diagnostic only.  With pre-aggregation
    (`preaggregate_layer1`) 'sample' includes the layer-1 aggregation and 'forward_l1' is its GEMM alone."""
    names = ['sample', 'forward_l1', 'forward_rest', 'backward', 'optimizer']
    acc = {n: 0.0 for n in names}
    self._cur = 0
    # `seeds` may hold several batches ([n_batches, batch]): rotating them keeps the feature rows
    # of every iteration cold in L2, like a real epoch
    batches = seeds if seeds.dim() == 2 else seeds.unsqueeze(0)
    for it in range(iters + 2):
      self._stage_seeds(self._seeds[0], batches[it % batches.shape[0]])
      ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
      ev[0].record()
      self._sample(0); ev[1].record()
      self._forward_layer(1); ev[2].record()
      for l in range(2, self.L + 1):
        self._forward_layer(l)
      self._forward_loss(); ev[3].record()
      self._backward(); ev[4].record()
      self._optimizer(); ev[5].record()
      torch.cuda.synchronize()
      if it >= 2:
        for i, n in enumerate(names):
          acc[n] += ev[i].elapsed_time(ev[i + 1]) / iters
    return acc

  def profile_kernels(self, seeds: torch.Tensor, iters: int = 10, queue_ahead_cycles: int = 6_000_000):
    """Device time (us) of EVERY launch of an eager, unpipelined step, in launch order: -> [(name, us)].
    Each native call is bracketed by CUDA events; a spin kernel at the head of the step lets the host queue the
    whole step ahead of the GPU, so an interval is the kernel's own run time with the previous kernel's data still
    in L2 (what `ncu`, which replays each kernel with cold caches, cannot show).  Diagnostic only."""
    eng = self
    log = []

    class _Timed(object):
      def __init__(self, obj, prefix=''):
        object.__setattr__(self, '_o', obj)
        object.__setattr__(self, '_p', prefix)

      def __getattr__(self, name):
        f = getattr(self._o, name)
        if name == 'TcGemm':
          return lambda *a, **k: _Timed(f(*a, **k), name + '.')
        if not callable(f) or name.startswith('_') or isinstance(f, type) or name in ('set_pdl',):
          return f

        def call(*a, **k):
          e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
          e0.record()
          r = f(*a, **k)
          e1.record()
          log.append((self._p + name, e0, e1))
          return r
        return call

    real_nat, real_plans, real_pgs = self.nat, self._tc_plans, self._peer_groups
    batches = seeds if seeds.dim() == 2 else seeds.unsqueeze(0)
    acc, names = None, None
    try:
      self.nat, self._tc_plans = _Timed(real_nat), {}
      self._peer_groups = [_Timed(pg, 'PeerGroup.') for pg in real_pgs]
      if real_pgs:
        self.peer_group = self._peer_groups[0]
      self._cur = 0
      for it in range(iters + 2):
        del log[:]
        self._stage_seeds(self._seeds[0], batches[it % batches.shape[0]])
        torch.cuda._sleep(int(queue_ahead_cycles))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ar = self._arenas[0]
        ar.sample(self.gh, self._seeds[0], None, self.seed, 0, False, False, True, len(self._arenas))
        e1.record()
        log.append(('arena.sample (all sampling kernels)', e0, e1))
        if self.preaggregate:
          # a pipelined step runs it on the sampling stream, outside the training chain
          self._aggregate_layer1(0)
          log[-1] = ('sage_aggregate (layer 1, sampling stream)',) + log[-1][1:]
        self._train()
        torch.cuda.synchronize()
        if it >= 2:
          if acc is None:
            names, acc = [n for n, _, _ in log], [0.0] * len(log)
          if len(log) == len(acc):
            for i, (_, a0, a1) in enumerate(log):
              acc[i] += a0.elapsed_time(a1) * 1e3 / iters
    finally:
      self.nat, self._tc_plans, self._peer_groups = real_nat, real_plans, real_pgs
      if real_pgs:
        self.peer_group = real_pgs[0]
    return list(zip(names, acc))

  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    """(loss, #correct, #seeds) for a batch without updating parameters."""
    assert not (self.pipeline and self._primed), 'call flush() before evaluate_batch()'
    n = seeds.numel()
    self.seeds_dev.fill_(-1)
    self.seeds_dev[:n].copy_(seeds)
    self._sample()
    self._forward(train=False)
    return float(self.loss.item()), int(self.correct.item()), int(self.arena.counters[1].item())

  def _project_first(self, l: int) -> bool:
    """Layer l >= 2 projects before it aggregates when it narrows the width: the neighbour rows it gathers are then
    dims_out wide instead of dims_in (DESIGN.md, "SURVEY §7.4 hard parts", row 2).  Layer 1 always aggregates first:
    its rows come from the feature table in place."""
    return l >= 2 and self.dims_out[l - 1] < self.dims_in[l - 1]

  @torch.no_grad()
  def inference(self, chunk_rows: Optional[int] = None) -> torch.Tensor:
    """Exact layer-wise full-neighbourhood inference: bf16 logits [num_nodes, num_classes] of every node.

    Every layer aggregates each node's complete CSR row (the `fanout >= degree` limit of training; what the
    reference's examples evaluate with, `SAGE.inference` over `sizes=[-1]`).  Aggregate-first layers run
    `sage_full_aggregate` (concat) over chunks of `chunk_rows` nodes into an A chunk, then the TcGemm forward of the
    layer; project-first layers run one TcGemm over the whole table, P = H . [W_neigh ; W_self]^T, then
    `sage_full_aggregate` (combine).  Uses the bf16 parameters of the training forward, applies no dropout, and runs
    on the current stream, so it sees every step queued before it.  The activation tables live for the call only;
    arenas, captured graphs, gradients and optimizer state are not touched.  `chunk_rows=None` sizes the chunk from
    free device memory.  The result is bitwise identical for any chunk size.

    Not collective: with several GPUs every rank maps all shards and reads peer rows in place."""
    nat, dev, bf = self.nat, self.device, torch.bfloat16
    N, L = self._num_nodes, self.L
    with torch.cuda.device(dev):
      wide = max(self.dims_out)
      bufs = [torch.empty(N, wide, dtype=bf, device=dev) for _ in range(2 if L > 1 else 1)]
      agg_dims = [self.dims_in[l - 1] for l in range(1, L + 1) if not self._project_first(l)]
      a_row = 2 * max(agg_dims)
      chunk_rows = infer_chunk_rows(chunk_rows, N, a_row * 2, dev)
      A = torch.empty(chunk_rows, a_row, dtype=bf, device=dev)
      rows_dev = torch.tensor([chunk_rows, N], dtype=torch.int32, device=dev)   # TcGemm row counts (device-side)
      H = None
      for l in range(1, L + 1):
        out = bufs[(l - 1) % len(bufs)][:, :self.dims_out[l - 1]]
        self._infer_layer(l, H, out, A, rows_dev, chunk_rows)
        H = out
      return H[:, :self.C].contiguous()

  def _infer_layer(self, l: int, H: Optional[torch.Tensor], out: torch.Tensor, A: torch.Tensor,
                   rows_dev: torch.Tensor, chunk_rows: int):
    """out = layer l of the full-neighbourhood forward over every node; H = the layer's input table (None: features)."""
    nat, N = self.nat, self._num_nodes
    d, n = self.dims_in[l - 1], self.dims_out[l - 1]
    relu = l < self.L
    if self._project_first(l):
      W = self.W(l)
      P = torch.empty(N, 2 * n, dtype=torch.bfloat16, device=self.device)
      infer_gemm(nat, H, torch.cat([W[:, :d], W[:, d:]], 0), None, False, P, rows_dev, 1)
      for r0, r1 in infer_chunks(N, chunk_rows):
        nat.sage_full_aggregate(self.gh, None, P, 0, n, n, r0, r1, True, self.b(l), relu, out[r0:r1])
      return
    for r0, r1 in infer_chunks(N, chunk_rows):
      a = A[:r1 - r0, :2 * d]
      nat.sage_full_aggregate(self.gh, self.feat if l == 1 else None, H, 0, 0, d, r0, r1, False, None, False, a)
      infer_gemm(nat, a, self.W(l), self.b(l), relu, out[r0:r1], rows_dev, 0)
