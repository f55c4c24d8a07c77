"""SealEngine: a device-resident SEAL link-prediction training step (the reference's examples/seal_link_pred.py model).

Per step, on the device, one CTA per link (csrc/cuda/seal.cu):

  seal extract    the num_hops enclosing subgraph of (s, d), its induced edges without s -> d and d -> s, and DRNL labels
  seal forward    the reference's DGCNN: GCNConv stack with tanh, sort-pool, Conv1d / MaxPool1d / Conv1d, MLP, BCE
  seal backward   the gradient of the link's loss term into a per-link row of partials
  seal reduce     gradient = the valid links' partials summed in link order
  adam            torch.optim.Adam over the flat fp32 parameter vector

No step reads anything back to the host and every sum has a fixed order, so the step is captured into one CUDA graph
and a replay equals an eager step bitwise.
"""
import math
from typing import Optional, Sequence, Union

import torch

from ..ops import require_native


class SealEngine:
  """SEAL (Zhang & Chen, 2018) with the reference's DGCNN, trained by one captured step per batch of links.

  Args:
    graph: a device `data.Graph` (mode 'CUDA' or 'ZERO_COPY') in CSR by source.  SEAL expects it symmetric.
    num_nodes: node count N; a link with an id outside [0, N), an id of -1, or s == d is padding.
    num_hops: hops of the enclosing subgraph (1 to 4), expanded over CSR rows from {s, d}.
    num_neighbors: None for full rows on every hop (the reference), or one cap per hop: a frontier node keeps a
      uniform subset of at most that many row entries, drawn without replacement (Floyd), keyed by Philox on
      (seed, device step, link, node).  A cap <= 0 takes the full row.
    max_nodes, max_edges: per-link capacities of the static arena (max_nodes in [2, 1024]).  max_edges=None takes
      1.5x the largest edge count of the calibration links' subgraphs.  A subgraph over a capacity keeps the first
      max_nodes nodes in discovery order (s, d, then hop by hop, frontier order, row order) and the first max_edges
      edges in (source local id, row position) order; each link so truncated adds 1 to `truncated()`.
    hidden, num_layers: num_layers GCNConv(hidden) layers and one GCNConv(1), each followed by tanh.
    sort_k: an int >= 10, or a float in (0, 1): the reference's percentile rule max(10, sizes[ceil(k n) - 1]) over
      the node counts of the calibration links' subgraphs.
    max_z: the largest DRNL label (input features are one_hot(z, max_z + 1)); None takes the largest label seen on the
      calibration links.  Labels above it are clamped.
    dropout: dropout probability after the MLP's first layer, in [0, 1).
    Shared memory bounds hidden and sort_k further: the per-link kernels hold a [hidden, hidden] weight stage, per-node
    vectors of max_nodes and sort-pool / conv buffers of about 49 * sort_k floats in one CTA, and construction raises
    ValueError when that exceeds the device's opt-in limit per block.  On an H100 (232,448 bytes), computed from the
    kernels' formula (seal_smem in seal.cu): hidden <= 238 at max_nodes=256 and <= 235 at max_nodes=1024 (sort_k 10);
    with num_layers <= 4, sort_k <= 1,123 at hidden 32 and <= 841 at hidden 128 (max_nodes=256), <= 1,091 and <= 809
    at max_nodes=1024.
    batch_size: links per step; fewer are padded.  lr: Adam learning rate (betas 0.9 / 0.999, eps 1e-8).
    calibration_links: int64 [2, n] links (typically the training links); needed when max_edges, max_z or a
      percentile sort_k must be calibrated.  This is the construction's only host read.
    seed: parameter initialisation (PyG's: glorot weights and zero biases for GCNConv, torch defaults for Conv1d and
      Linear, from a CPU generator) and the Philox draws of neighbour subsets and dropout.

  DRNL: ds = distance to s with d deleted, dd = distance to d with s deleted, over the subgraph's edges taken as
  undirected; z = 1 + min(ds, dd) + (D // 2) (D // 2 + D % 2 - 1) with D = ds + dd, z[s] = z[d] = 1, z = 0 where a
  distance is infinite.  GCNConv normalises as PyG: A + I with each input self-loop replaced by the added one, degrees
  on the destination.  Sort-pool keeps the k nodes with the largest last channel (ties to the lower local id) and pads
  with zero rows.  The loss is the mean BCE-with-logits over the batch's valid links.

  After a step, `mask` (fp32 [batch_size, 128]) holds the dropout scale of each MLP unit (0 or 1 / (1 - p)).
  """

  def __init__(self, graph, num_nodes: int, num_hops: int = 2, num_neighbors: Optional[Sequence[int]] = None,
               max_nodes: int = 256, max_edges: Optional[int] = None, hidden: int = 32, num_layers: int = 3,
               sort_k: Union[int, float] = 0.6, max_z: Optional[int] = None, dropout: float = 0.5,
               batch_size: int = 256, lr: float = 1e-4, calibration_links: Optional[torch.Tensor] = None,
               seed: int = 0, device: Optional[torch.device] = None, use_cuda_graph: bool = True):
    if getattr(graph, 'mode', 'CPU') == 'CPU':
      raise ValueError('graph must be a device graph (mode CUDA or ZERO_COPY)')
    N, hops, B = int(num_nodes), int(num_hops), int(batch_size)
    if N < 1:
      raise ValueError(f'num_nodes must be >= 1 (got {num_nodes})')
    if not 1 <= hops <= 4:
      raise ValueError(f'num_hops must be in [1, 4] (got {num_hops})')
    if num_neighbors is None:
      caps = [-1] * hops
    else:
      caps = [int(c) for c in num_neighbors]
      if len(caps) != hops:
        raise ValueError(f'num_neighbors needs one cap per hop ({hops}), got {len(caps)}')
    if not 2 <= int(max_nodes) <= 1024:
      raise ValueError(f'max_nodes must be in [2, 1024] (got {max_nodes})')
    if any(c > int(max_nodes) for c in caps):
      raise ValueError(f'a neighbour cap exceeds max_nodes ({max_nodes})')
    if max_edges is not None and not 1 <= int(max_edges) <= 2 ** 24:
      raise ValueError(f'max_edges must be in [1, 2^24] (got {max_edges})')
    if not 1 <= int(hidden) <= 256:
      raise ValueError(f'hidden must be in [1, 256], and shared memory bounds it further (got {hidden})')
    if not 1 <= int(num_layers) <= 8:
      raise ValueError(f'num_layers must be in [1, 8] (got {num_layers})')
    if isinstance(sort_k, bool) or not isinstance(sort_k, (int, float)):
      raise ValueError(f'sort_k must be an int >= 10 or a float in (0, 1) (got {sort_k!r})')
    if isinstance(sort_k, int) and not 10 <= sort_k <= 2048:
      raise ValueError(f'an int sort_k must be in [10, 2048], and shared memory bounds it further (got {sort_k})')
    if isinstance(sort_k, float) and not 0.0 < sort_k < 1.0:
      raise ValueError(f'a float sort_k must be in (0, 1) (got {sort_k})')
    if max_z is not None and not 1 <= int(max_z) < 2 ** 20:
      raise ValueError(f'max_z must be in [1, 2^20) (got {max_z})')
    if not 0.0 <= float(dropout) < 1.0:
      raise ValueError(f'dropout must be in [0, 1) (got {dropout})')
    if B < 1:
      raise ValueError(f'batch_size must be >= 1 (got {batch_size})')
    if not float(lr) > 0:
      raise ValueError(f'lr must be > 0 (got {lr})')
    needs_cal = max_edges is None or max_z is None or isinstance(sort_k, float)
    if needs_cal:
      if calibration_links is None:
        raise ValueError('calibration_links are needed to calibrate max_edges, max_z or a percentile sort_k')
      calibration_links = torch.as_tensor(calibration_links)
      if calibration_links.dim() != 2 or calibration_links.shape[0] != 2 or calibration_links.shape[1] == 0:
        raise ValueError('calibration_links must be a non-empty [2, n] tensor of node ids')

    self.nat = require_native()
    self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if self.device.index is None:
      self.device = torch.device('cuda', torch.cuda.current_device())
    self.graph, self.num_nodes, self.num_hops, self.caps = graph, N, hops, caps
    self.num_neighbors = None if num_neighbors is None else list(caps)
    self.max_nodes, self.hidden, self.num_layers = int(max_nodes), int(hidden), int(num_layers)
    self.dropout, self.batch_size, self.lr, self.seed = float(dropout), B, float(lr), int(seed)
    self.use_cuda_graph = bool(use_cuda_graph)
    self.cap_max = max(max(caps), 0)
    dev = self.device
    with torch.cuda.device(dev):
      self._handle = graph.graph_handler
      # state = [Adam steps taken, Adam's block ticket]; state[0] also keys the step's neighbour and dropout draws
      self.state = torch.zeros(2, dtype=torch.int32, device=dev)
      self.trunc = torch.zeros(1, dtype=torch.int32, device=dev)
      if needs_cal:
        sizes, zmax, emax = self._calibrate(calibration_links.to(torch.int64), max_edges)
        if not sizes:
          raise ValueError('calibration_links hold no valid link')
      if max_edges is None:
        max_edges = min(2 ** 24, max(64, int(math.ceil(1.5 * emax))))
      if max_z is None:
        max_z = max(1, zmax)
      if isinstance(sort_k, float):
        sizes = sorted(sizes)
        sort_k = max(10, sizes[int(math.ceil(sort_k * len(sizes))) - 1])
      self.max_edges, self.max_z, self.k = int(max_edges), int(max_z), int(sort_k)
      try:
        self.arena = self.nat.SealArena(dev.index, B, self.max_nodes, self.max_edges, self.hidden, self.num_layers,
                                        self.max_z + 1, self.k, self.cap_max)
      except RuntimeError as e:
        raise ValueError(str(e)) from None
      self.layout = [(name, off, tuple(shape)) for name, off, shape in self.arena.layout]
      self.num_params = self.arena.num_params
      self.params = self._init_params().to(dev)
      self.grad = torch.zeros_like(self.params)
      self.exp_avg = torch.zeros_like(self.params)
      self.exp_avg_sq = torch.zeros_like(self.params)
      self.links = torch.full((2, B), -1, dtype=torch.int64, device=dev)
      self.labels = torch.zeros(B, dtype=torch.float32, device=dev)
      self._pred_links = torch.full((2, B), -1, dtype=torch.int64, device=dev)
      self._pred_labels = torch.zeros(B, dtype=torch.float32, device=dev)
      self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self.mask = self.arena.mask
    self._graph = None

  def _calibrate(self, links: torch.Tensor, max_edges: Optional[int]):
    """Node counts, the largest DRNL label and the largest edge count of the links' subgraphs (unclamped)."""
    B, dev = self.batch_size, self.device
    trunc = torch.zeros(1, dtype=torch.int32, device=dev)
    buf = torch.full((2, B), -1, dtype=torch.int64, device=dev)
    links = links.to(dev)

    def run(arena):
      metas, zmax = [], 0
      for i in range(0, links.shape[1], B):
        chunk = links[:, i:i + B]
        buf.fill_(-1)
        buf[:, :chunk.shape[1]].copy_(chunk)
        arena.extract(self._handle, buf, self.num_nodes, self.num_hops, self.caps, self.seed, self.state, -1, trunc)
        meta = arena.meta[:chunk.shape[1]]
        valid = meta[:, 2] == 1
        inside = torch.arange(self.max_nodes, device=dev)[None, :] < meta[:, :1]
        zmax = max(zmax, int((arena.z[:chunk.shape[1]] * inside)[valid].max()) if bool(valid.any()) else 0)
        metas.append(meta[valid].clone())
      return torch.cat(metas).cpu(), zmax

    if max_edges is None:   # edge counts first (a 1-edge arena still counts them), then labels at that capacity
      meta, _ = run(self.nat.SealArena(dev.index, B, self.max_nodes, 1, 1, 1, 2, 10, self.cap_max))
      max_edges = max(1, int(meta[:, 4].max())) if meta.shape[0] else 1
    meta, zmax = run(self.nat.SealArena(dev.index, B, self.max_nodes, int(max_edges), 1, 1, 2, 10, self.cap_max))
    emax = int(meta[:, 4].max()) if meta.shape[0] else 0
    return meta[:, 0].tolist(), zmax, emax

  def _init_params(self) -> torch.Tensor:
    gen = torch.Generator().manual_seed(self.seed)
    flat = torch.zeros(self.num_params)
    fan_in = {}
    for name, off, shape in self.layout:
      n = math.prod(shape)
      if name.startswith('convs.'):
        if name.endswith('lin.weight'):          # glorot
          a = math.sqrt(6.0 / (shape[0] + shape[1]))
          flat[off:off + n] = torch.empty(n).uniform_(-a, a, generator=gen)
        continue                                 # GCNConv bias: zeros
      if name.endswith('weight'):                # torch default: kaiming_uniform(a=sqrt(5)) = U(+-1/sqrt(fan_in))
        fan_in[name[:-len('weight')]] = math.prod(shape[1:])
      bound = 1.0 / math.sqrt(fan_in[name.rsplit('.', 1)[0] + '.'])
      flat[off:off + n] = torch.empty(n).uniform_(-bound, bound, generator=gen)
    return flat

  # ------------------------------------------------------------------ step stages
  def _extract(self, links: torch.Tensor, graph=None):
    handle = self._handle if graph is None else graph.graph_handler
    self.arena.extract(handle, links, self.num_nodes, self.num_hops, self.caps, self.seed, self.state, self.max_z,
                       self.trunc)

  def _forward(self, labels: torch.Tensor, training: bool):
    self.arena.forward(self.params, labels, training, self.dropout, self.seed, self.state)

  def _backward(self):
    self.arena.backward(self.params)
    self.arena.reduce(self.grad, self.loss)

  def _update(self):
    self.nat.adam_step(self.params, self.grad, self.exp_avg, self.exp_avg_sq, None, self.lr, 0.9, 0.999, 1e-8, 0.0,
                       self.state, 1.0)

  def _step(self):
    self._extract(self.links)
    self._forward(self.labels, True)
    self._backward()
    self._update()

  # ------------------------------------------------------------------ public API
  def warmup_and_capture(self):
    """Load the step's kernels with one step on padding links (parameters, moments and counters are restored), then
    capture extract, forward, backward, reduce and Adam into one CUDA graph."""
    with torch.cuda.device(self.device):
      saved = [t.clone() for t in (self.state, self.trunc, self.params, self.exp_avg, self.exp_avg_sq)]
      self.links.fill_(-1)
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        self._step()
      torch.cuda.current_stream().wait_stream(side)
      for t, s in zip((self.state, self.trunc, self.params, self.exp_avg, self.exp_avg_sq), saved):
        t.copy_(s)
      torch.cuda.synchronize()
      self._graph = None
      if not self.use_cuda_graph:
        return
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        self._step()
      torch.cuda.synchronize()
      self._graph = g

  def _stage(self, links: torch.Tensor, dst: torch.Tensor, labels=None, lab_dst=None) -> int:
    links = torch.as_tensor(links)
    if links.dtype != torch.int64 or links.dim() != 2 or links.shape[0] != 2:
      raise ValueError(f'links must be int64 [2, n] (got {links.dtype} {tuple(links.shape)})')
    n = links.shape[1]
    if n > self.batch_size:
      raise ValueError(f'{n} links in a batch of {self.batch_size}')
    if n < self.batch_size:
      dst.fill_(-1)
    dst[:, :n].copy_(links, non_blocking=True)
    if labels is not None:
      labels = torch.as_tensor(labels).reshape(-1)
      if labels.numel() != n:
        raise ValueError(f'{labels.numel()} labels for {n} links')
      if n < self.batch_size:
        lab_dst.zero_()
      lab_dst[:n].copy_(labels, non_blocking=True)
    return n

  def train_step(self, links: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """One step on up to batch_size links (int64 [2, n]) with labels (float or bool [n]), pinned host or device;
    returns the device loss scalar."""
    with torch.cuda.device(self.device):
      self._stage(links, self.links, labels, self.labels)
      if self._graph is not None:
        self._graph.replay()
      else:
        self._step()
    return self.loss[0]

  @torch.no_grad()
  def predict(self, links: torch.Tensor, graph=None) -> torch.Tensor:
    """fp32 [n] logits of the links, without dropout; `graph` scores them on another device graph (val / test)."""
    links = torch.as_tensor(links)
    out = []
    with torch.cuda.device(self.device):
      for i in range(0, links.shape[1], self.batch_size):
        n = self._stage(links[:, i:i + self.batch_size], self._pred_links)
        self._extract(self._pred_links, graph)
        self._forward(self._pred_labels, False)
        out.append(self.arena.logits[:n].clone())
    if not out:
      return torch.zeros(0, dtype=torch.float32, device=self.device)
    return torch.cat(out)

  def truncated(self) -> int:
    """Links whose subgraph hit max_nodes or max_edges, over every step and prediction so far (reads the device)."""
    return int(self.trunc[0])

  def parameters_dict(self) -> dict:
    """{reference parameter name: view into the flat fp32 parameter vector}."""
    return {name: self.params[off:off + math.prod(shape)].view(shape) for name, off, shape in self.layout}

  def state_dict(self) -> dict:
    """'model': the reference DGCNN's parameter names and shapes (loads into it); 'optimizer': Adam's flat moments
    and step count."""
    return {'model': {k: v.clone() for k, v in self.parameters_dict().items()},
            'optimizer': {'exp_avg': self.exp_avg.clone(), 'exp_avg_sq': self.exp_avg_sq.clone(),
                          'step': int(self.state[0])}}

  def load_state_dict(self, sd: dict):
    """Copies in place, so a captured graph keeps running on the loaded state."""
    with torch.cuda.device(self.device):
      model = sd['model']
      for name, off, shape in self.layout:
        if name not in model:
          raise ValueError(f'state_dict has no {name!r}')
        w = torch.as_tensor(model[name])
        if tuple(w.shape) != shape:
          raise ValueError(f'{name} must be {list(shape)} (got {list(w.shape)})')
        self.params[off:off + math.prod(shape)].copy_(w.reshape(-1))
      opt = sd['optimizer']
      self.exp_avg.copy_(opt['exp_avg'])
      self.exp_avg_sq.copy_(opt['exp_avg_sq'])
      self.state.copy_(torch.tensor([int(opt['step']), 0], dtype=torch.int32))
