"""MetaPath2VecEngine: device-resident metapath2vec / DeepWalk skip-gram training.

The reference trains its featureless ogbn-mag node types on PyG's `MetaPath2Vec`; this engine learns the same kind of
embeddings with the project's sm_90a kernels (csrc/cuda/skipgram.cu).  Per step, on the device:

  m2v_begin        advance the device step counters (walk step, Adam step)
  metapath_walk    walks_per_node walks per start node along the metapath, -1 after a dead end
                   (node2vec_walk instead for node2vec's p / q walks)
  sgns_negatives   num_negative_samples negative windows per valid window
  sgns_loss_grad   SGNS loss and its gradient into fp32 gradient rows; marks the rows it looked up
  sparse_adam      torch.optim.SparseAdam on the marked rows, then clears their gradients and marks

No step reads anything back to the host, so the step is captured into one CUDA graph.
"""
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from ..ops import require_native

EdgeType = Tuple[str, str, str]


class MetaPath2VecEngine:
  """Skip-gram embeddings of the node types on a metapath (PyG `MetaPath2Vec`'s loss), one table per type.

  Args:
    graphs: {edge type (src, rel, dst): data.Graph} in CSR by source (rows = source ids, columns = destination ids),
      on the engine's device (mode 'CUDA' or 'ZERO_COPY').
    num_nodes: {node type: count} for every type on the metapath.
    metapath: up to 8 relations that chain (the destination of one is the source of the next); when walk_length
      exceeds their number the path must also close (the last destination is the first source).  A homogeneous
      graph with metapath [('n', 'to', 'n')] trains DeepWalk (node2vec with p = q = 1).
    p, q: node2vec's return and in-out parameters (default 1, 1: uniform walks).  Other values need a metapath of one
      relation from a type to itself, finite p, q > 0 and max(1, 1/p, 1/q) / min(1, 1/p, 1/q) <= 64.
    embedding_dim: a multiple of 8 in [8, 512].
    walk_length, context_size, walks_per_node, num_negative_samples: as PyG's `MetaPath2Vec`
      (2 <= context_size <= walk_length + 1).
    batch_size: start nodes per step (type metapath[0][0]); fewer starts are padded with -1.
    lr: SparseAdam learning rate (betas 0.9 / 0.999, eps 1e-8).
    seed: initialisation (N(0, 1) as `nn.Embedding`, from a CPU generator) and the Philox draws of walks and negatives.

  Walk i of a step starts at starts[i // walks_per_node]; step s moves to a uniform random neighbour in relation
  metapath[(s - 1) % R].  A node without a neighbour in the next relation ends the walk (-1 after it), and a window
  of context_size consecutive positions counts only when all its entries are nodes.  Loss, over valid windows:
    pos = -mean log(sigmoid(h_centre . h_ctx) + 1e-15),  neg = -mean log(1 - sigmoid(h_centre . h_neg) + 1e-15)
  A negative window keeps its positive window's centre and draws every context position uniformly from that
  position's node type (standard SGNS).  PyG instead slices independent random walks for its negatives, whose
  centres are random too.

  With p, q != 1 the walks are node2vec's second-order walks (PyG `Node2Vec(..., p=p, q=q)`): step 1 is uniform; at
  step s >= 2, at v coming from t, an entry x of v's row weighs 1/p if x == t, 1 if the graph holds the edge (t, x)
  and 1/q otherwise.  It is drawn by exact rejection sampling (propose uniformly from v's row, accept with probability
  weight / max(1, 1/p, 1/q)), as torch_cluster does; after 4096 rejected proposals the last one is taken, which at
  the ratio bound of 64 happens with probability < 1e-28 per walk step.  The edge test binary-searches t's row, so
  every CSR row must be column-sorted: graphs built through `Topology` are; shards handed to `Graph.from_shards` must
  be too.  A dead end ends the walk with -1 as above, where torch_cluster's walker instead stays on an isolated node.

  After a step, `walks` (int64 [batch_size * walks_per_node, walk_length + 1]) and `negatives` (int64
  [walks * windows * num_negative_samples, context_size], window-major, all -1 for an invalid window) hold what the
  step used.  `_sample`, `_loss_grad` and `_update` are the step's three stages, for inspection between them.
  """

  def __init__(self, graphs: Dict[EdgeType, object], num_nodes: Dict[str, int], metapath: Sequence[EdgeType],
               embedding_dim: int = 128, walk_length: int = 64, context_size: int = 7, walks_per_node: int = 5,
               num_negative_samples: int = 5, batch_size: int = 128, lr: float = 0.01, seed: int = 0,
               device: Optional[torch.device] = None, use_cuda_graph: bool = True, p: float = 1.0, q: float = 1.0):
    metapath = [tuple(e) for e in metapath]
    R = len(metapath)
    if not 1 <= R <= 8:
      raise ValueError(f'metapath needs 1 to 8 relations (got {R})')
    for e in metapath:
      if len(e) != 3:
        raise ValueError(f'metapath entries are (src, rel, dst) edge types (got {e})')
      if e not in graphs:
        raise ValueError(f'no graph for metapath relation {e}')
    for a, b in zip(metapath[:-1], metapath[1:]):
      if a[2] != b[0]:
        raise ValueError(f'metapath does not chain: {a} ends at {a[2]!r}, {b} starts at {b[0]!r}')
    if walk_length > R and metapath[-1][2] != metapath[0][0]:
      raise ValueError(f'walk_length {walk_length} > {R} relations needs a closed metapath '
                       f'({metapath[-1][2]!r} != {metapath[0][0]!r})')
    D, L, C, W, K, B = (int(x) for x in (embedding_dim, walk_length, context_size, walks_per_node,
                                         num_negative_samples, batch_size))
    if D % 8 != 0 or not 8 <= D <= 512:
      raise ValueError(f'embedding_dim must be a multiple of 8 in [8, 512] (got {embedding_dim})')
    if L < 1:
      raise ValueError(f'walk_length must be >= 1 (got {walk_length})')
    if not 2 <= C <= L + 1:
      raise ValueError(f'context_size must be in [2, walk_length + 1 = {L + 1}] (got {context_size})')
    if W < 1 or K < 1 or B < 1:
      raise ValueError('walks_per_node, num_negative_samples and batch_size must be >= 1')
    if not lr > 0:
      raise ValueError(f'lr must be > 0 (got {lr})')
    p, q = float(p), float(q)
    if not (math.isfinite(p) and math.isfinite(q) and p > 0 and q > 0):
      raise ValueError(f'p and q must be finite and > 0 (got p={p}, q={q})')
    ws = (1.0, 1.0 / p, 1.0 / q)
    if max(ws) / min(ws) > 64:
      raise ValueError(f'max(1, 1/p, 1/q) / min(1, 1/p, 1/q) must be <= 64 (got p={p}, q={q})')
    if (p, q) != (1.0, 1.0) and (R != 1 or metapath[0][0] != metapath[0][2]):
      raise ValueError('p and q other than 1 need a metapath of one relation from a node type to itself')
    slot_types = [metapath[0][0]] + [e[2] for e in metapath]
    for t in slot_types:
      if t not in num_nodes or not 1 <= int(num_nodes[t]) < 2 ** 32:
        raise ValueError(f'num_nodes needs a count in [1, 2^32) for node type {t!r}')
    for e in metapath:
      g = graphs[e]
      if getattr(g, 'mode', 'CPU') == 'CPU':
        raise ValueError(f'graph {e} must be a device graph (mode CUDA or ZERO_COPY)')

    self.nat = require_native()
    self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if self.device.index is None:
      self.device = torch.device('cuda', torch.cuda.current_device())
    self.metapath, self.R = metapath, R
    self.embedding_dim, self.walk_length, self.context_size = D, L, C
    self.walks_per_node, self.num_negative_samples, self.batch_size = W, K, B
    self.lr, self.seed, self.use_cuda_graph = float(lr), int(seed), bool(use_cuda_graph)
    self.p, self.q = p, q
    self.betas, self.eps = (0.9, 0.999), 1e-8
    # one table per node type, concatenated in order of first appearance on the path
    self.node_types: List[str] = list(dict.fromkeys(slot_types))
    self.num_nodes = {t: int(num_nodes[t]) for t in self.node_types}
    self.offsets, off = {}, 0
    for t in self.node_types:
      self.offsets[t] = off
      off += self.num_nodes[t]
    self.rows = off
    dev = self.device
    with torch.cuda.device(dev):
      handles = [graphs[e].graph_handler for e in metapath]
      self._graphs = [graphs[e] for e in metapath]
      self.mp = self.nat.MetaPath(dev.index, handles, [self.offsets[t] for t in slot_types],
                                  [self.num_nodes[t] for t in slot_types])
      gen = torch.Generator().manual_seed(self.seed)
      self.weight = torch.empty(self.rows, D, dtype=torch.float32, device=dev)
      for t in self.node_types:
        o, n = self.offsets[t], self.num_nodes[t]
        self.weight[o:o + n].copy_(torch.randn(n, D, generator=gen))
      self.grad = torch.zeros_like(self.weight)
      self.exp_avg = torch.zeros_like(self.weight)
      self.exp_avg_sq = torch.zeros_like(self.weight)
      self.touched = torch.zeros(self.rows, dtype=torch.uint8, device=dev)
      self.state = torch.zeros(3, dtype=torch.int32, device=dev)   # [next walk step, Adam step, current walk step]
      self.starts = torch.full((B,), -1, dtype=torch.int64, device=dev)
      self.n_walks = B * W
      self.windows_per_walk = L + 2 - C
      self.walks = torch.full((self.n_walks, L + 1), -1, dtype=torch.int64, device=dev)
      self.negatives = torch.full((self.n_walks * self.windows_per_walk * K, C), -1, dtype=torch.int64, device=dev)
      self.n_valid = torch.zeros(1, dtype=torch.int32, device=dev)
      self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self._graph = None

  # ------------------------------------------------------------------ step stages
  def _sample(self):
    nat, cur = self.nat, self.state[2:3]
    nat.m2v_begin(self.state)
    if (self.p, self.q) == (1.0, 1.0):
      nat.metapath_walk(self.mp, self.starts, self.walks_per_node, self.context_size, self.seed, cur, self.walks,
                        self.n_valid)
    else:
      nat.node2vec_walk(self.mp, self.starts, self.walks_per_node, self.context_size, self.seed, cur, self.walks,
                        self.n_valid, self.p, self.q)
    nat.sgns_negatives(self.mp, self.walks, self.context_size, self.num_negative_samples, self.seed, cur,
                       self.negatives)

  def _loss_grad(self):
    self.nat.sgns_loss_grad(self.mp, self.walks, self.negatives, self.context_size, self.num_negative_samples,
                            self.weight, self.n_valid, self.grad, self.touched, self.loss)

  def _update(self):
    self.nat.sparse_adam(self.mp, self.weight, self.grad, self.exp_avg, self.exp_avg_sq, self.touched,
                         self.state[1:2], self.lr, self.betas[0], self.betas[1], self.eps)

  def _step(self):
    self._sample()
    self._loss_grad()
    self._update()

  # ------------------------------------------------------------------ public API
  def warmup_and_capture(self):
    """Load the step's kernels with one step on padding starts (no row is touched; the step counters are restored),
    then capture walk, negatives, loss / gradient and SparseAdam into one CUDA graph."""
    with torch.cuda.device(self.device):
      saved = self.state.clone()
      self.starts.fill_(-1)
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        self._step()
      torch.cuda.current_stream().wait_stream(side)
      self.state.copy_(saved)
      torch.cuda.synchronize()
      self._graph = None
      if not self.use_cuda_graph:
        return
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        self._step()
      torch.cuda.synchronize()
      self._graph = g

  def _stage(self, starts: torch.Tensor):
    starts = torch.as_tensor(starts).reshape(-1)
    if starts.dtype != torch.int64:
      raise ValueError(f'starts must be int64 node ids (got {starts.dtype})')
    n = starts.numel()
    if n > self.batch_size:
      raise ValueError(f'{n} start nodes in a batch of {self.batch_size}')
    if n < self.batch_size:
      self.starts.fill_(-1)
    self.starts[:n].copy_(starts, non_blocking=True)

  def train_step(self, starts: torch.Tensor) -> torch.Tensor:
    """One step on up to batch_size start nodes (int64, pinned host or device); returns the device loss scalar."""
    with torch.cuda.device(self.device):
      self._stage(starts)
      if self._graph is not None:
        self._graph.replay()
      else:
        self._step()
    return self.loss[0]

  def embedding(self, node_type: str) -> torch.Tensor:
    """fp32 [num_nodes[node_type], embedding_dim] copy of the type's table."""
    o = self.offsets[node_type]
    return self.weight[o:o + self.num_nodes[node_type]].clone()

  def state_dict(self) -> dict:
    return {'weight': {t: self.embedding(t) for t in self.node_types},
            'exp_avg': self.exp_avg.clone(), 'exp_avg_sq': self.exp_avg_sq.clone(),
            'adam_step': int(self.state[1]), 'walk_step': int(self.state[0])}

  def load_state_dict(self, sd: dict):
    """Copies in place, so a captured graph keeps running on the loaded state."""
    with torch.cuda.device(self.device):
      for t in self.node_types:
        o, n = self.offsets[t], self.num_nodes[t]
        w = sd['weight'][t]
        if tuple(w.shape) != (n, self.embedding_dim):
          raise ValueError(f'weight[{t!r}] must be [{n}, {self.embedding_dim}] (got {tuple(w.shape)})')
        self.weight[o:o + n].copy_(w)
      self.exp_avg.copy_(sd['exp_avg'])
      self.exp_avg_sq.copy_(sd['exp_avg_sq'])
      self.state.copy_(torch.tensor([sd['walk_step'], sd['adam_step'], 0], dtype=torch.int32))
      self.grad.zero_()
      self.touched.zero_()
