"""KgeEngine: device-resident knowledge-graph embedding training (PyG's `torch_geometric.nn.kge`: TransE, DistMult,
ComplEx, RotatE) and filtered link ranking over all entities.

Per step, on the device (csrc/cuda/kge.cu; the counters and SparseAdam are skipgram.cu's):

  m2v_begin        advance the device step counters [next step, Adam step, current step]
  kge_negatives    num_negatives corrupted ids per positive: head for the first half of the batch, tail for the rest
  kge_loss_grad    margin ranking (TransE, DistMult) or BCE-with-logits (ComplEx, RotatE) loss and its gradient into
                   fp32 gradient rows; marks the entity and relation rows it looked up
  kge_sparse_adam  torch.optim.SparseAdam on the marked rows of the entity table, then of the relation table

No step reads anything back to the host, so the step is captured into one CUDA graph.
"""
import math
from typing import Optional, Tuple

import torch

from ..ops import require_native

MODELS = {'transe': 0, 'distmult': 1, 'complex': 2, 'rotate': 3}
_COMPLEX = ('complex', 'rotate')


def kge_filter(triples: torch.Tensor, num_nodes: int, num_relations: int) -> Tuple[torch.Tensor, torch.Tensor]:
  """Filter keys of known triples (int64 [3, m] = head, relation, tail), for `KgeEngine.rank` / `test`.

  Returns two sorted int64 [m] tensors on the triples' device: (h R + r) N + t for tail queries and (t R + r) N + h
  for head queries, so the known answers of a query (h, r, ?) are one contiguous, id-sorted range of the first.
  Duplicate triples are kept.  Needs N^2 R < 2^63."""
  N, R = int(num_nodes), int(num_relations)
  if N < 1 or R < 1:
    raise ValueError(f'num_nodes and num_relations must be >= 1 (got {N}, {R})')
  if N * N * R >= 2 ** 63:
    raise ValueError(f'num_nodes^2 * num_relations = {N * N * R} does not fit the int64 keys (< 2^63)')
  triples = torch.as_tensor(triples)
  if triples.dtype != torch.int64 or triples.dim() != 2 or triples.size(0) != 3:
    raise ValueError('triples must be int64 [3, m] (head, relation, tail)')
  h, r, t = triples[0], triples[1], triples[2]
  if triples.numel() and (int(h.min()) < 0 or int(t.min()) < 0 or int(r.min()) < 0 or int(h.max()) >= N
                          or int(t.max()) >= N or int(r.max()) >= R):
    raise ValueError('triple ids out of range')
  tail = torch.sort((h * R + r) * N + t).values
  head = torch.sort((t * R + r) * N + h).values
  return tail, head


class KgeEngine:
  """Knowledge-graph embeddings of N entities and R relations (PyG's `KGEModel` family), trained on the device.

  Args:
    num_nodes, num_relations: N and R, each in [1, 2^31).
    model: 'transe', 'distmult', 'complex' or 'rotate'.
    hidden_channels: D, a multiple of 8 in [8, 512].  ComplEx and RotatE entity rows, and ComplEx relation rows,
      hold a real and an imaginary part of D each.
    margin: the margin of the TransE / DistMult ranking loss and RotatE's score offset; None is 1.0 as in PyG
      (ComplEx has no margin).
    p_norm: TransE's norm, 1 or 2.
    num_negatives: K >= 1 corrupted triples per positive.  K = 1 is PyG's `random_sample`.
    batch_size: positives per step (fewer may be given).
    lr: SparseAdam learning rate (betas 0.9 / 0.999, eps 1e-8, no weight decay).  PyG's example runs dense Adam;
      this engine updates only the rows a step looked up, as `torch.optim.SparseAdam` would.
    seed: initialisation (a CPU `torch.Generator`, following PyG's `reset_parameters`) and the Philox negatives.

  Scores: TransE -||n(h) + r - n(t)||_p with n = F.normalize; DistMult sum h r t; ComplEx Re(sum h r conj(t));
  RotatE margin - ||h e^{iθ} - t||.  Loss: TransE and DistMult sum max(0, margin - s_i + s_ij) / (n K); ComplEx and
  RotatE (sum softplus(-s_i) + sum softplus(s_ij)) / (n + n K).  Positive i of a step's n corrupts its head when
  i < n // 2 and its tail otherwise, with ids drawn uniformly from [0, N) (not filtered, as in PyG).  A training
  triple with an id out of range is skipped.  After a step, `negatives` (int64 [batch_size, K]) holds the drawn ids
  of the first n rows.  `_sample`, `_loss_grad` and `_update` are the step's three stages.
  """

  def __init__(self, num_nodes: int, num_relations: int, model: str = 'transe', hidden_channels: int = 128,
               margin: Optional[float] = None, p_norm: float = 1.0, num_negatives: int = 1, batch_size: int = 1024,
               lr: float = 0.01, seed: int = 0, device: Optional[torch.device] = None, use_cuda_graph: bool = True):
    if model not in MODELS:
      raise ValueError(f'model must be one of {sorted(MODELS)} (got {model!r})')
    N, R, D, K, B = (int(x) for x in (num_nodes, num_relations, hidden_channels, num_negatives, batch_size))
    if not 1 <= N < 2 ** 31 or not 1 <= R < 2 ** 31:
      raise ValueError(f'num_nodes and num_relations must be in [1, 2^31) (got {num_nodes}, {num_relations})')
    if D % 8 != 0 or not 8 <= D <= 512:
      raise ValueError(f'hidden_channels must be a multiple of 8 in [8, 512] (got {hidden_channels})')
    if float(p_norm) not in (1.0, 2.0):
      raise ValueError(f'p_norm must be 1 or 2 (got {p_norm})')
    if K < 1 or B < 1:
      raise ValueError(f'num_negatives and batch_size must be >= 1 (got {num_negatives}, {batch_size})')
    if B * K >= 2 ** 31:
      raise ValueError('batch_size * num_negatives must be < 2^31')
    if not lr > 0:
      raise ValueError(f'lr must be > 0 (got {lr})')
    margin = 1.0 if margin is None else float(margin)
    if not math.isfinite(margin):
      raise ValueError(f'margin must be finite (got {margin})')

    self.nat = require_native()
    self.device = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    if self.device.index is None:
      self.device = torch.device('cuda', torch.cuda.current_device())
    self.model, self.model_id = model, MODELS[model]
    self.num_nodes, self.num_relations, self.hidden_channels = N, R, D
    self.margin, self.p_norm = margin, int(p_norm)
    self.num_negatives, self.batch_size = K, B
    self.lr, self.seed, self.use_cuda_graph = float(lr), int(seed), bool(use_cuda_graph)
    self.betas, self.eps = (0.9, 0.999), 1e-8
    pe = 2 if model in _COMPLEX else 1
    pr = 2 if model == 'complex' else 1
    dev = self.device
    with torch.cuda.device(dev):
      self.ent = torch.empty(N, pe * D, dtype=torch.float32, device=dev)
      self.rel = torch.empty(R, pr * D, dtype=torch.float32, device=dev)
      self._init_tables()
      self.grad_ent, self.grad_rel = torch.zeros_like(self.ent), torch.zeros_like(self.rel)
      self.exp_avg_ent, self.exp_avg_sq_ent = torch.zeros_like(self.ent), torch.zeros_like(self.ent)
      self.exp_avg_rel, self.exp_avg_sq_rel = torch.zeros_like(self.rel), torch.zeros_like(self.rel)
      self.touched_ent = torch.zeros(N, dtype=torch.uint8, device=dev)
      self.touched_rel = torch.zeros(R, dtype=torch.uint8, device=dev)
      self.state = torch.zeros(3, dtype=torch.int32, device=dev)   # [next step, Adam step, current step]
      self.trip = torch.zeros(3, B, dtype=torch.int64, device=dev)
      self.count = torch.zeros(1, dtype=torch.int32, device=dev)
      self.negatives = torch.full((B, K), -1, dtype=torch.int64, device=dev)
      self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self._graph = None
    self.kernels_per_step = None

  def _init_tables(self):
    """PyG's reset_parameters, drawn from a CPU generator in PyG's order."""
    gen = torch.Generator().manual_seed(self.seed)
    N, R, D = self.num_nodes, self.num_relations, self.hidden_channels

    def xavier(rows):
      w = torch.empty(rows, D)
      torch.nn.init.xavier_uniform_(w, generator=gen)
      return w

    if self.model == 'transe':
      bound = 6.0 / math.sqrt(D)
      ent = torch.empty(N, D).uniform_(-bound, bound, generator=gen)
      rel = torch.empty(R, D).uniform_(-bound, bound, generator=gen)
      rel = torch.nn.functional.normalize(rel, p=self.p_norm, dim=-1)
    elif self.model == 'distmult':
      ent, rel = xavier(N), xavier(R)
    elif self.model == 'complex':
      ent_re, ent_im, rel_re, rel_im = xavier(N), xavier(N), xavier(R), xavier(R)
      ent, rel = torch.cat([ent_re, ent_im], 1), torch.cat([rel_re, rel_im], 1)
    else:
      ent_re, ent_im = xavier(N), xavier(N)
      rel = torch.empty(R, D).uniform_(0, 2 * math.pi, generator=gen)
      ent = torch.cat([ent_re, ent_im], 1)
    self.ent.copy_(ent)
    self.rel.copy_(rel)

  # ------------------------------------------------------------------ step stages
  def _sample(self):
    self.nat.m2v_begin(self.state)
    self.nat.kge_negatives(self.count, self.batch_size, self.num_negatives, self.num_nodes, self.seed,
                           self.state[2:3], self.negatives)

  def _loss_grad(self):
    self.nat.kge_loss_grad(self.model_id, self.trip, self.count, self.negatives, self.ent, self.rel, self.margin,
                           self.p_norm, self.grad_ent, self.grad_rel, self.touched_ent, self.touched_rel, self.loss)

  def _update(self):
    b1, b2 = self.betas
    t = self.state[1:2]
    self.nat.kge_sparse_adam(self.ent, self.grad_ent, self.exp_avg_ent, self.exp_avg_sq_ent, self.touched_ent, t,
                             self.lr, b1, b2, self.eps)
    self.nat.kge_sparse_adam(self.rel, self.grad_rel, self.exp_avg_rel, self.exp_avg_sq_rel, self.touched_rel, t,
                             self.lr, b1, b2, self.eps)

  def _step(self):
    self._sample()
    self._loss_grad()
    self._update()

  # ------------------------------------------------------------------ training
  def warmup_and_capture(self):
    """Load the step's kernels with one step on an empty batch (no row is touched; the step counters are restored),
    then capture negatives, loss / gradient and SparseAdam into one CUDA graph.  `kernels_per_step` is the captured
    graph's node count."""
    with torch.cuda.device(self.device):
      saved = self.state.clone()
      self.count.zero_()
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        self._step()
      torch.cuda.current_stream().wait_stream(side)
      self.state.copy_(saved)
      torch.cuda.synchronize()
      self._graph = None
      g = torch.cuda.CUDAGraph(keep_graph=True)
      with torch.cuda.graph(g):
        self._step()
      self.kernels_per_step = sum(self.nat.graph_node_counts(g.raw_cuda_graph()))
      if self.use_cuda_graph:
        g.instantiate()
        self._graph = g
      torch.cuda.synchronize()

  def _stage(self, triples: torch.Tensor):
    triples = torch.as_tensor(triples)
    if triples.dtype != torch.int64 or triples.dim() != 2 or triples.size(0) != 3:
      raise ValueError('triples must be int64 [3, n] (head, relation, tail)')
    n = triples.size(1)
    if n > self.batch_size:
      raise ValueError(f'{n} triples in a batch of {self.batch_size}')
    if n:
      self.trip[:, :n].copy_(triples, non_blocking=True)
    self.count.fill_(n)

  def train_step(self, triples: torch.Tensor) -> torch.Tensor:
    """One step on up to batch_size triples (int64 [3, n], pinned host or device); returns the device loss scalar."""
    with torch.cuda.device(self.device):
      self._stage(triples)
      if self._graph is not None:
        self._graph.replay()
      else:
        self._step()
    return self.loss[0]

  # ------------------------------------------------------------------ evaluation
  def _ids(self, h, r, t):
    return [torch.as_tensor(x).to(self.device, torch.int64).reshape(-1).contiguous() for x in (h, r, t)]

  def score(self, h, r, t) -> torch.Tensor:
    """fp32 [n] scores of the triples (h[i], r[i], t[i]), forward only."""
    h, r, t = self._ids(h, r, t)
    with torch.cuda.device(self.device):
      return self.nat.kge_score(self.model_id, self.ent, self.rel, h, r, t, self.margin, self.p_norm)

  def rank(self, h, r, t, mode: str = 'tail', filter: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
           _splits: int = 0) -> torch.Tensor:
    """float64 [n] rank of the true tail (mode 'tail') or head ('head') among all N entities:
    1 + #{c : s_c > s_true} + #{c : s_c = s_true} / 2 over the entities c other than the true one and, with a
    `kge_filter` result, other than every c that forms a known triple with the query."""
    if mode not in ('tail', 'head'):
      raise ValueError(f"mode must be 'tail' or 'head' (got {mode!r})")
    h, r, t = self._ids(h, r, t)
    keys = None
    if filter is not None:
      keys = filter[0 if mode == 'tail' else 1].to(self.device, torch.int64).contiguous()
    with torch.cuda.device(self.device):
      return self.nat.kge_rank(self.model_id, self.ent, self.rel, h, r, t, mode == 'tail', keys, self.margin,
                               self.p_norm, int(_splits))

  def test(self, h, r, t, k: int = 10, filter: Optional[Tuple[torch.Tensor, torch.Tensor]] = None,
           mode: str = 'both') -> Tuple[float, float, float]:
    """(mean rank, mean reciprocal rank, Hits@k) over the triples, in one direction or averaged over both."""
    if mode not in ('tail', 'head', 'both'):
      raise ValueError(f"mode must be 'tail', 'head' or 'both' (got {mode!r})")
    modes = ('tail', 'head') if mode == 'both' else (mode,)
    ranks = torch.cat([self.rank(h, r, t, m, filter) for m in modes])
    if ranks.numel() == 0:
      return float('nan'), float('nan'), float('nan')
    return float(ranks.mean()), float((1.0 / ranks).mean()), float((ranks <= k).double().mean())

  # ------------------------------------------------------------------ checkpoints
  def _model_tensors(self):
    D = self.hidden_channels
    out = {'node_emb.weight': self.ent[:, :D], 'rel_emb.weight': self.rel[:, :D]}
    if self.model in _COMPLEX:
      out['node_emb_im.weight'] = self.ent[:, D:]
    if self.model == 'complex':
      out['rel_emb_im.weight'] = self.rel[:, D:]
    return out

  def state_dict(self) -> dict:
    """`sd['model']` holds the tables under PyG's parameter names; optimizer state and step counters sit beside it."""
    return {'model': {k: v.clone() for k, v in self._model_tensors().items()},
            'exp_avg_ent': self.exp_avg_ent.clone(), 'exp_avg_sq_ent': self.exp_avg_sq_ent.clone(),
            'exp_avg_rel': self.exp_avg_rel.clone(), 'exp_avg_sq_rel': self.exp_avg_sq_rel.clone(),
            'adam_step': int(self.state[1]), 'step': int(self.state[0])}

  def load_state_dict(self, sd: dict):
    """Copies in place, so a captured graph keeps running on the loaded state."""
    with torch.cuda.device(self.device):
      dst = self._model_tensors()
      if set(sd['model']) != set(dst):
        raise ValueError(f"model tensors must be {sorted(dst)} (got {sorted(sd['model'])})")
      for k, v in dst.items():
        if tuple(sd['model'][k].shape) != tuple(v.shape):
          raise ValueError(f'{k} must be {list(v.shape)} (got {list(sd["model"][k].shape)})')
        v.copy_(sd['model'][k])
      for k in ('exp_avg_ent', 'exp_avg_sq_ent', 'exp_avg_rel', 'exp_avg_sq_rel'):
        getattr(self, k).copy_(sd[k])
      self.state.copy_(torch.tensor([sd['step'], sd['adam_step'], 0], dtype=torch.int32))
      self.grad_ent.zero_()
      self.grad_rel.zero_()
      self.touched_ent.zero_()
      self.touched_rel.zero_()
