"""`GraphSageTrainer` / `GraphSageMultiLabelTrainer` / `GraphSageLinkTrainer`: the device-agnostic counterparts of
`GraphSageEngine` / `GraphSageMultiLabelEngine` / `GraphSageLinkEngine`.

Same step-level API (`train_step(seeds)`, `evaluate_batch(seeds)`, `state_dict()` / `load_state_dict()`), built
from the public pieces -- `NeighborSampler`, `Feature`, the eager `GraphSAGE` module and `torch.optim.Adam` -- so it
runs on a CPU as well as on any GPU.  Two uses:

* code that must run without an H100 (CI, notebooks) keeps the engine's call pattern and switches class;
* it is the *semantic reference* of the fused engine: same sampler stream, same model family, autograd backward.

(The reference has no engine; its examples hand-write this loop, e.g. examples/train_sage_ogbn_products.py:61-110.)
"""
from typing import List, Optional

import torch
import torch.nn.functional as F

from ..sampler import EdgeSamplerInput, NegativeSampling, NeighborSampler, NodeSamplerInput
from .sage import GraphSAGE
from .sage_multilabel import check_multilabel


@torch.no_grad()
def _layerwise_inference(model: GraphSAGE, graph, features, device, chunk_rows: int) -> torch.Tensor:
  """Every node's output of the eager `model`, layer by layer over complete CSR rows, `chunk_rows` targets at a time."""
  model.eval()
  topo = graph.topo
  if topo is None:
    raise ValueError('inference() needs the graph topology (a Graph built from a Topology)')
  indptr, indices = topo.indptr.to(device), topo.indices.to(device)
  n = indptr.numel() - 1
  ids = torch.arange(n)
  x = features[ids] if not isinstance(features, torch.Tensor) else features[:n]
  x = x.to(device, dtype=torch.float32)
  convs = model.convs
  for i, conv in enumerate(convs):
    out = torch.empty(n, conv.lin_l.out_features, device=device)
    for r0 in range(0, n, chunk_rows):
      r1 = min(n, r0 + chunk_rows)
      e0, e1 = int(indptr[r0]), int(indptr[r1])
      deg = indptr[r0 + 1:r1 + 1] - indptr[r0:r1]
      dst = torch.repeat_interleave(torch.arange(r1 - r0, device=device), deg)
      out[r0:r1] = conv((x, x[r0:r1]), torch.stack([indices[e0:e1].long(), dst]), r1 - r0)
    x = torch.relu(out) if i < len(convs) - 1 else out
  return x


class GraphSageTrainer(object):
  def __init__(self, graph, features, labels: torch.Tensor, in_dim: int, fanouts: List[int] = (15, 10, 5),
               hidden: int = 256, num_classes: int = 47, lr: float = 3e-3, weight_decay: float = 0.0, seed: int = 0,
               device: Optional[torch.device] = None):
    self.device = torch.device(device) if device is not None else torch.device('cpu')
    self.graph = graph
    self.features, self.labels = features, labels.to(self.device)
    self.fanouts = list(fanouts)
    self.sampler = NeighborSampler(graph, self.fanouts, device=self.device, seed=seed)
    torch.manual_seed(seed)
    self.model = GraphSAGE(in_dim, hidden, num_classes, len(self.fanouts)).to(self.device)
    self.opt = torch.optim.Adam(self.model.parameters(), lr=lr, weight_decay=weight_decay)
    self.step_idx = 0
    self.loss = torch.zeros((), device=self.device)

  def _batch(self, seeds: torch.Tensor):
    out = self.sampler.sample_from_nodes(NodeSamplerInput(node=seeds.to(self.sampler.device)))
    x = self.features[out.node] if not isinstance(self.features, torch.Tensor) else self.features[out.node.cpu()]
    x = x.to(self.device, dtype=torch.float32)
    edge_index = torch.stack([out.row, out.col]).to(self.device)
    n_seed = out.batch.numel() if out.batch is not None else seeds.numel()
    y = self.labels[out.node[:n_seed].to(self.device)]
    return x, edge_index, out.num_sampled_nodes, out.num_sampled_edges, y, n_seed

  def train_step(self, seeds: torch.Tensor) -> torch.Tensor:
    """One optimisation step on a batch of seed ids; returns the (device) mean NLL loss."""
    self.model.train()
    x, ei, nn_, ne_, y, n = self._batch(seeds)
    logits = self.model(x, ei, nn_, ne_)[:n]
    loss = self._loss(logits, y)
    self.opt.zero_grad(set_to_none=True)
    loss.backward()
    self.opt.step()
    self.step_idx += 1
    self.loss = loss.detach()
    return self.loss

  def _loss(self, logits: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return F.cross_entropy(logits, y)

  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    """(loss, #correct, #seeds) without updating parameters -- same tuple as GraphSageEngine.evaluate_batch."""
    self.model.eval()
    x, ei, nn_, ne_, y, n = self._batch(seeds)
    logits = self.model(x, ei, nn_, ne_)[:n]
    return float(F.cross_entropy(logits, y)), int((logits.argmax(1) == y).sum()), int(n)

  @torch.no_grad()
  def inference(self, chunk_rows: int = 65536) -> torch.Tensor:
    """Exact layer-wise full-neighbourhood inference: fp32 logits [num_nodes, num_classes] of every node, computed
    layer by layer with the model's `SAGEConv`s over every node's complete CSR row, `chunk_rows` target nodes at a
    time -- the same result as `GraphSageEngine.inference()` (which rounds to bf16 where the engine stores bf16)."""
    return _layerwise_inference(self.model, self.graph, self.features, self.device, chunk_rows)

  def flush(self):          # API compatibility with the pipelined engine
    return None

  def close(self):
    return None

  def state_dict(self):
    s = {'model': self.model.state_dict(), 'optimizer': self.opt.state_dict(), 'step': self.step_idx}
    if hasattr(self.sampler, 'state_dict'):
      s['sampler'] = self.sampler.state_dict()
    return s

  def load_state_dict(self, s):
    self.model.load_state_dict(s['model'])
    self.opt.load_state_dict(s['optimizer'])
    self.step_idx = int(s.get('step', 0))
    if 'sampler' in s and hasattr(self.sampler, 'load_state_dict'):
      self.sampler.load_state_dict(s['sampler'])


class GraphSageMultiLabelTrainer(GraphSageTrainer):
  """Device-agnostic counterpart of `GraphSageMultiLabelEngine` (same step-level API): `labels` is a [N, T] tensor of
  0/1 values, the loss the mean `F.binary_cross_entropy_with_logits` over the batch's seeds and tasks.  Runs on a CPU as
  well as on any GPU, and is the semantic reference of the engine."""

  def __init__(self, graph, features, labels: torch.Tensor, in_dim: int, fanouts: List[int] = (15, 10, 5),
               hidden: int = 256, lr: float = 3e-3, weight_decay: float = 0.0, seed: int = 0,
               device: Optional[torch.device] = None):
    T = check_multilabel(labels)
    super().__init__(graph, features, labels.float(), in_dim, fanouts=fanouts, hidden=hidden, num_classes=T, lr=lr,
                     weight_decay=weight_decay, seed=seed, device=device)

  def _loss(self, logits: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    return F.binary_cross_entropy_with_logits(logits, y)

  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    """(loss, TP, FP, FN, #seeds) without updating parameters, as GraphSageMultiLabelEngine.evaluate_batch."""
    self.model.eval()
    x, ei, nn_, ne_, y, n = self._batch(seeds)
    logits = self.model(x, ei, nn_, ne_)[:n]
    pred, yb = logits > 0, y.bool()
    return (float(self._loss(logits, y)), int((pred & yb).sum()), int((pred & ~yb).sum()), int((~pred & yb).sum()),
            int(n))


class GraphSageLinkTrainer(object):
  """Device-agnostic counterpart of `GraphSageLinkEngine` (same step-level API): `NeighborSampler.sample_from_edges`
  with binary negatives, the eager `GraphSAGE`, mean BCE-with-logits on the dot products of the `edge_label_index`
  pairs, and `torch.optim.Adam`.  Runs on a CPU as well as on any GPU, and is the semantic reference of the engine."""

  def __init__(self, graph, features, in_dim: int, fanouts: List[int] = (15, 10, 5), hidden: int = 256,
               out_channels: int = 256, neg_ratio: int = 1, lr: float = 3e-3, weight_decay: float = 0.0,
               seed: int = 0, device: Optional[torch.device] = None):
    self.device = torch.device(device) if device is not None else torch.device('cpu')
    self.graph, self.features = graph, features
    self.fanouts = list(fanouts)
    self.neg_sampling = NegativeSampling('binary', int(neg_ratio))
    self.sampler = NeighborSampler(graph, self.fanouts, device=self.device, with_neg=True, seed=seed)
    torch.manual_seed(seed)
    self.model = GraphSAGE(in_dim, hidden, out_channels, len(self.fanouts)).to(self.device)
    self.opt = torch.optim.Adam(self.model.parameters(), lr=lr, weight_decay=weight_decay)
    self.step_idx = 0
    self.loss = torch.zeros((), device=self.device)

  def _logits(self, pairs: torch.Tensor):
    """(logits, labels) of the batch's positive pairs followed by their sampled negatives."""
    pairs = pairs.to(self.sampler.device, dtype=torch.int64)
    out = self.sampler.sample_from_edges(EdgeSamplerInput(pairs[0], pairs[1], neg_sampling=self.neg_sampling))
    x = self.features[out.node] if not isinstance(self.features, torch.Tensor) else self.features[out.node.cpu()]
    x = x.to(self.device, dtype=torch.float32)
    edge_index = torch.stack([out.row, out.col]).to(self.device)
    h = self.model(x, edge_index, out.num_sampled_nodes, out.num_sampled_edges)
    eli = out.metadata['edge_label_index'].to(self.device)
    logits = (h[eli[0]] * h[eli[1]]).sum(-1)
    return logits, out.metadata['edge_label'].to(self.device, dtype=torch.float32)

  def train_step(self, pairs: torch.Tensor) -> torch.Tensor:
    """One optimisation step on int64 [2, n] positive pairs; returns the (device) mean BCE loss."""
    self.model.train()
    logits, y = self._logits(pairs)
    loss = F.binary_cross_entropy_with_logits(logits, y)
    self.opt.zero_grad(set_to_none=True)
    loss.backward()
    self.opt.step()
    self.step_idx += 1
    self.loss = loss.detach()
    return self.loss

  @torch.no_grad()
  def evaluate_batch(self, pairs: torch.Tensor):
    """(loss, #correct, #pairs) without updating parameters -- same tuple as GraphSageLinkEngine.evaluate_batch."""
    self.model.eval()
    logits, y = self._logits(pairs)
    return (float(F.binary_cross_entropy_with_logits(logits, y)), int(((logits > 0).float() == y).sum()),
            int(y.numel()))

  @torch.no_grad()
  def inference(self, chunk_rows: int = 65536) -> torch.Tensor:
    """fp32 embeddings [num_nodes, out_channels] of every node by exact layer-wise full-neighbourhood inference."""
    return _layerwise_inference(self.model, self.graph, self.features, self.device, chunk_rows)

  def flush(self):          # API compatibility with the pipelined engine
    return None

  def close(self):
    return None

  def state_dict(self):
    return {'model': self.model.state_dict(), 'optimizer': self.opt.state_dict(), 'step': self.step_idx,
            'sampler': self.sampler.state_dict()}

  def load_state_dict(self, s):
    self.model.load_state_dict(s['model'])
    self.opt.load_state_dict(s['optimizer'])
    self.step_idx = int(s.get('step', 0))
    if 'sampler' in s:
      self.sampler.load_state_dict(s['sampler'])
