"""GraphSageLinkEngine: the CUDA-graphed GraphSAGE training step for link prediction.

A `GraphSageEngine` whose batch is a set of positive node pairs instead of seed nodes, and whose loss is binary
cross-entropy on the dot products of the pair endpoints' last-layer embeddings (the unsupervised GraphSAGE of the
reference's `graph_sage_unsup_ppi.py` / `LinkNeighborLoader` with binary negatives).  Per step, on the device:

  k_link_seeds   positives [2, B] -> seeds [2P], P = (1 + k) B: the positives, then k uniform strict negatives per
                 positive drawn in-graph (csrc/cuda/link.cu)
  arena.sample   the same sampler as the node engine; its ordered seed dedup gives every pair position its local id
  layers 1..L    inherited (fused or unfused layer 1, dropout, bf16 / MXFP8 features)
  k_link_bce     loss, #correct and the fp32 embedding gradient of every valid pair
  cast           dPre[L] = bf16(dZ) + last-layer bias gradient (relu_bwd_cast without the ReLU mask)
  backward, Adam inherited

No step reads anything back to the host, so the step is captured into one CUDA graph like the node engine's.
"""
from typing import List, Optional

import torch

from .sage import GraphSageEngine


def link_auc(emb: torch.Tensor, pos: torch.Tensor, neg: torch.Tensor) -> float:
  """ROC AUC of dot-product link scores: positive pairs `pos` [2, n] against negative pairs `neg` [2, m] (rank
  statistic, tied scores get their mean rank)."""
  emb = emb.float()
  s = torch.cat([(emb[pos[0]] * emb[pos[1]]).sum(-1), (emb[neg[0]] * emb[neg[1]]).sum(-1)])
  _, inv, cnt = torch.unique(s, return_inverse=True, return_counts=True)
  mean_rank = cnt.cumsum(0).double() - (cnt.double() - 1) / 2          # 1-based mean rank of each distinct score
  r = mean_rank[inv]
  n_pos, n_neg = pos.shape[1], neg.shape[1]
  return float((r[:n_pos].sum() - n_pos * (n_pos + 1) / 2) / (n_pos * n_neg))


class GraphSageLinkEngine(GraphSageEngine):
  """Static-shape, CUDA-graph-captured GraphSAGE link-prediction step (binary negatives, mean BCE-with-logits).

  Args:
    graph, feature_table, in_dim, num_nodes, fanouts, hidden: as `GraphSageEngine`.
    batch_size: positive pairs per step (B).  The sampler arena holds 2 (1 + neg_ratio) B seeds.
    out_channels: embedding width, a multiple of 8 up to 512 (stored padded to 64 columns that stay zero).
    neg_ratio: negatives per positive (k >= 1).  Negative j of positive i is a uniform node pair redrawn up to 5 times
      while it is an edge of `graph`, keyed by (seed, arena step, pair position): a checkpoint's `sample_step`
      reproduces them.
    calibration_pairs: optional int64 [2, M] pairs; their endpoints plus uniform node ids for the negatives form the
      node pool that sizes the arena (`calibration_seeds` of the base class).
    **engine_kwargs: every other `GraphSageEngine` option (lr, seed, device, use_fused, use_cuda_graph, pipeline,
      dropout, feature_format, ...).

  `train_step(pairs)` takes int64 [2, n <= batch_size] pairs (host, pinned or device) and returns the device loss
  scalar; `evaluate_batch(pairs)` returns (loss, #correct, #pairs) with negatives drawn as in training;
  `inference()` returns the bf16 [num_nodes, out_channels] embeddings (the last layer has no ReLU).
  """

  def __init__(self, graph, feature_table, in_dim: int, num_nodes: int, fanouts: List[int] = (15, 10, 5),
               batch_size: int = 1024, hidden: int = 256, out_channels: int = 256, neg_ratio: int = 1,
               calibration_pairs: Optional[torch.Tensor] = None, **engine_kwargs):
    k, C, B = int(neg_ratio), int(out_channels), int(batch_size)
    if k < 1:
      raise ValueError(f'neg_ratio must be an integer >= 1 (got {neg_ratio})')
    if C % 8 != 0 or not 8 <= C <= 512:
      raise ValueError(f'out_channels must be a multiple of 8 in [8, 512] (got {out_channels})')
    self.pos_bs, self.neg_ratio, self.P = B, k, (1 + k) * B
    pool = None
    if calibration_pairs is not None:
      pairs = calibration_pairs.reshape(2, -1).cpu().to(torch.int64)
      g = torch.Generator(device='cpu')
      g.manual_seed(int(engine_kwargs.get('seed', 0)) + 29)
      pool = torch.cat([pairs.flatten(), torch.randint(0, int(num_nodes), (2 * k * pairs.shape[1],), generator=g)])
    # layer 1 aggregates inside the forward here (pre-aggregation on the sampling stream is a node-engine feature)
    engine_kwargs.setdefault('preaggregate_layer1', False)
    super().__init__(graph, feature_table, torch.zeros(1, dtype=torch.int64), in_dim, num_nodes, fanouts=fanouts,
                     batch_size=2 * self.P, hidden=hidden, num_classes=C, calibration_seeds=pool, **engine_kwargs)
    dev = self.device
    with torch.cuda.device(dev):
      # staged positives per arena (pipelined engines sample the next batch while this one trains); zeros, like the
      # base class's seed buffers, so that warm-up steps run on a real (tiny) batch
      self._pos = [torch.zeros(2, B, dtype=torch.int64, device=dev) for _ in self._seeds]
      self._n_pairs = [torch.zeros(1, dtype=torch.int32, device=dev) for _ in self._seeds]
      self._dZ32 = torch.zeros(2 * self.P, self.n_out_pad, dtype=torch.float32, device=dev)

  def _stage_seeds(self, buf: torch.Tensor, pairs: torch.Tensor):
    pos = next(p for s, p in zip(self._seeds, self._pos) if s is buf)
    if pairs.dim() != 2 or pairs.shape[0] != 2:
      raise ValueError(f'pairs must be [2, n] (got {tuple(pairs.shape)})')
    n = pairs.shape[1]
    if n > self.pos_bs:
      raise ValueError(f'{n} pairs in a batch of {self.pos_bs}')
    if n < self.pos_bs:
      pos.fill_(-1)
    pos[:, :n].copy_(pairs, non_blocking=True)

  def _sample(self, which: Optional[int] = None):
    which = self._cur if which is None else which
    ar = self._arenas[which]
    # reads ar.step before the arena's first kernel advances it (same stream)
    self.nat.link_seeds(self.gh, self._pos[which], self._num_nodes, self.neg_ratio, self.seed, ar.step,
                        self._seeds[which], self._n_pairs[which])
    super()._sample(which)

  def _forward_loss(self, train: bool = True):
    nat, ar, L = self.nat, self.arena, self.L
    if train:
      self._begin_grads()
      nat.zero_rows(self._dZ32, ar.counters, 1)
    else:
      self.loss.zero_()
      self.correct.zero_()
    nat.link_bce(self.Z[L], self.C, ar.seed_local, self.P, self.pos_bs, self._n_pairs[self._cur], self.loss,
                 self.correct, self._dZ32 if train else None)
    if not train:
      return
    boff, n = self._b_off[L - 1]
    nat.relu_bwd_cast(self._dZ32, self.Z[L], ar.counters, 1, self.dPre[L], self.g32[boff:boff + n], True, 1.0,
                      relu=False)

  @torch.no_grad()
  def evaluate_batch(self, pairs: torch.Tensor):
    """(loss, #correct, #pairs) of a batch of positive pairs and their freshly drawn negatives, without updating
    parameters (no dropout)."""
    assert not (self.pipeline and self._primed), 'call flush() before evaluate_batch()'
    self._stage_seeds(self.seeds_dev, pairs)
    self._sample()
    self._forward(train=False)
    return float(self.loss.item()), int(self.correct.item()), int(self._n_pairs[self._cur].item())
