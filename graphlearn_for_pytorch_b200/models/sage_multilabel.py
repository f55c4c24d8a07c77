"""GraphSageMultiLabelEngine: the CUDA-graphed GraphSAGE training step for multi-label node classification.

A `GraphSageEngine` whose nodes carry T independent binary labels (ogbn-proteins' 112 tasks, PPI's 121, Yelp, Amazon)
instead of one class, trained with the mean sigmoid binary cross-entropy of `F.binary_cross_entropy_with_logits`.
Sampling, layers, backward and Adam are the node engine's; only the loss launch differs:

  k_sigmoid_bce  per seed row: BCE forward and backward over the T logits, labels read from a device bit matrix
                 through the batch's node list, last-layer bias gradient in the same pass (csrc/cuda/multilabel.cu)

so the captured step has the same launches as a `GraphSageEngine` with T classes.
"""
from typing import List

import torch

from .sage import GraphSageEngine


def check_multilabel(labels: torch.Tensor, num_nodes: int = None) -> int:
  """Validates a [N, T] tensor of 0/1 labels (bool, integer or floating) and returns T; raises ValueError otherwise."""
  if not torch.is_tensor(labels) or labels.dim() != 2 or labels.shape[1] < 1:
    raise ValueError(f'labels must be a [num_nodes, T] tensor with T >= 1 (got {getattr(labels, "shape", labels)})')
  if num_nodes is not None and labels.shape[0] != int(num_nodes):
    raise ValueError(f'labels has {labels.shape[0]} rows for {num_nodes} nodes')
  if labels.dtype != torch.bool and not bool(((labels == 0) | (labels == 1)).all()):
    raise ValueError('labels must hold only 0 and 1')
  return int(labels.shape[1])


def pack_label_bits(labels: torch.Tensor) -> torch.Tensor:
  """uint32 [N, ceil(T / 32)] bit matrix of 0/1 labels [N, T]: task c of node v is bit c % 32 of word c // 32 of row v
  (the layout `sigmoid_bce` reads).  Built on the labels' device."""
  T = check_multilabel(labels)
  N, W = labels.shape[0], (T + 31) // 32
  y = torch.nn.functional.pad(labels.to(torch.int64), (0, 32 * W - T)).view(N, W, 32)
  words = (y << torch.arange(32, device=labels.device)).sum(-1)
  # to uint32 through the int32 of the same bits (a reinterpreting view; int64 -> uint32 casts are CPU-only)
  return torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32).view(torch.uint32).contiguous()


def multilabel_f1(logits: torch.Tensor, y: torch.Tensor) -> float:
  """Micro-averaged F1 of the predictions logit > 0 against 0/1 labels y (both [n, T])."""
  pred, y = logits.float() > 0, y.bool()
  tp = int((pred & y).sum())
  den = tp + int((pred & ~y).sum()) + tp + int((~pred & y).sum())
  return 2 * tp / den if den else 0.0


def multilabel_auc(logits: torch.Tensor, y: torch.Tensor) -> float:
  """Mean ROC-AUC over the tasks (columns) whose labels hold both classes, ties at their mean rank (ogbn-proteins'
  metric); nan when no task has both classes."""
  s, y = logits.double(), y.bool()
  aucs = []
  for t in range(y.shape[1]):
    pos = y[:, t]
    n_pos = int(pos.sum())
    n_neg = pos.numel() - n_pos
    if n_pos == 0 or n_neg == 0:
      continue
    _, inv, cnt = torch.unique(s[:, t], return_inverse=True, return_counts=True)
    mean_rank = cnt.cumsum(0).double() - (cnt.double() - 1) / 2          # 1-based mean rank of each distinct score
    r = mean_rank[inv][pos].sum()
    aucs.append(float((r - n_pos * (n_pos + 1) / 2) / (n_pos * n_neg)))
  return sum(aucs) / len(aucs) if aucs else float('nan')


class GraphSageMultiLabelEngine(GraphSageEngine):
  """Static-shape, CUDA-graph-captured GraphSAGE step for multi-label node classification (mean BCE-with-logits).

  Args:
    graph, feature_table, in_dim, num_nodes, fanouts, batch_size, hidden: as `GraphSageEngine`.
    labels: [num_nodes, T] tensor of 0/1 values (bool, integer or floating); kept on the device as a packed bit matrix
      (`pack_label_bits`, T / 8 bytes per node).  T plays the part of `num_classes`.
    **engine_kwargs: every other `GraphSageEngine` option (lr, weight_decay, seed, device, group, use_fused,
      use_cuda_graph, pipeline, dropout, feature_format, deterministic_sampling, calibration_*, ...).

  `train_step(seeds)` returns the device scalar of the mean BCE over the batch's seeds and tasks;
  `evaluate_batch(seeds)` returns (loss, TP, FP, FN, #seeds) with predictions at logit 0; `inference()` returns the bf16
  logits [num_nodes, T] (score them with `multilabel_auc` / `multilabel_f1`).
  """

  def __init__(self, graph, feature_table, labels: torch.Tensor, in_dim: int, num_nodes: int,
               fanouts: List[int] = (15, 10, 5), batch_size: int = 1024, hidden: int = 256, **engine_kwargs):
    T = check_multilabel(labels, num_nodes)
    bits = pack_label_bits(labels)
    super().__init__(graph, feature_table, torch.zeros(1, dtype=torch.int64), in_dim, num_nodes, fanouts=fanouts,
                     batch_size=batch_size, hidden=hidden, num_classes=T, **engine_kwargs)
    self.label_bits = bits.to(self.device)
    self.counts = torch.zeros(3, dtype=torch.int32, device=self.device)    # TP, FP, FN of evaluate_batch

  def _forward_loss(self, train: bool = True):
    nat, ar = self.nat, self.arena
    boff, n = self._b_off[self.L - 1]
    if train:                      # as the base class: zeroes the gradients and the loss, so the kernel skips memsets
      self._begin_grads()
    # evaluation (not prezeroed): the launch zeroes the loss and the counts, and writes no gradient
    nat.sigmoid_bce(self.Z[self.L], self.C, self.label_bits, ar.nodes, ar.counters, self.loss, self.dPre[self.L],
                    None if train else self.counts, self.g32[boff:boff + n] if train else None, train)

  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    """(loss, TP, FP, FN, #seeds) for a batch without updating parameters (no dropout)."""
    loss, _, n = super().evaluate_batch(seeds)
    tp, fp, fn = self.counts.tolist()
    return loss, tp, fp, fn, n
