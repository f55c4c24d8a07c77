"""`HeteroGatEngine`: device-resident relational GAT (R-GAT) training step for heterogeneous graphs.

The model is the reference's IGBH R-GAT (examples/igbh/rgnn.py): per layer a `HeteroConv` of
`GATConv(in, H // heads, heads=heads, add_self_loops=False)` per relation, summed over the relations of each destination
type; `leaky_relu(., 0.01)` and dropout between layers; a final `Linear(H, classes)` on the seed type.  For a relation
r = (s -> t) at layer l:

  h_j = W_src x_s[j],  g_i = W_dst x_t[i]                   one weight per relation when d_s == d_t (PyG's
                                                            GATConv(int, ...)), separate weights otherwise (tuple form)
  e_ij,h = leaky_relu(<att_src[h], h_j,h> + <att_dst[h], g_i,h>, 0.2),  alpha = softmax over i's sampled in-neighbours
  out_i = concat_h sum_j alpha_ij,h h_j,h + bias_r          (a target without neighbours in r gets bias_r)

The step keeps everything of `HeteroSageEngine` -- the grouped sampling arena, the per-type id spaces, CUDA-graph
capture, the fused Adam (and its peer all-reduce), `state_dict`, `evaluate_batch` -- and replaces the layers:

  layer l  per relation: projection GEMM(s) (TMA/wgmma TcGemm; a relation whose two ends are the same type projects
           once, the targets being a prefix of the source rows), per-node scores (gat_scores), the attention
           aggregation (gat_aggregate: softmax, weighted sum, fp32 sum over the type's relations in a fixed order; the
           last relation adds the biases and the activation and writes bf16 Z)
  head     Linear GEMM with bias, fused log-softmax / NLL
  backward per relation: gat_backward (softmax backward from the saved alpha, fp32 red.add of alpha G into the source
           rows), gat_score_bwd (score terms, attention gradients, bf16 projection gradients), wgrad (split-K) and,
           below the top layer, dgrad GEMMs whose bf16 outputs are summed into the previous layer's fp32 gradient
           (add_block_f32: a dgrad's TMA store overwrites); then the activation backward with the dropout mask
           regenerated from its Philox key and the bias gradients of every relation (gat_act_bwd)

Biases are one parameter per relation, each with its own Adam state, as in PyG.  Initialisation is PyG's: Glorot for W
and att, zero GAT biases, `torch.nn.Linear`'s default for the head, drawn from the engine's seeded generator.
"""
import math
from typing import Dict, Optional, Sequence, Union

import torch

from .hetero_engine import HeteroSageEngine, EdgeType
from .sage import infer_chunks


class HeteroGatEngine(HeteroSageEngine):
  """Args: those of `HeteroSageEngine`, plus
    heads: attention heads; hidden / heads = C must be a multiple of 8.
    dropout: dropout probability between layers (the reference's default 0.2), in [0, 1).

  Widths: every node type's `in_dim` and `hidden` must be multiples of 64 in [64, 1024].  Other widths raise ValueError
  at construction.
  """

  def __init__(self, graphs: Dict[EdgeType, object], feature_tables: Dict[str, object], labels: torch.Tensor,
               in_dim: Union[int, Dict[str, int]], num_nodes: Dict[str, int], seed_type: str,
               fanouts: Union[Sequence[int], Dict[EdgeType, Sequence[int]]] = (15, 10, 5), batch_size: int = 1024,
               hidden: int = 512, num_classes: int = 19, heads: int = 4, dropout: float = 0.2, edge_dir: str = 'in',
               lr: float = 1e-3, weight_decay: float = 0.0, seed: int = 0, device: Optional[torch.device] = None,
               use_cuda_graph: bool = True, cap_limit: int = 1 << 21, group=None,
               feature_format: Union[str, Dict[str, str]] = 'bf16'):
    self.heads = self._check_heads(heads, hidden)
    self.dropout = float(dropout)
    if not 0.0 <= self.dropout < 1.0:
      raise ValueError(f'dropout must be in [0, 1) (got {dropout})')
    self._training = True
    super().__init__(graphs, feature_tables, labels, in_dim, num_nodes, seed_type, fanouts=fanouts,
                     batch_size=batch_size, hidden=hidden, num_classes=num_classes, edge_dir=edge_dir, lr=lr,
                     weight_decay=weight_decay, seed=seed, device=device, use_cuda_graph=use_cuda_graph,
                     cap_limit=cap_limit, group=group, feature_format=feature_format)

  # ------------------------------------------------------------------ buffers / parameters
  def _X(self, l: int, t: int) -> torch.Tensor:
    return self.X0[t] if l == 0 else self.Z[l][t]

  def _alloc(self):
    self._check_attention_schema()
    z, f32 = self._zeros, torch.float32
    H, nhd = self.hidden, self.heads
    # layer 1 reads the features of its targets and of its relations' sources (a source type can be sampled only at
    # the deepest hop, outside targets[1])
    self.in_types = sorted(set(self.targets[1]) | {self.nt[r] for t in self.targets[1] for r in self.in_rel[1][t]})
    self.X0 = {t: z(self._rows(0, t), self.dim_in[self.ntypes[t]]) for t in self.in_types}
    self.Z, self.G, self.dH = [None], [None], [None]
    for l in range(1, self.L + 1):
      self.Z.append({t: z(self._rows(l, t), H) for t in self.targets[l]})
      self.G.append({t: z(self._rows(l, t), H) for t in self.targets[l]})        # gradient of the pre-activation
      self.dH.append({t: z(self._rows(l, t), H, dt=f32) for t in self.targets[l]} if l < self.L else {})
    # relation sums of types with several relations (shared by the layers: a layer's sum is consumed within it)
    acc_rows = {}
    for l in range(1, self.L + 1):
      for t in self.targets[l]:
        if len(self.in_rel[l][t]) > 1:
          acc_rows[t] = max(acc_rows.get(t, 0), self._rows(l, t))
    self.acc = {t: z(n, H, dt=f32) for t, n in acc_rows.items()}
    # per (layer, relation): saved projections, alpha, the per-source score gradient
    self.Ps, self.Pd, self.alpha, self.dsrc = {}, {}, {}, {}
    used = {}
    for l in range(1, self.L + 1):
      nh = self.L - l + 1
      for t in self.targets[l]:
        for r in self.in_rel[l][t]:
          s = self.nt[r]
          used.setdefault(r, []).append(l)
          self.Ps[(l, r)] = z(self._rows(l - 1, s), H)
          # the targets of a relation between rows of one type are a prefix of its source rows: one projection
          self.Pd[(l, r)] = None if s == t else z(self._rows(l, t), H)
          self.alpha[(l, r)] = [z(max(self.arena.ell_of(r, h).numel(), 1) * nhd, dt=f32) for h in range(nh)]
          self.dsrc[(l, r)] = z(self._rows(l - 1, s), nhd, dt=f32)
    # per-relation scratch, sized for the widest layer that uses the relation
    self.as_, self.ad_, self.dal, self.dP32, self.dPs, self.dPd, self.dadst = {}, {}, {}, {}, {}, {}, {}
    for r, ls in used.items():
      s, t = self.nt[r], self.kt[r]
      ns, nt_ = max(self._rows(l - 1, s) for l in ls), max(self._rows(l, t) for l in ls)
      self.as_[r], self.ad_[r] = z(ns, nhd, dt=f32), z(nt_, nhd, dt=f32)
      self.dal[r] = [z(a.numel(), dt=f32) for a in self.alpha[(min(ls), r)]]
      self.dP32[r], self.dPs[r] = z(ns, H, dt=f32), z(ns, H)
      self.dadst[r] = z(nt_, nhd, dt=f32)
      if s != t:
        self.dPd[r] = z(nt_, H)
    # bf16 dgrad outputs (a TMA store overwrites), added into the fp32 gradient of the previous layer
    self.dX = {}
    for l in range(2, self.L + 1):
      for t in self.targets[l - 1]:
        self.dX[t] = z(max(self._rows(l - 1, t), self.dX[t].shape[0] if t in self.dX else 0), H)
    self._alloc_head()

  def _param_layout(self):
    """Names ('W_src', l, r), ('W_dst', l, r) (only when the two ends have different widths), ('att_src', l, r),
    ('att_dst', l, r), ('bias', l, r), ('head_W',), ('head_b',).  The biases of the relations into one (layer, type)
    are contiguous."""
    H = self.hidden
    for l in range(1, self.L + 1):
      for t in self.targets[l]:
        for r in self.in_rel[l][t]:
          ds = self._width_in(l, self.nt[r])
          dt = self._width_in(l, t)
          yield ('W_src', l, r), (H, ds)
          if ds != dt:
            yield ('W_dst', l, r), (H, dt)
          yield ('att_src', l, r), (H,)
          yield ('att_dst', l, r), (H,)
        for r in self.in_rel[l][t]:
          yield ('bias', l, r), (H,)
    yield ('head_W',), (self.n_out_pad, H)
    yield ('head_b',), (self.n_out_pad,)

  def _param_init(self, name, shape, g: torch.Generator) -> torch.Tensor:
    H, nhd = self.hidden, self.heads
    kind = name[0]
    if kind in ('W_src', 'W_dst'):
      return (torch.rand(*shape, generator=g) * 2 - 1) * math.sqrt(6.0 / (shape[0] + shape[1]))   # glorot on [H, d]
    if kind in ('att_src', 'att_dst'):
      return (torch.rand(*shape, generator=g) * 2 - 1) * math.sqrt(6.0 / (nhd + H // nhd))   # glorot on [1, heads, C]
    if kind == 'bias':
      return torch.zeros(shape)
    v = (torch.rand(*shape, generator=g) * 2 - 1) / math.sqrt(H)       # torch.nn.Linear(H, classes) defaults
    v[self.C:] = 0
    return v

  def _w_dst(self, l, r, grad=False):
    return self.param(('W_dst', l, r) if ('W_dst', l, r) in self.param_index else ('W_src', l, r), grad)

  # ------------------------------------------------------------------ step pieces
  def _views(self, l, r):
    """(source rows, target rows, Ps, Pd or None) of relation r at layer l."""
    s, t = self.nt[r], self.kt[r]
    return self._rows(l - 1, s), self._rows(l, t), self.Ps[(l, r)], self.Pd[(l, r)]

  def _gat_plan(self, kind: str, l: int, r: int):
    key = ('gat', kind, l, r)
    pl = self._plans.get(key)
    if pl is not None:
      return pl
    pl = self.nat.TcGemm(self.device.index)
    nh = self.L - l + 1
    s, t = self.nt[r], self.kt[r]
    ns, ntr, Ps, Pd = self._views(l, r)
    Xs, Xt = self._X(l - 1, s), self._X(l - 1, t)[:ntr]
    cs, ct = self._ctr[s], self._ctr[t]
    if kind == 'proj':
      pl.add_forward(Xs, self.param(('W_src', l, r)), None, False, Ps, cs, nh + 1)
      if Pd is not None:
        pl.add_forward(Xt, self._w_dst(l, r), None, False, Pd, ct, nh)
    elif kind == 'wgrad':      # a shared weight receives both contributions in the same fp32 slice
      pl.add_wgrad(self.dPs[r][:ns], Xs, self.param(('W_src', l, r), True), cs, nh + 1)
      if Pd is not None:
        pl.add_wgrad(self.dPd[r][:ntr], Xt, self._w_dst(l, r, True), ct, nh)
    else:
      pl.add_dgrad(self.dPs[r][:ns], self.param(('W_src', l, r)), self.dX[s][:ns], cs, nh + 1)
      if Pd is not None:
        pl.add_dgrad(self.dPd[r][:ntr], self._w_dst(l, r), self.dX[t][:ntr], ct, nh)
    self._plans[key] = pl
    return pl

  def _forward(self):
    nat, ar, hd = self.nat, self.arena, self.heads
    p = self.dropout if self._training else 0.0
    for t in self.in_types:
      self._gather_input(t)
    for l in range(1, self.L + 1):
      nh = self.L - l + 1
      for t in self.targets[l]:
        rels = self.in_rel[l][t]
        for j, r in enumerate(rels):
          s = self.nt[r]
          ns, ntr, Ps, Pd = self._views(l, r)
          self._gat_plan('proj', l, r).run()
          nat.gat_scores(Ps, self.param(('att_src', l, r)), self.as_[r][:ns], self._ctr[s], nh + 1,
                         Pd if Pd is not None else Ps[:ntr], self.param(('att_dst', l, r)), self.ad_[r][:ntr],
                         self._ctr[t], nh, zero=self.dsrc[(l, r)], heads=hd)
          ell, ks = self._rel_ell(r, nh)
          last = j == len(rels) - 1
          nat.gat_aggregate(Ps, self.as_[r][:ns], self.ad_[r][:ntr], hd, self._ctr[t], nh, ell, ks, ar.deg_of(r),
                            self.alpha[(l, r)], acc=self.acc[t][:ntr] if len(rels) > 1 else None, first=j == 0,
                            last=last, bias=self._rel_params('bias', l, t) if last else None, act=l < self.L,
                            p=p if l < self.L else 0.0, seed=self.seed, layer=l, step_dev=self.step_dev,
                            Z=self.Z[l][t] if last else None)
    self._head_plan().run()
    self._loss(self.logits, self.dlogits, self.param(('head_b',), True))

  def _backward(self):
    nat, ar, hd, H = self.nat, self.arena, self.heads, self.hidden
    st = self.tid[self.seed_type]
    self._head_plan(self.G[self.L][st]).run()
    nat.gat_act_bwd(None, None, self.G[self.L][st], self._ctr[st], 1, bias_g=self._rel_params('bias', self.L, st, True))
    for l in range(self.L, 0, -1):
      nh = self.L - l + 1
      if l > 1:
        for u in self.targets[l - 1]:
          nat.zero_rows(self.dH[l - 1][u], self._ctr[u], nh + 1)
      for t in self.targets[l]:
        for r in self.in_rel[l][t]:
          s = self.nt[r]
          ns, ntr, Ps, Pd = self._views(l, r)
          ell, ks = self._rel_ell(r, nh)
          nat.gat_backward(self.G[l][t], Ps, hd, self._ctr[t], nh, ell, ks, ar.deg_of(r), self.alpha[(l, r)],
                           self.dal[r][:nh], self.dP32[r][:ns], self.dsrc[(l, r)], self.dadst[r][:ntr])
          nat.gat_score_bwd(Ps, self.dP32[r][:ns], self.dsrc[(l, r)], self.param(('att_src', l, r)),
                            self.param(('att_src', l, r), True), self.dPs[r][:ns], self._ctr[s], nh + 1,
                            self.dadst[r][:ntr], self.param(('att_dst', l, r)), self.param(('att_dst', l, r), True),
                            self._ctr[t], nh, P_dst=Pd, dPb_dst=self.dPd[r][:ntr] if Pd is not None else None,
                            heads=hd)
          self._gat_plan('wgrad', l, r).run()
          if l > 1:
            self._gat_plan('dgrad', l, r).run()
            nat.add_block_f32(self.dX[s][:ns], 0, H, self._ctr[s], nh + 1, self.dH[l - 1][s])
            if Pd is not None:
              nat.add_block_f32(self.dX[t][:ntr], 0, H, self._ctr[t], nh, self.dH[l - 1][t])
      if l > 1:
        for u in self.targets[l - 1]:
          nat.gat_act_bwd(self.dH[l - 1][u], self.Z[l - 1][u], self.G[l - 1][u], self._ctr[u], nh + 1,
                          p=self.dropout, seed=self.seed, layer=l - 1, step_dev=self.step_dev,
                          bias_g=self._rel_params('bias', l - 1, u, True))

  # ------------------------------------------------------------------ full-neighbourhood inference
  def _infer_chunk_row_bytes(self) -> int:
    return 2 * max(self.dim_in.values()) + 4 * self.hidden

  _infer_head = HeteroSageEngine._infer_linear_head

  def _infer_project(self, l: int, X, s: int, W: torch.Tensor, buf: torch.Tensor, chunk_rows: int) -> torch.Tensor:
    """bf16 [N_s, H] projection X_s W^T of every node of type s (layer 1: feature chunks gathered into buf first)."""
    P = torch.empty(self._n_nodes[s], self.hidden, dtype=torch.bfloat16, device=self.device)
    if l > 1:
      self._gemm(X[s], W, None, False, P, 1 + s)
      return P
    for r0, r1 in infer_chunks(self._n_nodes[s], chunk_rows):
      self._gemm(self._gather_chunk(s, r0, r1, buf), W, None, False, P[r0:r1], 0)
    return P

  def _infer_layer(self, l: int, X, Z, chunk_rows: int):
    """R-GAT layer l, per relation r = (s -> t): projections over every source (and every target when W_dst is a
    separate weight), per-node scores (gat_scores), then per chunk of targets the attention over complete rows
    (gat_full_aggregate), summed over t's relations in relation order; the last adds the biases and the activation."""
    nat, dev, H, hd = self.nat, self.device, self.hidden, self.heads
    buf = torch.empty(chunk_rows * max(self.dim_in.values()), dtype=torch.bfloat16, device=dev) if l == 1 else None
    for t in self.targets[l]:
      rels = self.in_rel[l][t]
      ops = []
      for r in rels:
        s = self.nt[r]
        Ps = self._infer_project(l, X, s, self.param(('W_src', l, r)), buf, chunk_rows)
        Pd = Ps if s == t and ('W_dst', l, r) not in self.param_index else \
            self._infer_project(l, X, t, self._w_dst(l, r), buf, chunk_rows)
        as_ = torch.empty(self._n_nodes[s], hd, dtype=torch.float32, device=dev)
        ad = torch.empty(self._n_nodes[t], hd, dtype=torch.float32, device=dev)
        nat.gat_scores(Ps, self.param(('att_src', l, r)), as_, self._rows_dev, 1 + s, Pd, self.param(('att_dst', l, r)),
                       ad, self._rows_dev, 1 + t, heads=hd)
        del Pd
        ops.append((r, Ps, as_, ad))
      acc = torch.empty(chunk_rows, H, dtype=torch.float32, device=dev) if len(rels) > 1 else None
      for r0, r1 in infer_chunks(self._n_nodes[t], chunk_rows):
        for j, (r, Ps, as_, ad) in enumerate(ops):
          last = j == len(ops) - 1
          nat.gat_full_aggregate(self._gh(r), Ps, as_, ad, hd, r0, r1, acc=acc[:r1 - r0] if acc is not None else None,
                                 first=j == 0, last=last, bias=self._rel_params('bias', l, t) if last else None,
                                 act=l < self.L, Z=Z[t][r0:r1] if last else None)

  # ------------------------------------------------------------------ public API
  @torch.no_grad()
  def evaluate_batch(self, seeds: torch.Tensor):
    """Loss, #correct and #seeds of one batch, forward only and without dropout."""
    self._training = False
    try:
      return super().evaluate_batch(seeds)
    finally:
      self._training = True
