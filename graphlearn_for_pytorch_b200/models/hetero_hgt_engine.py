"""`HeteroHgtEngine`: device-resident Heterogeneous Graph Transformer (HGT) training step.

The model is the reference's OGB-MAG HGT (examples/hetero/train_hgt_mag.py): a per-type input `Linear` + ReLU, then
L `HGTConv(H, H, heads)` layers, then a `Linear(H, classes)` head on the seed type.  For a destination type t, its
incoming relations r = (s -> t) and heads of width D = H / heads, layer l computes

  k, q, v = Lin_k/q/v(x)                                  one [3H, H] Linear per type, rows [K | Q | V]
  s_ij,h  = <q_i,h, k_j,h W_att[r, h]> prior[r, h] / sqrt(D)
  alpha   = softmax over ALL sampled in-neighbours of i across every relation into t, per head
  agg_i   = sum_r sum_j alpha_ij (v_j,h W_msg[r, h])
  out_i   = sigmoid(skip_t) Lin_a,t(gelu(agg_i)) + (1 - sigmoid(skip_t)) x_i

(`models.HGTConv` with in == out).  Both relation transforms move to the target side, so a type needs two GEMMs for
all of its relations: qq = Q [W_att,r1 | W_att,r2 | ...]^T before the attention kernel, and agg = [u_r1 | u_r2 | ...]
[W_msg,r1; W_msg,r2; ...] after it, where u_r = sum_j alpha v_j over r's slots.  The GEMM weights are the block-
diagonal images of the [heads, D, D] parameters, rebuilt from the bf16 shadow every step; only the diagonal blocks are
parameters.

The step keeps everything of `HeteroSageEngine` -- the grouped sampling arena, the per-type id spaces, CUDA-graph
capture, the fused Adam (and its peer all-reduce), `state_dict`, `evaluate_batch` -- and replaces the layers:

  input    per type: feature gather, then a TcGemm with the bias + ReLU epilogue
  layer l  per type: the K/Q/V GEMM over its rows of hops 0..L-l+1;  per destination type: relation images
           (hgt_blocks), the qq GEMM, the attention (hgt_attention), the message GEMM, GELU, Lin_a, the skip gate
  head     Linear GEMM with bias, fused log-softmax / NLL
  backward the gate backward (dA, the residual into the previous layer's fp32 gradient, the skip gradient), Lin_a
           wgrad + dgrad, GELU backward, message wgrad + dgrad, the attention backward (hgt_attention_bwd: dqq, the
           prior gradient, dK / dV with fp32 red.add into the source rows), qq wgrad + dgrad, the diagonal blocks of the
           two dense weight gradients; then per type the K/Q/V gradient cast with its bias gradient, K/Q/V wgrad +
           dgrad, and the dgrad added into the previous layer's fp32 gradient

Initialisation follows `models/hgt.py`: `torch.nn.Linear` defaults, randn / sqrt(D) for the relation transforms, ones
for prior and skip, all drawn from the engine's seeded generator.  There is no dropout (the reference has none).
"""
import math
from typing import Dict, Optional, Sequence, Union

import torch

from .hetero_engine import HeteroSageEngine, EdgeType
from .sage import infer_chunks

MAX_RELATIONS = 8      # incoming relations of one destination type that the attention kernels take


class HeteroHgtEngine(HeteroSageEngine):
  """Args: those of `HeteroSageEngine`, plus
    heads: attention heads; hidden / heads = D must be a multiple of 8.

  Widths: every node type's `in_dim` and `hidden` must be multiples of 64 in [64, 1024].  Other widths, a destination
  type without incoming relations at some layer, and more than 8 relations into one type raise ValueError at
  construction.
  """

  def __init__(self, graphs: Dict[EdgeType, object], feature_tables: Dict[str, object], labels: torch.Tensor,
               in_dim: Union[int, Dict[str, int]], num_nodes: Dict[str, int], seed_type: str,
               fanouts: Union[Sequence[int], Dict[EdgeType, Sequence[int]]] = (10, 10), batch_size: int = 1024,
               hidden: int = 64, num_classes: int = 349, heads: int = 2, edge_dir: str = 'in', lr: float = 1e-2,
               weight_decay: float = 0.0, seed: int = 0, device: Optional[torch.device] = None,
               use_cuda_graph: bool = True, cap_limit: int = 1 << 21, group=None,
               feature_format: Union[str, Dict[str, str]] = 'bf16'):
    self.heads = self._check_heads(heads, hidden)
    super().__init__(graphs, feature_tables, labels, in_dim, num_nodes, seed_type, fanouts=fanouts,
                     batch_size=batch_size, hidden=hidden, num_classes=num_classes, edge_dir=edge_dir, lr=lr,
                     weight_decay=weight_decay, seed=seed, device=device, use_cuda_graph=use_cuda_graph,
                     cap_limit=cap_limit, group=group, feature_format=feature_format)

  # ------------------------------------------------------------------ buffers / parameters
  def _alloc(self):
    self._check_attention_schema()
    z, f32 = self._zeros, torch.float32
    H, L = self.hidden, self.L
    for l in range(1, L + 1):
      for t in self.targets[l]:
        if len(self.in_rel[l][t]) > MAX_RELATIONS:
          raise ValueError(f'node type {self.ntypes[t]!r} has {len(self.in_rel[l][t])} incoming relations at layer '
                           f'{l}; the attention kernels take at most {MAX_RELATIONS}')
    # types whose K/Q/V layer l computes (message sources and destinations), and the input layer's types
    self.srcs = [None] + [sorted({self.nt[r] for t in self.targets[l] for r in self.in_rel[l][t]})
                          for l in range(1, L + 1)]
    self.kqv_types = [None] + [sorted(set(self.targets[l]) | set(self.srcs[l])) for l in range(1, L + 1)]
    self.in_types = sorted(set(self.targets[1]) | set(self.srcs[1]))
    self.X0 = {u: z(self._rows(0, u), self.dim_in[self.ntypes[u]]) for u in self.in_types}
    self.Z = [{u: z(self._rows(0, u), H) for u in self.in_types}]
    self.dH = [{u: z(self._rows(0, u), H, dt=f32) for u in self.in_types}]
    self.dPre0 = {u: z(self._rows(0, u), H) for u in self.in_types}
    self.KQV, self.QQ, self.U, self.AGG, self.GE, self.A = [None], [None], [None], [None], [None], [None]
    self.att_img, self.msg_img = {}, {}
    for l in range(1, L + 1):
      self.KQV.append({u: z(self._rows(l - 1, u), 3 * H) for u in self.kqv_types[l]})
      for buf in (self.QQ, self.U):
        buf.append({t: z(self._rows(l, t), len(self.in_rel[l][t]) * H) for t in self.targets[l]})
      for buf in (self.AGG, self.GE, self.A):
        buf.append({t: z(self._rows(l, t), H) for t in self.targets[l]})
      self.Z.append({t: z(self._rows(l, t), H) for t in self.targets[l]})
      self.dH.append({t: z(self._rows(l, t), H, dt=f32) for t in self.targets[l]} if l < L else {})
      for t in self.targets[l]:
        R = len(self.in_rel[l][t])
        self.att_img[(l, t)] = z(R * H, H)
        self.msg_img[(l, t)] = z(H, R * H)
    self._alloc_head()
    self.dZL = z(self._rows(L, self.tid[self.seed_type]), H)   # head dgrad: gradient of the last layer's output
    # alpha per (layer, relation, hop) and the backward's per-relation scratch (two floats per alpha entry)
    self.alpha, self.dal = {}, {}
    for l in range(1, L + 1):
      nh = L - l + 1
      for t in self.targets[l]:
        for r in self.in_rel[l][t]:
          self.alpha[(l, r)] = [z(max(self.arena.ell_of(r, h).numel(), 1) * self.heads, dt=f32) for h in range(nh)]
          if r not in self.dal:       # the lowest layer using r has the most hops
            self.dal[r] = [z(2 * a.numel(), dt=f32) for a in self.alpha[(l, r)]]
    # per-type backward scratch, sized for the widest layer that uses it (a layer's scratch is consumed within it)
    t_rows, t_rel, u_rows = {}, {}, {}
    for l in range(1, L + 1):
      for t in self.targets[l]:
        t_rows[t] = max(t_rows.get(t, 0), self._rows(l, t))
        t_rel[t] = max(t_rel.get(t, 0), len(self.in_rel[l][t]))
      for u in self.kqv_types[l]:
        u_rows[u] = max(u_rows.get(u, 0), self._rows(l - 1, u))
    self.dQQ = {t: z(n * t_rel[t] * H) for t, n in t_rows.items()}      # flat: viewed [rows, n_rel * H] per layer
    self.dU = {t: z(n * t_rel[t] * H) for t, n in t_rows.items()}
    self.dA = {t: z(n, H) for t, n in t_rows.items()}
    self.dGE = {t: z(n, H) for t, n in t_rows.items()}
    self.dAGG = {t: z(n, H) for t, n in t_rows.items()}
    self.dQ = {t: z(n, H) for t, n in t_rows.items()}
    self.g_att = {t: z(t_rel[t] * H * H, dt=f32) for t in t_rows}     # dense weight gradients of the two GEMMs
    self.g_msg = {t: z(t_rel[t] * H * H, dt=f32) for t in t_rows}
    self.dKV32 = {u: z(n, 2 * H, dt=f32) for u, n in u_rows.items()}
    self.dKQV = {u: z(n, 3 * H) for u, n in u_rows.items()}
    self.dX = {u: z(n, H) for u, n in u_rows.items()}

  def _param_layout(self):
    """Names ('in_W', t), ('in_b', t), ('kqv_W', l, t), ('kqv_b', l, t), ('att', l, r), ('msg', l, r), ('prior', l, r),
    ('a_W', l, t), ('a_b', l, t), ('skip', l, t), ('head_W',), ('head_b',).  The att and msg blocks of the relations
    into one (layer, type) are contiguous."""
    H, nhd = self.hidden, self.heads
    D = H // nhd
    for u in self.in_types:
      yield ('in_W', u), (H, self.dim_in[self.ntypes[u]])
      yield ('in_b', u), (H,)
    for l in range(1, self.L + 1):
      for u in self.kqv_types[l]:
        yield ('kqv_W', l, u), (3 * H, H)
        yield ('kqv_b', l, u), (3 * H,)
      for t in self.targets[l]:
        for kind in ('att', 'msg'):
          for r in self.in_rel[l][t]:
            yield (kind, l, r), (nhd, D, D)
        for r in self.in_rel[l][t]:
          yield ('prior', l, r), (nhd,)
        yield ('a_W', l, t), (H, H)
        yield ('a_b', l, t), (H,)
        yield ('skip', l, t), (1,)
    yield ('head_W',), (self.n_out_pad, H)
    yield ('head_b',), (self.n_out_pad,)

  def _param_init(self, name, shape, g: torch.Generator) -> torch.Tensor:
    kind = name[0]
    if kind in ('att', 'msg'):
      return torch.randn(*shape, generator=g) / math.sqrt(self.hidden // self.heads)
    if kind in ('prior', 'skip'):
      return torch.ones(*shape)
    # torch.nn.Linear defaults: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias, fan_in from the weight [out, in]
    fan_in = self.param_index[(kind[:-1] + 'W',) + name[1:]][1][1]
    v = (torch.rand(*shape, generator=g) * 2 - 1) / math.sqrt(fan_in)
    if kind in ('head_W', 'head_b'):
      v[self.C:] = 0
    return v

  def _blocks(self, kind, l, t, grad=False):
    """[n_rel, heads, D, D] view of the att or msg blocks of the relations into (l, t)."""
    D = self.hidden // self.heads
    return self._rel_params(kind, l, t, grad).view(-1, self.heads, D, D)

  def _rel_view(self, buf, l, t):
    """[rows, n_rel * H] contiguous view of a flat per-type buffer for the relations into (l, t)."""
    n, w = self._rows(l, t), len(self.in_rel[l][t]) * self.hidden
    return buf[t][:n * w].view(n, w)

  # ------------------------------------------------------------------ step pieces
  def _hgt_plan(self, kind: str, l: int, t: int):
    key = ('hgt', kind, l, t)
    pl = self._plans.get(key)
    if pl is not None:
      return pl
    pl = self.nat.TcGemm(self.device.index)
    H, L = self.hidden, self.L
    nh = L - l + 1
    c = self._ctr[t]
    if kind == 'in_fwd':
      pl.add_forward(self.X0[t], self.param(('in_W', t)), self.param(('in_b', t)), True, self.Z[0][t], c, L + 1)
    elif kind == 'in_bwd':
      pl.add_wgrad(self.dPre0[t], self.X0[t], self.param(('in_W', t), True), c, L + 1)
    elif kind == 'kqv_fwd':
      pl.add_forward(self.Z[l - 1][t], self.param(('kqv_W', l, t)), self.param(('kqv_b', l, t)), False,
                     self.KQV[l][t], c, nh + 1)
    elif kind == 'kqv_bwd':
      n = self._rows(l - 1, t)
      pl.add_wgrad(self.dKQV[t][:n], self.Z[l - 1][t], self.param(('kqv_W', l, t), True), c, nh + 1)
      pl.add_dgrad(self.dKQV[t][:n], self.param(('kqv_W', l, t)), self.dX[t][:n], c, nh + 1)
    else:
      n, R = self._rows(l, t), len(self.in_rel[l][t])
      Q = self.KQV[l][t][:n, H:2 * H]
      if kind == 'qq_fwd':
        pl.add_forward(Q, self.att_img[(l, t)], None, False, self.QQ[l][t], c, nh)
      elif kind == 'qq_bwd':
        dQQ = self._rel_view(self.dQQ, l, t)
        pl.add_wgrad(dQQ, Q, self.g_att[t][:R * H * H].view(R * H, H), c, nh)
        pl.add_dgrad(dQQ, self.att_img[(l, t)], self.dQ[t][:n], c, nh)
      elif kind == 'msg_fwd':
        pl.add_forward(self.U[l][t], self.msg_img[(l, t)], None, False, self.AGG[l][t], c, nh)
      elif kind == 'msg_bwd':
        pl.add_wgrad(self.dAGG[t][:n], self.U[l][t], self.g_msg[t][:R * H * H].view(H, R * H), c, nh)
        pl.add_dgrad(self.dAGG[t][:n], self.msg_img[(l, t)], self._rel_view(self.dU, l, t), c, nh)
      elif kind == 'a_fwd':
        pl.add_forward(self.GE[l][t], self.param(('a_W', l, t)), self.param(('a_b', l, t)), False, self.A[l][t], c, nh)
      elif kind == 'a_bwd':
        pl.add_wgrad(self.dA[t][:n], self.GE[l][t], self.param(('a_W', l, t), True), c, nh)
        pl.add_dgrad(self.dA[t][:n], self.param(('a_W', l, t)), self.dGE[t][:n], c, nh)
      else:
        raise KeyError(kind)
    self._plans[key] = pl
    return pl

  def _attn_rel_args(self, l, t):
    nh = self.L - l + 1
    rels = self.in_rel[l][t]
    ells, kss = zip(*[self._rel_ell(r, nh) for r in rels])
    kv = [self.KQV[l][self.nt[r]] for r in rels]
    prior = [self._p32(('prior', l, r)) for r in rels]
    deg = [self.arena.deg_of(r) for r in rels]
    alpha = [self.alpha[(l, r)] for r in rels]
    return kv, prior, list(ells), list(kss), deg, alpha

  def _forward(self):
    nat, L = self.nat, self.L
    for u in self.in_types:
      self._gather_input(u)
      self._hgt_plan('in_fwd', 0, u).run()
    for l in range(1, L + 1):
      nh = L - l + 1
      for t in self.targets[l]:
        nat.hgt_blocks(self._blocks('att', l, t), self._blocks('msg', l, t), self.att_img[(l, t)],
                       self.msg_img[(l, t)])
      for u in self.kqv_types[l]:
        self._hgt_plan('kqv_fwd', l, u).run()
      for t in self.targets[l]:
        c = self._ctr[t]
        self._hgt_plan('qq_fwd', l, t).run()
        kv, prior, ells, kss, deg, alpha = self._attn_rel_args(l, t)
        nat.hgt_attention(self.QQ[l][t], self.U[l][t], self.heads, c, nh, kv, prior, ells, kss, deg, alpha)
        self._hgt_plan('msg_fwd', l, t).run()
        nat.hgt_gelu(self.AGG[l][t], self.GE[l][t], c, nh)
        self._hgt_plan('a_fwd', l, t).run()
        nat.hgt_gate(self.A[l][t], self.Z[l - 1][t][:self._rows(l, t)], self.Z[l][t], self._p32(('skip', l, t)), c, nh)
    self._head_plan().run()
    self._loss(self.logits, self.dlogits, self.param(('head_b',), True))

  def _backward(self):
    nat, L, H = self.nat, self.L, self.hidden
    self._head_plan(self.dZL).run()
    for l in range(L, 0, -1):
      nh = L - l + 1
      below = self.dH[l - 1]
      for u in below:
        nat.zero_rows(below[u], self._ctr[u], nh + 1)
      for t in self.targets[l]:
        c, n, R = self._ctr[t], self._rows(l, t), len(self.in_rel[l][t])
        dZ = self.dZL if l == L else self.dH[l][t]
        nat.hgt_gate(self.A[l][t], self.Z[l - 1][t][:n], self.dA[t][:n], self._p32(('skip', l, t)), c, nh, dZ=dZ,
                     dX=below[t][:n], skip_g=self._p32(('skip', l, t), True))
        nat.colsum_bf16(self.dA[t][:n], c, nh, self.param(('a_b', l, t), True))
        self._hgt_plan('a_bwd', l, t).run()
        nat.hgt_gelu(self.AGG[l][t], self.dAGG[t][:n], c, nh, dY=self.dGE[t][:n])
        self._hgt_plan('msg_bwd', l, t).run()
        kv, prior, ells, kss, deg, alpha = self._attn_rel_args(l, t)
        rels = self.in_rel[l][t]
        nat.hgt_attention_bwd(self._rel_view(self.dU, l, t), self.QQ[l][t], self._rel_view(self.dQQ, l, t), self.heads,
                              c, nh, kv,
                              prior, ells, kss, deg, alpha, [self.dal[r][:nh] for r in rels],
                              [self.dKV32[self.nt[r]] for r in rels], [self._p32(('prior', l, r), True) for r in rels])
        self._hgt_plan('qq_bwd', l, t).run()
        nat.hgt_blocks(self._blocks('att', l, t), self._blocks('msg', l, t), self.att_img[(l, t)],
                       self.msg_img[(l, t)], att_dense=self.g_att[t][:R * H * H], msg_dense=self.g_msg[t][:R * H * H],
                       att_g=self._blocks('att', l, t, True), msg_g=self._blocks('msg', l, t, True))
      for u in self.kqv_types[l]:
        n = self._rows(l - 1, u)
        is_t = u in self.targets[l]
        nat.hgt_kqv_cast(self.dKV32[u][:n], self.dQ[u] if is_t else None, self.dKQV[u][:n],
                         self._p32(('kqv_b', l, u), True), self._ctr[u], nh + 1, nh)
        self._hgt_plan('kqv_bwd', l, u).run()
        nat.add_block_f32(self.dX[u][:n], 0, H, self._ctr[u], nh + 1, below[u])
    for u in self.in_types:
      nat.relu_bwd_cast(self.dH[0][u], self.Z[0][u], self._ctr[u], L + 1, self.dPre0[u],
                        self.param(('in_b', u), True), True, 1.0, True)
      self._hgt_plan('in_bwd', 0, u).run()

  # ------------------------------------------------------------------ full-neighbourhood inference
  def _infer_chunk_row_bytes(self) -> int:
    R = max(len(self.in_rel[l][t]) for l in range(1, self.L + 1) for t in self.targets[l])
    return 2 * max(max(self.dim_in.values()), (2 * R + 3) * self.hidden)

  _infer_head = HeteroSageEngine._infer_linear_head

  def _infer_input(self, chunk_rows: int):
    """Input layer: relu(x W_in^T + b_in) of every node of the input types, from gathered feature chunks."""
    dev = self.device
    buf = torch.empty(chunk_rows * max(self.dim_in.values()), dtype=torch.bfloat16, device=dev)
    X = {}
    for u in self.in_types:
      X[u] = torch.empty(self._n_nodes[u], self.hidden, dtype=torch.bfloat16, device=dev)
      for r0, r1 in infer_chunks(self._n_nodes[u], chunk_rows):
        self._gemm(self._gather_chunk(u, r0, r1, buf), self.param(('in_W', u)), self.param(('in_b', u)), True,
                   X[u][r0:r1], 0)
    return X

  def _infer_layer(self, l: int, X, Z, chunk_rows: int):
    """HGT layer l: K/Q/V of every node of the layer's types, then per destination type and chunk of targets the qq
    GEMM, the attention over the complete rows of every relation into t (hgt_full_attention), the message GEMM, GELU,
    Lin_a and the skip gate."""
    nat, dev, H, hd = self.nat, self.device, self.hidden, self.heads
    bf = torch.bfloat16
    KQV = {}
    for u in self.kqv_types[l]:
      KQV[u] = torch.empty(self._n_nodes[u], 3 * H, dtype=bf, device=dev)
      self._gemm(X[u], self.param(('kqv_W', l, u)), self.param(('kqv_b', l, u)), False, KQV[u], 1 + u)
    for t in self.targets[l]:
      rels = self.in_rel[l][t]
      R = len(rels)
      att_img = torch.empty(R * H, H, dtype=bf, device=dev)
      msg_img = torch.empty(H, R * H, dtype=bf, device=dev)
      nat.hgt_blocks(self._blocks('att', l, t), self._blocks('msg', l, t), att_img, msg_img)
      qq = torch.empty(chunk_rows, R * H, dtype=bf, device=dev)
      U = torch.empty(chunk_rows, R * H, dtype=bf, device=dev)
      AGG, GE, A = (torch.empty(chunk_rows, H, dtype=bf, device=dev) for _ in range(3))
      graphs = [self._gh(r) for r in rels]
      kv = [KQV[self.nt[r]] for r in rels]
      prior = [self._p32(('prior', l, r)) for r in rels]
      for r0, r1 in infer_chunks(self._n_nodes[t], chunk_rows):
        n = r1 - r0
        self._gemm(KQV[t][r0:r1, H:2 * H], att_img, None, False, qq[:n], 0)
        nat.hgt_full_attention(graphs, qq[:n], U[:n], hd, r0, r1, kv, prior)
        self._gemm(U[:n], msg_img, None, False, AGG[:n], 0)
        nat.hgt_gelu(AGG[:n], GE[:n], self._rows_dev, 0)
        self._gemm(GE[:n], self.param(('a_W', l, t)), self.param(('a_b', l, t)), False, A[:n], 0)
        nat.hgt_gate(A[:n], X[t][r0:r1], Z[t][r0:r1], self._p32(('skip', l, t)), self._rows_dev, 0)
