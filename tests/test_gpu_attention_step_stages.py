"""Every launch of real R-GAT (HeteroGatEngine) and HGT (HeteroHgtEngine) training steps against float64, over
consecutive steps, eager and captured.

The kernel tests check each attention kernel on hand-built buffers, and the engine tests compare one step from fresh
parameters with an fp32 recomputation to a few per cent.  Here the engines run their public `train_step` over four
batches of bs, about bs / 3 (padded with -1), one isolated paper (no in-neighbour in any relation) and bs seeds, so
that steps 2 and 3 run far below the previous step's row counts on top of its rows.

A recorder local to this file replaces `eng.nat` right after construction (the GEMM plans are built lazily, so every
`TcGemm` is wrapped too).  Each native launch and `TcGemm.run()` clones its tensor arguments before and after the
launch; while the stream is capturing only the clones are issued, so they are captured into the step's graph and
refresh on every replay, and a captured step is audited launch by launch like an eager one.  Once the step is done,
every launch is checked in float64.  The call's arguments only identify the stage (which layer, relation or type and
which kind); the reference reads the buffers the model says feed that stage -- the pre-step parameters, the arena's
ELL edges of the relation and hops, the counters, the outputs of the earlier stages -- and the float64 sums that
build the fp32 gradient accumulators (dH, dKV32, dP32, the dense HGT weight gradients) are chained across launches
from zero, so a stale accumulator, a dropped or doubled contribution and a zero tail the next GEMM would read all
stand out.  A launch the audit has no check for fails the test, as does a stage the model requires that never ran.

The references and bounds are the kernel tests' own functions in tests/helpers.py (gemm_bound, gat_score_bound,
gat_alpha_bound, weighted_sum_bound, gat_dscore_tol, score_bwd_bound, act_bwd_ref, gelu_ref, gate_ref, skip_g_ref,
hgt_alpha_rel, hgt_bwd_tol, colsum_bound, ...), called with this step's parameters: where a stage's reference reads
the kernel's own alpha rather than a float64 one, the alpha terms are 0, and the sums are sized by the batch's row
degrees and source counts; each helper documents the difference.  Exact equality holds where a kernel only moves or
masks bits.  Every bound allows
results below fp32's normal range to be flushed to zero (FTZ): attention weights of e^-90 and less occur after a few
steps at the wide hidden widths, and the kernels flush them and their products.  Negative controls feed each defect,
applied to a perturbed copy of the recorded buffers, through the check that guards its stage and show that the check
rejects it; the controls configurations assert that every control ran.  `-s` prints the worst error / bound ratio per
stage, configuration and step, and the controls' ratios.
"""
import collections
import math
import os
import sys

import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.data import dequantize_mxfp8, quantize_mxfp8
from graphlearn_for_pytorch_b200.models import HeteroGatEngine, HeteroHgtEngine
from helpers import (EPS32, GAT_ISOLATED_EDGES, Ratios, _batches, _check_adam, _check_linear, _check_softmax, _f32,
                     _snapshot, _table, act_bwd_ref, add_isolated_papers, bf16_ulp, block_grads, block_images,
                     bound_ratio, colsum_bound, gat_alpha_bound, gat_dscore_tol, gat_score_bound, gate_da_ref,
                     gate_dx_ref, gate_ref, gelu_bwd_ref, gelu_ref, gemm_bound, hgt_alpha_rel, hgt_bwd_tol,
                     hgt_score_err, score_bwd_bound, skip_g_ref, softmax_seg, weighted_sum_bound)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'examples'))
ISOLATED = 64
FTZ = 2.0 ** -118                 # 256 flushed terms below 2^-126


def _ratio(got, ref, bound):
  """bound_ratio with an allowance for results below fp32's normal range: the kernels flush subnormal values to
  zero (a softmax weight of e^-90 and what it scales), which the float64 reference keeps."""
  return bound_ratio(got, ref, bound + FTZ)


def _round(n, m):
  return (n + m - 1) // m * m


# --------------------------------------------------------------------------- the recorder
class _Launch(object):
  """One native launch: its arguments, and clones of its tensor arguments before and after it."""

  def __init__(self, name, args, kwargs, tensors, pre, post, plan=None):
    self.name, self.args, self.kwargs, self.plan = name, args, kwargs, plan
    self.tensors, self._pre, self._post = tensors, pre, post

  def _find(self, clones, buf, what):
    for t, c in zip(self.tensors, clones):
      if t.data_ptr() == buf.data_ptr() and t.dtype == buf.dtype:
        if c.numel() == buf.numel():
          return c.reshape(buf.shape)
        if c.numel() > buf.numel() and buf.is_contiguous():
          return c.reshape(-1)[:buf.numel()].view(buf.shape)
        if c.dim() == buf.dim() and c.shape[1:] == buf.shape[1:]:
          return c                                           # the call passed a row prefix of buf
    raise AssertionError(f'{self.name}: the launch did not {what} the buffer the model feeds it')

  def pre(self, buf):
    return self._find(self._pre, buf, 'read')

  def post(self, buf):
    return self._find(self._post, buf, 'write')


def _tensors(obj, out):
  if torch.is_tensor(obj):
    if not any(t is obj for t in out):
      out.append(obj)
  elif isinstance(obj, (list, tuple)):
    for o in obj:
      _tensors(o, out)
  elif isinstance(obj, dict):
    for o in obj.values():
      _tensors(o, out)
  return out


class _Plan(object):
  """A TcGemm plan whose run() is recorded with its operands."""

  def __init__(self, rec, plan):
    self.rec, self.pl, self.ops = rec, plan, []

  def add_forward(self, *a):
    self.ops.append(('fwd', a))
    self.pl.add_forward(*a)

  def add_wgrad(self, *a):
    self.ops.append(('wgrad', a))
    self.pl.add_wgrad(*a)

  def add_dgrad(self, *a):
    self.ops.append(('dgrad', a))
    self.pl.add_dgrad(*a)

  def run(self):
    self.rec.launch('gemm', (self.ops,), {}, self.pl.run, plan=self)


AUDITED = {'gat_scores', 'gat_aggregate', 'gat_backward', 'gat_score_bwd', 'gat_act_bwd', 'hgt_blocks',
           'hgt_attention', 'hgt_attention_bwd', 'hgt_gelu', 'hgt_gate', 'hgt_kqv_cast', 'softmax_nll', 'zero_grads',
           'zero_rows', 'add_block_f32', 'colsum_bf16', 'relu_bwd_cast', 'adam_step'}


class Recorder(object):
  """Stands in for the native module of one engine.  `log` holds the launches of eager steps; launches issued while
  the stream captures are kept in `graph_log` (their clones are graph nodes, refreshed by every replay)."""

  def __init__(self, nat):
    self.nat, self.log, self.graph_log = nat, [], []

  def __getattr__(self, name):
    f = getattr(self.nat, name)
    if name == 'TcGemm':
      return lambda dev: _Plan(self, f(dev))
    if name == 'graph_node_counts':
      return f
    if name not in AUDITED:
      raise AssertionError(f'unaudited launch: {name}')
    return lambda *a, **k: self.launch(name, a, k, lambda: f(*a, **k))

  def launch(self, name, args, kwargs, run, plan=None):
    ts = _tensors([args, kwargs], [])
    pre = [t.clone() for t in ts]
    run()
    post = [t.clone() for t in ts]
    rec = _Launch(name, args, kwargs, ts, pre, post, plan)
    (self.graph_log if torch.cuda.is_current_stream_capturing() else self.log).append(rec)


# --------------------------------------------------------------------------- shared audit pieces
class Audit(object):
  """State of the audit of one step: pre-step parameters, counters, float64 chains of the fp32 accumulators, the
  stages audited so far."""

  def __init__(self, R, eng, snap, controls):
    torch.cuda.synchronize()
    self.R, self.eng, self.snap, self.controls = R, eng, snap, controls
    NT = len(eng.ntypes)
    cnt = eng.arena.counters.tolist()
    self.ctr = [cnt[t * 8:t * 8 + 8] for t in range(NT)]
    self.seen = collections.Counter()
    self.chain = {}                        # data_ptr of an fp32 accumulator -> (float64 value, bound)
    self.dgrad = {}                        # data_ptr of a dgrad output -> (float64 value, bound, rows)
    self.g_names = {}
    for name, (o, shape) in eng.param_index.items():
      self.g_names[eng.g32[o:].data_ptr()] = name
    self.negatives = {}
    self._ctr_ptr = {eng._ctr[t].data_ptr(): self.ctr[t] for t in range(NT)}
    self.prev = {}                         # previous step's buffers after their launches (negative controls)
    self.alpha_post = {}                   # (l, r) -> alpha of gat_aggregate (the relation-swap control)
    self.dense_stale = {}                  # data_ptr of a dense HGT gradient -> its value before hgt_blocks cleared it

  def ctr_of(self, c):
    return self._ctr_ptr[c.data_ptr()]

  def T_call(self, c, idx, rows):
    """Rows a launch takes from its own counter arguments."""
    return max(0, min(self.ctr_of(c)[idx], rows))

  def prev_tail(self, buf, T):
    p = self.prev.get(buf.data_ptr())
    return p[T:T + 64] if p is not None else torch.zeros_like(buf[T:T + 64])

  def p16(self, name):
    o, shape = self.eng.param_index[name]
    return self.snap['p16'][o:o + math.prod(shape)].view(*shape)

  def p32(self, name):
    o, shape = self.eng.param_index[name]
    return self.snap['p32'][o:o + math.prod(shape)].view(*shape)

  def grad_name(self, t):
    name = self.g_names.get(t.data_ptr())
    assert name is not None, 'a gradient argument outside the parameter layout'
    return name

  def T(self, t, idx, rows):
    return max(0, min(self.ctr[t][idx], rows))

  def mark(self, *key):
    self.seen[key] += 1

  def negative(self, what, ratio):
    """A control: the defect `what` must exceed its bound."""
    self.negatives[what] = ratio
    assert ratio > 1.0, f'the check must reject {what} (error / bound = {ratio})'

  def slots(self, r, nh, T):
    """Edges of relation r over the hops < nh with target rows < T: (hop, ELL slot, target row, source row) as int64
    tensors, from the arena's ELL blocks, degrees and counters.  A hop of fan-out 0 has no ELL block; its rows must have
    degree 0."""
    eng, ar = self.eng, self.eng.arena
    t = eng.kt[r]
    c = self.ctr[t]
    deg = ar.deg_of(r)
    hs, ss, tg, sr = [], [], [], []
    for h in range(nh):
      k = eng.fan[r][h]
      n = max(0, min(c[h + 1] - c[h], eng.cap_rows[t][h], T - c[h]))
      if n <= 0:
        continue
      if k == 0:
        assert not bool(deg[c[h]:c[h] + n].any()), f'rows of hop {h} (fan-out 0) must have degree 0'
        continue
      e = ar.ell_of(r, h).view(-1, k)[:n].long()
      m = (torch.arange(k, device=DEV).unsqueeze(0) < deg[c[h]:c[h] + n].long().unsqueeze(1)) & (e >= 0)
      rows = torch.arange(n, device=DEV).unsqueeze(1).expand(n, k)
      ss.append((rows * k + torch.arange(k, device=DEV))[m])
      tg.append((rows + c[h])[m])
      sr.append(e[m])
      hs.append(torch.full_like(ss[-1], h))
    z = torch.zeros(0, dtype=torch.int64, device=DEV)
    return torch.cat(hs + [z]), torch.cat(ss + [z]), torch.cat(tg + [z]), torch.cat(sr + [z])

  # ---- fp32 accumulators chained in float64
  def chain_zero(self, buf, T):
    self.chain[buf.data_ptr()] = [torch.zeros(buf.shape, dtype=torch.float64, device=DEV),
                                  torch.zeros(buf.shape, dtype=torch.float64, device=DEV)]

  def chain_add(self, buf, rows, ref, bound):
    v = self.chain.get(buf.data_ptr())
    assert v is not None, 'an fp32 accumulator added to before it was cleared in this step'
    n = ref.shape[0]
    v[1][:n] += bound + EPS32 * (v[0][:n].abs() + ref.abs())
    v[0][:n] += ref

  def chain_check(self, stage, buf, got):
    v = self.chain[buf.data_ptr()]
    n = got.shape[0]
    self.R.check(stage, _ratio(got, v[0][:n], v[1][:n]))
    return v


def _gemm_key(eng, plan):
  for k, v in eng._plans.items():
    if v is plan:
      return k
  raise AssertionError('a TcGemm plan outside the engine')


def _gemm_rows(op, a):
  """Rows (forward / dgrad) or contraction length (wgrad) a TcGemm op takes from its counter."""
  kind, args = op
  if kind == 'fwd':
    ctr, idx, rows = args[5], args[6], args[4].shape[0]
  else:
    ctr, idx, rows = args[3], args[4], args[0].shape[0]
  return max(0, min(int(a.ctr_of(ctr)[idx]), rows))


def _check_gemm(a, L, stage, spec):
  """Check one recorded TcGemm run against `spec`: the model's list of ops, each ('fwd', A, W, b, relu, out, T) /
  ('wgrad', dP, A, gW name, T) / ('dgrad', dP, W, out, T), with W / b pre-step parameters (or a model buffer).  The
  ops that share a gradient slice (a shared W_src) are summed."""
  R = a.R
  kinds = [op[0] for op in L.plan.ops]
  assert kinds == [s[0] for s in spec], f'{stage}: ops {kinds}, the model needs {[s[0] for s in spec]}'
  wg = collections.OrderedDict()
  for op, s in zip(L.plan.ops, spec):
    if s[0] == 'fwd':
      _, A, W, b, relu, out, T = s
      assert _gemm_rows(op, a) == T, f'{stage}: forward over {_gemm_rows(op, a)} rows, the model has {T}'
      Ain = L.pre(A)
      _check_linear(R, f'{stage}', Ain, W, b if b is not None else torch.zeros(W.shape[0], device=DEV),
                    L.post(out), T, relu)
    elif s[0] == 'wgrad':
      _, dP, A, gname, T = s
      assert _gemm_rows(op, a) == T, f'{stage}: wgrad over {_gemm_rows(op, a)} rows, the model has {T}'
      dPin, Ain = L.pre(dP), L.pre(A)
      tail = min(dPin.shape[0], _round(T, 64))
      R.exact(f'{stage} dP tail', bool((dPin[T:tail] == 0).all()))
      Pd, Ad = dPin[:T].double(), Ain[:T].double()
      ent = wg.setdefault(gname, [0, 0, []])
      ent[0] = ent[0] + Pd.t() @ Ad
      ent[1] = ent[1] + gemm_bound(None, Pd.abs().t() @ Ad.abs(), T, bf16_out=False)
      ent[2].append((dPin, Ain, T, dP))
    else:
      _, dP, W, out, T = s
      assert _gemm_rows(op, a) == T, f'{stage}: dgrad over {_gemm_rows(op, a)} rows, the model has {T}'
      Pd, Wd = L.pre(dP)[:T].double(), W.double()
      ref = Pd @ Wd
      bound = gemm_bound(ref, Pd.abs() @ Wd.abs(), W.shape[0])
      R.check(f'{stage} dgrad', _ratio(L.post(out)[:T], ref, bound))
      a.dgrad[out.data_ptr()] = (ref, bound)
  for gname, (ref, bound, parts) in wg.items():
    gbuf = a.eng.param(gname, True) if isinstance(gname, tuple) else gname
    got, before = L.post(gbuf), L.pre(gbuf)
    # the weight gradient starts from zero: gradients are cleared by zero_grads, the dense HGT buffers by hgt_blocks
    R.exact(f'{stage} dW start', bool((before == 0).all()))
    R.check(f'{stage} dW', _ratio(got.view(ref.shape), ref, bound))
    stale = a.dense_stale.get(gbuf.data_ptr()) if not isinstance(gname, tuple) else None
    if a.controls and stale is not None and 'a dense g_att not cleared' not in a.negatives:
      # the previous layer's dense gradient left in the buffer: this wgrad would start from it (the start check) and
      # its result would carry it (the dW check)
      stale = stale.reshape(-1)[:ref.numel()].view(ref.shape)
      if bool(stale.any()):
        bad = got.view(ref.shape).double() + stale.double()
        a.negative('a dense g_att not cleared', float('inf') if bool((before + stale != 0).any()) else 0.0)
        a.negative('a dense g_att not cleared (dW)', _ratio(bad, ref, bound))
    if a.controls and len(parts) == 2:
      # a shared weight must receive both contributions
      dPin, Ain, T, _ = parts[1]
      one = got.view(ref.shape).double() - dPin[:T].double().t() @ Ain[:T].double()
      a.negative('a shared weight missing one contribution', _ratio(one, ref, bound))
    dPin, Ain, T, dPm = parts[0]
    if a.controls and 'a stale 64-row tail before wgrad' not in a.negatives and \
        T + 64 <= min(dPin.shape[0], Ain.shape[0]):
      # the previous, larger step's rows past T left in dP: their products with the A rows past T
      stale = a.prev_tail(dPm, T).double().t() @ Ain[T:T + 64].double()
      if bool(stale.any()):
        a.negative('a stale 64-row tail before wgrad', _ratio(got.view(ref.shape).double() + stale, ref, bound))


def _check_gather(a, u, X0, feats):
  """X0[u]: the feature rows of every sampled node of u bit for bit (MXFP8: the de-quantised rows); rows past the
  device count are zero."""
  eng = a.eng
  n = min(X0.shape[0], eng.cap_nodes[u])
  cnt = min(a.ctr[u][eng.L + 1], n)
  ref = feats[u][eng.arena.nodes_of(u)[:cnt]].to(torch.bfloat16)
  a.R.exact('X0', torch.equal(X0[:cnt], ref))
  a.R.exact('X0 tail', bool((X0[cnt:n] == 0).all()))


def _check_common(a, L, st):
  """zero_grads and softmax_nll (with the head's bias gradient); True when handled."""
  eng, R = a.eng, a.R
  if L.name == 'zero_grads':
    R.exact('zero_grads', bool((L.post(eng.g32) == 0).all()) and float(L.post(eng.loss)) == 0.0 and
            int(L.post(eng.correct)) == 0)
    a.mark('zero_grads')
    return True
  if L.name == 'softmax_nll':
    T = a.T(st, 1, eng.logits.shape[0])
    bg = L.post(eng.param(('head_b',), True))
    R.exact('head_b grad start', bool((L.pre(eng.param(('head_b',), True)) == 0).all()))
    _check_softmax(R, L.pre(eng.logits), eng.C, eng.labels, eng.arena.nodes_of(st), T, L.post(eng.dlogits), bg,
                   L.post(eng.loss), L.post(eng.correct))
    R.exact('dlogits tail', bool((L.post(eng.dlogits)[T:_round(T, 64)] == 0).all()))
    a.mark('softmax_nll')
    return True
  return False


def _head_spec(a, st, dZ):
  eng = a.eng
  T = a.T(st, 1, eng.logits.shape[0])
  Z = eng.Z[eng.L][st]
  if dZ is None:
    return [('fwd', Z, a.p16(('head_W',)), a.p16(('head_b',)), False, eng.logits, T)]
  return [('wgrad', eng.dlogits, Z, ('head_W',), T), ('dgrad', eng.dlogits, a.p16(('head_W',)), dZ, T)]


CONTROLS = {
    HeteroGatEngine: {'a stale 64-row tail before wgrad', 'dP32 not re-zeroed', 'two relations swapped',
                      'the dropout scale missing', 'a backward without the dropout scale',
                      'a shared weight missing one contribution', 'Adam without weight decay',
                      'Adam with t off by one'},
    HeteroHgtEngine: {'a stale 64-row tail before wgrad', 'dKV32 not re-zeroed', 'a dense g_att not cleared',
                      'a dense g_att not cleared (dW)', 'skip_g with the sign of (A - X) flipped',
                      'Adam without weight decay', 'Adam with t off by one'},
}


def _finish(a, expected, step_controls):
  eng, R = a.eng, a.R
  for what, ratio in _check_adam(R, eng, a.snap, eng.wd, step_controls and eng.wd > 0).items():
    a.negative(what, ratio)
  a.mark('adam_step')
  if step_controls:
    ran = set(a.negatives)
    assert ran == CONTROLS[type(eng)], f'negative controls that did not run: {CONTROLS[type(eng)] - ran}'
  R.exact('padded head_W rows', bool((eng.param(('head_W',)).float()[eng.C:] == 0).all()) and
          bool((eng.p32[eng.param_index[('head_W',)][0]:][:eng.n_out_pad * eng.hidden]
                .view(eng.n_out_pad, eng.hidden)[eng.C:] == 0).all()))
  missing = expected - a.seen
  extra = a.seen - expected
  assert not missing, f'stages the model requires that never ran: {sorted(missing)}'
  assert not extra, f'launches the model does not have: {sorted(extra)}'


# --------------------------------------------------------------------------- R-GAT
def _heads_dot(X, Y, heads):
  """per-row, per-head dot products of [E, H] rows (float64), and of their absolute values"""
  E, H = X.shape
  x, y = X.double().view(E, heads, H // heads), Y.double().view(E, heads, H // heads)
  return (x * y).sum(-1), (x.abs() * y.abs()).sum(-1)


def _expand(v, heads, H):
  """[rows, heads] -> [rows, H] (each head's value over its C columns)"""
  return v.unsqueeze(-1).expand(v.shape[0], heads, H // heads).reshape(v.shape[0], H)


def _gat_ident(eng, L):
  """(kind, layer, relation or type) of a native launch of the R-GAT step, from its arguments."""
  n, A = L.name, L.args
  ps = {eng.Ps[k].data_ptr(): k for k in eng.Ps}
  if n in ('gat_scores', 'gat_aggregate', 'gat_score_bwd'):
    return ps[A[0].data_ptr()]
  if n == 'gat_backward':
    return ps[A[1].data_ptr()]
  if n in ('zero_rows', 'add_block_f32'):
    buf = A[0] if n == 'zero_rows' else A[5]
    for l in range(1, eng.L):
      for u, b in eng.dH[l].items():
        if b.data_ptr() == buf.data_ptr():
          return l, u
  raise AssertionError(f'{n}: no stage of the model')


def _gat_audit(a, log, feats, step_controls):
  eng, R = a.eng, a.R
  Lyr, H, hd = eng.L, eng.hidden, eng.heads
  C = H // hd
  st = eng.tid[eng.seed_type]
  p = eng.dropout
  dscale = _f32(1.0 / (1.0 - p))
  expected = collections.Counter()
  for l in range(1, Lyr + 1):
    for t in eng.targets[l]:
      for r in eng.in_rel[l][t]:
        for k in ('proj', 'scores', 'aggregate', 'backward', 'score_bwd', 'wgrad') + (('dgrad',) if l > 1 else ()):
          expected[(k, l, r)] += 1
        if l > 1:
          expected[('add_block', l - 1, eng.nt[r])] += 1
          if eng.Pd[(l, r)] is not None:
            expected[('add_block', l - 1, t)] += 1
    if l < Lyr:
      for u in eng.targets[l]:
        expected[('zero_rows', l, u)] += 1
        expected[('act_bwd', l, u)] += 1
  for k in ('zero_grads', 'softmax_nll', 'head fwd', 'head bwd', 'adam_step'):
    expected[(k,)] += 1
  expected[('act_bwd', Lyr, st)] += 1
  for u in eng.in_types:
    _check_gather(a, u, eng.X0[u], feats)
  acc = {}                                   # (l, t) -> [float64 relation sum, bound, covered rows]
  for L in log:
    if _check_common(a, L, st):
      continue
    if L.name == 'adam_step':
      continue
    if L.name == 'gemm':
      key = _gemm_key(eng, L.plan)
      if key[0] == 'head':
        spec = _head_spec(a, st, None if key[1] else eng.G[Lyr][st])
        _check_gemm(a, L, 'head', spec)
        a.mark('head fwd' if key[1] else 'head bwd')
        continue
      _, kind, l, r = key
      nh = Lyr - l + 1
      s, t = eng.nt[r], eng.kt[r]
      ns, ntr, Ps, Pd = eng._views(l, r)
      Ts, Tt = a.T(s, nh + 1, ns), a.T(t, nh, ntr)
      Xs, Xt = eng._X(l - 1, s), eng._X(l - 1, t)[:ntr]
      wname = ('W_dst', l, r) if ('W_dst', l, r) in eng.param_index else ('W_src', l, r)
      if kind == 'proj':
        spec = [('fwd', Xs, a.p16(('W_src', l, r)), None, False, Ps, Ts)]
        if Pd is not None:
          spec.append(('fwd', Xt, a.p16(wname), None, False, Pd, Tt))
      elif kind == 'wgrad':
        spec = [('wgrad', eng.dPs[r][:ns], Xs, ('W_src', l, r), Ts)]
        if Pd is not None:
          spec.append(('wgrad', eng.dPd[r][:ntr], Xt, wname, Tt))
      else:
        spec = [('dgrad', eng.dPs[r][:ns], a.p16(('W_src', l, r)), eng.dX[s][:ns], Ts)]
        if Pd is not None:
          spec.append(('dgrad', eng.dPd[r][:ntr], a.p16(wname), eng.dX[t][:ntr], Tt))
      _check_gemm(a, L, f'{kind}{l}', spec)
      a.mark(kind, l, r)
      continue
    if L.name == 'gat_act_bwd':
      bg = L.kwargs['bias_g']
      name = a.grad_name(bg)
      l, t = name[1], eng.kt[name[2]]
      nb = len(eng.in_rel[l][t])
      G = eng.G[l][t]
      T = a.T(t, Lyr - l + 1, G.shape[0])
      if L.args[0] is None:
        Gv = L.pre(G)
      else:
        dH = L.pre(eng.dH[l][t])
        a.chain_check(f'dH{l}', eng.dH[l][t], dH[:T])
        Z = eng.Z[l][t]
        keep = torch.ones_like(Z)
        if p > 0:
          a.nat.dropout_bf16(keep, eng._ctr[t], Lyr - l + 1, p, eng.seed, l, a.snap['step'])
        keep = keep[:T] != 0
        ref, gbound = act_bwd_ref(dH[:T], Z[:T], keep, dscale)
        Gv = L.post(G)
        R.check(f'G{l}', _ratio(Gv[:T], ref, gbound))
        R.exact(f'G{l} tail', bool((Gv[T:] == 0).all()))
        if a.controls and p > 0 and bool((ref != 0).any()):
          a.negative('a backward without the dropout scale', _ratio(Gv[:T].double() / dscale, ref, gbound))
      x = Gv[:T].double()
      b0 = L.pre(bg).view(nb, H).double()
      R.check(f'bias{l}', _ratio(L.post(bg).view(nb, H), b0 + x.sum(0), colsum_bound(x, b0, T)))
      a.mark('act_bwd', l, t)
      continue
    l, x = _gat_ident(eng, L)
    if L.name == 'zero_rows':
      u, buf = x, eng.dH[l][x]
      T = a.T(u, Lyr - l + 1, buf.shape[0])
      R.exact('zero_rows', bool((L.post(buf)[:T] == 0).all()))
      a.chain_zero(buf, T)
      a.mark('zero_rows', l, u)
      continue
    if L.name == 'add_block_f32':
      u, buf = x, eng.dH[l][x]
      dX = eng.dX[u]
      Xin, before, after = L.pre(dX), L.pre(buf), L.post(buf)
      ref, bound = a.dgrad[dX.data_ptr()]
      T = ref.shape[0]                     # the rows of the dgrad that wrote dX, from the counters of its side
      R.exact('add_block rows', a.T_call(L.args[3], L.args[4], buf.shape[0]) == T)
      R.exact('add_block_f32', torch.equal(after[:T], before[:T] + Xin[:T].float()) and
              torch.equal(after[T:], before[T:]))
      a.chain_add(buf, T, ref, bound)
      a.chain_check(f'dH{l}', buf, after[:T])
      a.mark('add_block', l, u)
      continue
    r = x
    nh = Lyr - l + 1
    s, t = eng.nt[r], eng.kt[r]
    rels = eng.in_rel[l][t]
    j = rels.index(r)
    ns, ntr, Ps, Pd = eng._views(l, r)
    Ts, Tt = a.T(s, nh + 1, ns), a.T(t, nh, ntr)
    Pdst = Pd if Pd is not None else Ps[:ntr]
    if L.name == 'gat_scores':
      for got, P, att, T in ((L.post(eng.as_[r][:ns]), Ps, a.p16(('att_src', l, r)), Ts),
                             (L.post(eng.ad_[r][:ntr]), Pdst, a.p16(('att_dst', l, r)), Tt)):
        ref, ab = _heads_dot(P[:T], att.unsqueeze(0).expand(T, H), hd)
        R.check('scores', _ratio(got[:T], ref, gat_score_bound(ab, C)))
      R.exact('dsrc cleared', bool((L.post(eng.dsrc[(l, r)])[:Ts] == 0).all()))
      a.mark('scores', l, r)
      continue
    hop, slot, tg, sr = a.slots(r, nh, Tt)
    al_bufs = eng.alpha[(l, r)]
    if L.name == 'gat_aggregate':
      as_, ad = L.pre(eng.as_[r][:ns]), L.pre(eng.ad_[r][:ntr])
      ga = torch.cat([L.post(al_bufs[h]).view(-1, hd)[slot[hop == h]] for h in range(nh)] +
                     [torch.zeros(0, hd, device=DEV)])
      order = torch.cat([torch.nonzero(hop == h).flatten() for h in range(nh)] +
                        [torch.zeros(0, dtype=torch.int64, device=DEV)])
      tg_o, sr_o = tg[order], sr[order]
      raw32 = as_[sr_o] + ad[tg_o]                           # the kernel's fp32 score sum
      neg = ~(raw32 > 0)
      raw = as_[sr_o].double() + ad[tg_o].double()
      e = torch.where(neg, 0.2 * raw, raw)
      al = softmax_seg(e, tg_o, max(Tt, 1))
      emax = float(e.abs().max()) + 1.0 if e.numel() else 1.0

      def alpha_ratio(g_):
        sign_ok = bool(torch.signbit(g_).eq(neg).all())
        return _ratio(g_.abs(), al, gat_alpha_bound(al, emax)) if sign_ok else float('inf')
      R.check('alpha', alpha_ratio(ga))
      a.alpha_post[(l, r)] = [L.post(al_bufs[h]) for h in range(nh)]
      if a.controls and 'two relations swapped' not in a.negatives:
        # the alpha blocks of an earlier relation into t with the same ELL shape in this relation's place
        for q in rels[:j]:
          other = a.alpha_post.get((l, q))
          if other and all(o.numel() == b.numel() for o, b in zip(other, a.alpha_post[(l, r)])):
            sw = torch.cat([other[h].view(-1, hd)[slot[hop == h]] for h in range(nh)] +
                           [torch.zeros(0, hd, device=DEV)])
            if not torch.equal(sw, ga):
              a.negative('two relations swapped', alpha_ratio(sw))
              break
      w = ga.abs().double()
      terms = (_expand(w, hd, H) * Ps[sr_o].double())
      out = torch.zeros(Tt, H, dtype=torch.float64, device=DEV).index_add_(0, tg_o, terms)
      ab = torch.zeros(Tt, H, dtype=torch.float64, device=DEV).index_add_(0, tg_o, terms.abs())
      deg = torch.bincount(tg_o, minlength=Tt).double().unsqueeze(1)
      if j == 0:
        acc[(l, t)] = [torch.zeros_like(out), torch.zeros_like(out), torch.zeros(Tt, dtype=torch.bool, device=DEV)]
      st_ = acc[(l, t)]
      st_[1] += weighted_sum_bound(out, ab, deg, bf16_out=False) + EPS32 * (st_[0].abs() + out.abs())
      st_[0] += out
      st_[2][tg_o] = True
      if j < len(rels) - 1:
        R.check('acc', _ratio(L.post(eng.acc[t][:ntr])[:Tt], st_[0], st_[1]))
      else:
        bs = torch.stack([a.p16(('bias', l, q)) for q in rels]).double()
        pre = st_[0] + bs.sum(0)
        bound = st_[1] + colsum_bound(bs, st_[0], len(rels))
        Z = L.post(eng.Z[l][t])
        act = l < Lyr
        if act:
          keep = torch.ones_like(Z)
          if p > 0:
            a.nat.dropout_bf16(keep, eng._ctr[t], nh, p, eng.seed, l, L.pre(eng.step_dev))
          keep = (keep[:Tt] != 0).double()
          ref = torch.where(pre > 0, pre, 0.01 * pre) * keep * dscale
          bound = bound * keep * dscale
        else:
          ref, keep = pre, None
        R.check(f'Z{l}', _ratio(Z[:Tt], ref, bound + bf16_ulp(ref)))
        # an isolated target (no edge in any relation): exactly the fp32 bias sum, activation and mask
        iso = ~st_[2]
        o = torch.zeros(H, device=DEV)
        for q in rels:
          o = o + a.p16(('bias', l, q)).float()
        if act:
          o = torch.where(o > 0, o, o * 0.01)
          exp_iso = torch.where(keep[iso] > 0, (o * dscale).unsqueeze(0), torch.zeros_like(o).unsqueeze(0))
        else:
          exp_iso = o.unsqueeze(0).expand(int(iso.sum()), H)
        R.exact('isolated rows', torch.equal(Z[:Tt][iso], exp_iso.to(torch.bfloat16)))
        a.n_iso = getattr(a, 'n_iso', 0) + int(iso.sum())
        if a.controls and act and p > 0:
          a.negative('the dropout scale missing',
                     _ratio(Z[:Tt].double() / dscale, ref, bound + bf16_ulp(ref)) if bool((ref != 0).any())
                     else float('inf'))
      a.mark('aggregate', l, r)
      continue
    if L.name == 'gat_backward':
      ga = torch.cat([L.pre(al_bufs[h]).view(-1, hd)[slot[hop == h]] for h in range(nh)] +
                     [torch.zeros(0, hd, device=DEV)])
      order = torch.cat([torch.nonzero(hop == h).flatten() for h in range(nh)] +
                        [torch.zeros(0, dtype=torch.int64, device=DEV)])
      tg_o, sr_o, hop_o, slot_o = tg[order], sr[order], hop[order], slot[order]
      w = ga.abs().double()
      slope = torch.where(torch.signbit(ga), 0.2, 1.0).double()
      kmax = max(eng.fan[r][:nh])
      G = L.pre(eng.G[l][t])
      dal, adot = _heads_dot(G[tg_o], Ps[sr_o], hd)
      gd = G[tg_o].double() * _expand(w, hd, H)
      ref = torch.zeros(ns, H, dtype=torch.float64, device=DEV).index_add_(0, sr_o, gd)
      ab = torch.zeros_like(ref).index_add_(0, sr_o, gd.abs())
      cnt = torch.bincount(sr_o, minlength=ns).double().unsqueeze(1)
      dP = L.post(eng.dP32[r][:ns])
      bound = weighted_sum_bound(ref, ab, cnt, bf16_out=False)
      R.check('dP32', _ratio(dP, ref, bound))
      if a.controls and bool((ref != 0).any()):
        # not re-zeroed after its use, dP32 would start the next use from these sums
        a.negative('dP32 not re-zeroed', _ratio(dP.double() * 2, ref, bound))
      got_dal = torch.cat([L.post(eng.dal[r][h]).view(-1, hd)[slot_o[hop_o == h]] for h in range(nh)] +
                          [torch.zeros(0, hd, device=DEV)])
      R.check('dal', _ratio(got_dal, dal, gat_score_bound(adot, C)))
      S = torch.zeros(Tt, hd, dtype=torch.float64, device=DEV).index_add_(0, tg_o, w * dal)
      Sab = torch.zeros(Tt, hd, dtype=torch.float64, device=DEV).index_add_(0, tg_o, w * adot)
      ds = w * (dal - S[tg_o]) * slope
      term = w * (adot + Sab[tg_o])
      # the reference reads the kernel's alpha (emax 0); the sums run over a row's slots and a source's edges
      tol = gat_dscore_tol(C, 0.0, kmax + int(cnt.max()) + 10 if cnt.numel() else kmax + 10)
      # (rows of dsrc past the source rows keep an earlier step's values; gat_score_bwd reads rows < Ts only)
      for got, idx, n in ((L.post(eng.dsrc[(l, r)])[:Ts], sr_o, Ts), (L.post(eng.dadst[r][:ntr])[:Tt], tg_o, Tt)):
        ref = torch.zeros(n, hd, dtype=torch.float64, device=DEV).index_add_(0, idx, ds)
        tb = torch.zeros(n, hd, dtype=torch.float64, device=DEV).index_add_(0, idx, term)
        R.check('dscore', _ratio(got, ref, tol * tb + 1e-30))
      a.mark('backward', l, r)
      continue
    assert L.name == 'gat_score_bwd', L.name
    dP = L.pre(eng.dP32[r][:ns]).double()
    da_s, da_d = L.pre(eng.dsrc[(l, r)])[:ns].double(), L.pre(eng.dadst[r][:ntr])[:Tt].double()
    att_s, att_d = a.p16(('att_src', l, r)).double(), a.p16(('att_dst', l, r)).double()
    ref_s = dP[:Ts] + _expand(da_s[:Ts], hd, H) * att_s
    terms_s = dP[:Ts].abs() + _expand(da_s[:Ts].abs(), hd, H) * att_s.abs()
    dst_ref = _expand(da_d, hd, H) * att_d
    dst_terms = _expand(da_d.abs(), hd, H) * att_d.abs()
    if Pd is None:
      m = min(Tt, Ts)
      ref_s[:m] += dst_ref[:m]
      terms_s[:m] += dst_terms[:m]
    dPs = L.post(eng.dPs[r][:ns])
    R.check('dPs', _ratio(dPs[:Ts], ref_s, score_bwd_bound(ref_s, terms_s)))
    R.exact('dPs tail', bool((dPs[Ts:min(ns, _round(Ts, 128))] == 0).all()))
    if Pd is not None:
      dPd = L.post(eng.dPd[r][:ntr])
      R.check('dPd', _ratio(dPd[:Tt], dst_ref, score_bwd_bound(dst_ref, dst_terms)))
      R.exact('dPd tail', bool((dPd[Tt:min(ntr, _round(Tt, 128))] == 0).all()))
    R.exact('dP32 zero', bool((L.post(eng.dP32[r]) == 0).all()))
    Psd = Ps[:Ts].double()
    Pdd = Pdst[:Tt].double()
    for name, da, P, n in ((('att_src', l, r), da_s[:Ts], Psd, Ts), (('att_dst', l, r), da_d, Pdd, Tt)):
      g = eng.param(name, True)
      g0 = L.pre(g).double()
      x = _expand(da, hd, H) * P
      R.check('d' + name[0], _ratio(L.post(g), g0 + x.sum(0), colsum_bound(x, g0, n) + 1e-30))
    a.mark('score_bwd', l, r)
  return expected


# --------------------------------------------------------------------------- HGT
def _hgt_ident(eng, L):
  n, A = L.name, L.args
  if n in ('hgt_blocks',):
    for k, v in eng.att_img.items():
      if v.data_ptr() == A[2].data_ptr():
        return k
  if n in ('hgt_attention', 'hgt_attention_bwd'):
    q = A[0] if n == 'hgt_attention' else A[1]
    for l in range(1, eng.L + 1):
      for t, v in eng.QQ[l].items():
        if v.data_ptr() == q.data_ptr():
          return l, t
  if n in ('hgt_gelu', 'hgt_gate'):
    for l in range(1, eng.L + 1):
      for t, v in (eng.AGG if n == 'hgt_gelu' else eng.A)[l].items():
        if v.data_ptr() == A[0].data_ptr():
          return l, t
  if n in ('zero_rows', 'add_block_f32'):
    buf = A[0] if n == 'zero_rows' else A[5]
    for l in range(0, eng.L):
      for u, b in eng.dH[l].items():
        if b.data_ptr() == buf.data_ptr():
          return l, u
  raise AssertionError(f'{n}: no stage of the model')


def _hgt_audit(a, log, feats, step_controls):
  eng, R = a.eng, a.R
  Lyr, H, hd = eng.L, eng.hidden, eng.heads
  D = H // hd
  st = eng.tid[eng.seed_type]
  scale = _f32(1.0 / math.sqrt(D))
  expected = collections.Counter()
  for u in eng.in_types:
    for k in ('in_fwd', 'in_bwd', 'relu_bwd_cast'):
      expected[(k, 0, u)] += 1
    expected[('zero_rows', 0, u)] += 1
  for l in range(1, Lyr + 1):
    for u in eng.kqv_types[l]:
      for k in ('kqv_fwd', 'kqv_bwd', 'kqv_cast', 'add_block'):
        expected[(k, l, u)] += 1
    for t in eng.targets[l]:
      for k in ('blocks', 'qq_fwd', 'attention', 'msg_fwd', 'gelu', 'a_fwd', 'gate', 'gate_bwd', 'colsum', 'a_bwd',
                'gelu_bwd', 'msg_bwd', 'attention_bwd', 'qq_bwd', 'blocks_grad'):
        expected[(k, l, t)] += 1
    if 1 < l:
      for u in eng.dH[l - 1]:
        expected[('zero_rows', l - 1, u)] += 1
  for k in ('zero_grads', 'softmax_nll', 'head fwd', 'head bwd', 'adam_step'):
    expected[(k,)] += 1
  for u in eng.in_types:
    _check_gather(a, u, eng.X0[u], feats)
  kv_chain = {}
  for L in log:
    if _check_common(a, L, st) or L.name == 'adam_step':
      continue
    if L.name == 'gemm':
      key = _gemm_key(eng, L.plan)
      if key[0] == 'head':
        _check_gemm(a, L, 'head', _head_spec(a, st, None if key[1] else eng.dZL))
        a.mark('head fwd' if key[1] else 'head bwd')
        continue
      _, kind, l, t = key
      nh = Lyr - l + 1
      if kind in ('in_fwd', 'in_bwd'):
        T = a.T(t, Lyr + 1, eng.X0[t].shape[0])
        spec = ([('fwd', eng.X0[t], a.p16(('in_W', t)), a.p16(('in_b', t)), True, eng.Z[0][t], T)]
                if kind == 'in_fwd' else [('wgrad', eng.dPre0[t], eng.X0[t], ('in_W', t), T)])
      elif kind in ('kqv_fwd', 'kqv_bwd'):
        n = eng._rows(l - 1, t)
        T = a.T(t, nh + 1, n)
        if kind == 'kqv_fwd':
          spec = [('fwd', eng.Z[l - 1][t], a.p16(('kqv_W', l, t)), a.p16(('kqv_b', l, t)), False, eng.KQV[l][t], T)]
        else:
          spec = [('wgrad', eng.dKQV[t][:n], eng.Z[l - 1][t], ('kqv_W', l, t), T),
                  ('dgrad', eng.dKQV[t][:n], a.p16(('kqv_W', l, t)), eng.dX[t][:n], T)]
      else:
        n, Rn = eng._rows(l, t), len(eng.in_rel[l][t])
        T = a.T(t, nh, n)
        Q = eng.KQV[l][t][:n, H:2 * H]
        att_img, msg_img = a.images[(l, t)]
        if kind == 'qq_fwd':
          spec = [('fwd', Q, att_img, None, False, eng.QQ[l][t], T)]
        elif kind == 'qq_bwd':
          dQQ = eng._rel_view(eng.dQQ, l, t)
          spec = [('wgrad', dQQ, Q, eng.g_att[t][:Rn * H * H].view(Rn * H, H), T),
                  ('dgrad', dQQ, att_img, eng.dQ[t][:n], T)]
        elif kind == 'msg_fwd':
          spec = [('fwd', eng.U[l][t], msg_img, None, False, eng.AGG[l][t], T)]
        elif kind == 'msg_bwd':
          spec = [('wgrad', eng.dAGG[t][:n], eng.U[l][t], eng.g_msg[t][:Rn * H * H].view(H, Rn * H), T),
                  ('dgrad', eng.dAGG[t][:n], msg_img, eng._rel_view(eng.dU, l, t), T)]
        elif kind == 'a_fwd':
          spec = [('fwd', eng.GE[l][t], a.p16(('a_W', l, t)), a.p16(('a_b', l, t)), False, eng.A[l][t], T)]
        else:
          spec = [('wgrad', eng.dA[t][:n], eng.GE[l][t], ('a_W', l, t), T),
                  ('dgrad', eng.dA[t][:n], a.p16(('a_W', l, t)), eng.dGE[t][:n], T)]
      _check_gemm(a, L, f'{kind}{l}', spec)
      a.mark(kind, l, t)
      continue
    if L.name in ('colsum_bf16', 'hgt_kqv_cast', 'relu_bwd_cast'):
      bg = L.args[3] if L.name != 'relu_bwd_cast' else L.args[5]
      name = a.grad_name(bg)
      if L.name == 'colsum_bf16':
        l, t = name[1], name[2]
        n = eng._rows(l, t)
        T = a.T(t, Lyr - l + 1, n)
        x = L.pre(eng.dA[t][:n])[:T].double()
        a.mark('colsum', l, t)
      elif L.name == 'relu_bwd_cast':
        u = name[1]
        T = a.T(u, Lyr + 1, eng.dPre0[u].shape[0])
        dH = L.pre(eng.dH[0][u])
        a.chain_check('dH0', eng.dH[0][u], dH[:T])
        Z = eng.Z[0][u]
        exp = torch.where(Z[:T] > 0, dH[:T], torch.zeros_like(dH[:T])).to(torch.bfloat16)
        dP = L.post(eng.dPre0[u])
        R.exact('dPre0', torch.equal(dP[:T].view(torch.int16), exp.view(torch.int16)) and bool((dP[T:] == 0).all()))
        x = dP[:T].double()
        a.mark('relu_bwd_cast', 0, u)
      else:
        l, u = name[1], name[2]
        nh = Lyr - l + 1
        n = eng._rows(l - 1, u)
        T = a.T(u, nh + 1, n)
        dkv = L.pre(eng.dKV32[u][:n])
        v = kv_chain.get(u)
        assert v is not None or not bool(dkv.any()), 'dKV32 holds gradients no attention backward wrote'
        if v is not None:
          R.check(f'dKV{l}', _ratio(dkv, v[0][:n], v[1][:n]))
        out = L.post(eng.dKQV[u][:n])
        bits = lambda z: z.contiguous().view(torch.int16)   # noqa: E731
        R.exact('dK', torch.equal(bits(out[:T, :H]), bits(dkv[:T, :H].to(torch.bfloat16))))
        R.exact('dV', torch.equal(bits(out[:T, 2 * H:]), bits(dkv[:T, H:].to(torch.bfloat16))))
        is_t = u in eng.targets[l]
        nq = min(a.ctr[u][nh], T, eng.dQ[u].shape[0]) if is_t else 0
        if is_t:
          R.exact('dQ', torch.equal(out[:nq, H:2 * H], L.pre(eng.dQ[u])[:nq]))
        R.exact('dQ rows >= nq', bool((out[nq:T, H:2 * H] == 0).all()))
        R.exact('dKQV tail', bool((out[T:min(n, _round(T, 128))] == 0).all()))
        R.exact('dKV32 zero', bool((L.post(eng.dKV32[u]) == 0).all()))
        kv_chain.pop(u, None)
        x = out[:T].double()
        a.mark('kqv_cast', l, u)
      b0 = L.pre(bg).double()
      R.check('bias grad', _ratio(L.post(bg), b0 + x.sum(0), colsum_bound(x, b0, x.shape[0])))
      continue
    l, t = _hgt_ident(eng, L)
    if L.name == 'zero_rows':
      buf = eng.dH[l][t]
      T = a.T(t, Lyr - l + 1, buf.shape[0])
      R.exact('zero_rows', bool((L.post(buf)[:T] == 0).all()))
      a.chain_zero(buf, T)
      a.mark('zero_rows', l, t)
      continue
    if L.name == 'add_block_f32':
      u, buf = t, eng.dH[l][t]
      n = eng._rows(l, u)
      T = a.T(u, Lyr - l + 1, n)
      Xin, before, after = L.pre(eng.dX[u][:n]), L.pre(buf), L.post(buf)
      R.exact('add_block_f32', torch.equal(after[:T], before[:T] + Xin[:T].float()) and
              torch.equal(after[T:], before[T:]))
      ref, bound = a.dgrad[eng.dX[u].data_ptr()]
      R.exact('add_block rows', ref.shape[0] == T and a.T_call(L.args[3], L.args[4], buf.shape[0]) == T)
      a.chain_add(buf, T, ref, bound)
      a.chain_check(f'dH{l}', buf, after[:T])
      a.mark('add_block', l + 1, u)
      continue
    nh = Lyr - l + 1
    n, rels = eng._rows(l, t), eng.in_rel[l][t]
    Rn = len(rels)
    T = a.T(t, nh, n)
    if L.name == 'hgt_blocks':
      o = eng.param_index[('att', l, rels[0])][0]
      att = a.snap['p16'][o:o + Rn * H * D].view(Rn, hd, D, D)
      o = eng.param_index[('msg', l, rels[0])][0]
      msg = a.snap['p16'][o:o + Rn * H * D].view(Rn, hd, D, D)
      if 'att_g' not in L.kwargs:
        ref_a, ref_m = block_images(att, msg)
        ia, im = L.post(eng.att_img[(l, t)]), L.post(eng.msg_img[(l, t)])
        R.exact('images', torch.equal(ia.view(torch.int16), ref_a.view(torch.int16)) and
                torch.equal(im.view(torch.int16), ref_m.view(torch.int16)))
        a.images[(l, t)] = (ia, im)
        a.mark('blocks', l, t)
      else:
        att_d = L.pre(eng.g_att[t][:Rn * H * H]).view(Rn * H, H)
        msg_d = L.pre(eng.g_msg[t][:Rn * H * H]).view(H, Rn * H)
        blk_a, blk_m = block_grads(att_d, msg_d, Rn, hd, D)
        ga, gm = eng._blocks('att', l, t, True), eng._blocks('msg', l, t, True)
        ok = torch.equal(L.post(ga), L.pre(ga) + blk_a) and torch.equal(L.post(gm), L.pre(gm) + blk_m)
        R.exact('block gradients', ok and bool((L.pre(ga) == 0).all()) and bool((L.pre(gm) == 0).all()))
        R.exact('dense gradients zero', bool((L.post(eng.g_att[t]) == 0).all()) and
                bool((L.post(eng.g_msg[t]) == 0).all()))
        # what the dense buffer would still hold for the next layer's qq wgrad if this launch did not clear it
        a.dense_stale[eng.g_att[t].data_ptr()] = L.pre(eng.g_att[t])
        a.mark('blocks_grad', l, t)
      continue
    if L.name == 'hgt_gelu':
      X = L.pre(eng.AGG[l][t])[:T].double()
      if 'dY' not in L.kwargs:
        Y = L.post(eng.GE[l][t])
        ref, bound = gelu_ref(X)
        R.check('gelu', _ratio(Y[:T], ref, bound))
        a.mark('gelu', l, t)
      else:
        gy = L.pre(eng.dGE[t][:n])[:T].double()
        dX = L.post(eng.dAGG[t][:n])
        ref, bound = gelu_bwd_ref(X, gy)
        R.check('gelu bwd', _ratio(dX[:T], ref, bound))
        R.exact('dAGG tail', bool((dX[T:min(n, _round(T, 128))] == 0).all()))
        a.mark('gelu_bwd', l, t)
      continue
    if L.name == 'hgt_gate':
      sk = a.p32(('skip', l, t))
      sg = torch.sigmoid(sk.double())
      A_ = L.pre(eng.A[l][t])[:T].double()
      Xz = eng.Z[l - 1][t][:T].double()
      if 'dZ' not in L.kwargs:
        ref, bound = gate_ref(A_, Xz, sg)
        R.check('gate', _ratio(L.post(eng.Z[l][t])[:T], ref, bound))
        a.mark('gate', l, t)
        continue
      dZb = eng.dZL if l == Lyr else eng.dH[l][t]
      gz = L.pre(dZb)[:T].double()
      if l < Lyr:
        a.chain_check(f'dH{l}', dZb, L.pre(dZb)[:T])
      dA = L.post(eng.dA[t][:n])
      ref, bound = gate_da_ref(gz, sg)
      R.check('gate dA', _ratio(dA[:T], ref, bound))
      R.exact('dA tail', bool((dA[T:min(n, _round(T, 128))] == 0).all()))
      below = eng.dH[l - 1][t]
      d0 = L.pre(below)[:T].double()
      refx, bx = gate_dx_ref(d0, gz, sg)
      R.check('gate dX', _ratio(L.post(below)[:T], refx, bx))
      ref0, b0 = gate_dx_ref(torch.zeros_like(gz), gz, sg)
      a.chain_add(below, T, ref0, b0)
      tt = gz * (A_ - Xz)
      dsg = sg * (1 - sg)
      sgr = eng._p32(('skip', l, t), True)
      s0 = L.pre(sgr)
      # the kernel's longest chain of fp32 roundings: each thread's grid-stride share of 8-column vectors, a warp
      # tree (5), the CTA's warps (8) and one atomic per CTA (grid = hgt_gate's launch, capped at 132 * 8 CTAs)
      nvec = H // 8
      grid = min(132 * 8, (n * nvec + 255) // 256)
      per_thread = 8 * ((T * nvec + grid * 256 - 1) // (grid * 256))
      ref_s, bound_s = skip_g_ref(s0, sg, tt, per_thread + 13 + grid)
      R.check('skip_g', _ratio(L.post(sgr), ref_s, bound_s))
      if a.controls and bool(tt.any()):
        wrong = s0.double() + dsg * (gz * (Xz - A_)).sum()
        a.negative('skip_g with the sign of (A - X) flipped', _ratio(wrong, ref_s, bound_s))
      a.mark('gate_bwd', l, t)
      continue
    # the attention and its backward: every edge of every relation into t
    ed = []
    for j, r in enumerate(rels):
      hop, slot, tg, sr = a.slots(r, nh, T)
      ed.append((j, r, hop, slot, tg, sr))
    QQ = L.pre(eng.QQ[l][t])
    tg_all = torch.cat([e[4] for e in ed])
    parts = []
    for j, r, hop, slot, tg, sr in ed:
      K = L.pre(eng.KQV[l][eng.nt[r]])
      qq = QQ[tg, j * H:(j + 1) * H]
      c, cabs = _heads_dot(qq, K[sr, :H], hd)
      pr = (a.p32(('prior', l, r)).float() * scale).double()
      parts.append((c, cabs, pr, K))
    al_pre = torch.cat([torch.cat([L.pre(eng.alpha[(l, r)][h]).view(-1, hd)[slot[hop == h]] for h in range(nh)] +
                                  [torch.zeros(0, hd, device=DEV)]) for j, r, hop, slot, tg, sr in ed])
    # edges of each relation ordered by hop (the concatenation order of the gathers above)
    perm = []
    off = 0
    for j, r, hop, slot, tg, sr in ed:
      perm.append(torch.cat([torch.nonzero(hop == h).flatten() for h in range(nh)] +
                            [torch.zeros(0, dtype=torch.int64, device=DEV)]) + off)
      off += hop.numel()
    perm = torch.cat(perm + [torch.zeros(0, dtype=torch.int64, device=DEV)])
    tg_p = tg_all[perm]
    c_all = torch.cat([p_[0] for p_ in parts] + [torch.zeros(0, hd, dtype=torch.float64, device=DEV)])[perm]
    cabs_all = torch.cat([p_[1] for p_ in parts] + [torch.zeros(0, hd, dtype=torch.float64, device=DEV)])[perm]
    pr_all = torch.cat([p_[2].unsqueeze(0).expand(ed[k][4].numel(), hd) for k, p_ in enumerate(parts)] +
                       [torch.zeros(0, hd, dtype=torch.float64, device=DEV)])[perm]
    src_p = torch.cat([e[5] for e in ed] + [torch.zeros(0, dtype=torch.int64, device=DEV)])[perm]
    rel_p = torch.cat([torch.full_like(e[5], e[0]) for e in ed] + [torch.zeros(0, dtype=torch.int64, device=DEV)])[perm]
    if L.name == 'hgt_attention':
      al_got = torch.cat([torch.cat([L.post(eng.alpha[(l, r)][h]).view(-1, hd)[slot[hop == h]] for h in range(nh)] +
                                    [torch.zeros(0, hd, device=DEV)]) for j, r, hop, slot, tg, sr in ed])
      s = c_all * pr_all
      al = softmax_seg(s, tg_p, max(T, 1))
      arel = hgt_alpha_rel(s, hgt_score_err(cabs_all, pr_all.abs(), s, D), tg_p, max(T, 1))
      R.check('alpha', _ratio(al_got, al, arel * al + 1e-30))
      U = L.post(eng.U[l][t])
      for j, r, hop, slot, tg, sr in ed:
        V = parts[j][3]
        m = rel_p == j
        w = al_got[m].double()
        terms = _expand(w, hd, H) * V[src_p[m], 2 * H:].double()
        ref = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add_(0, tg_p[m], terms)
        ab = torch.zeros_like(ref).index_add_(0, tg_p[m], terms.abs())
        dg = torch.bincount(tg_p[m], minlength=T).double().unsqueeze(1)
        # the reference reads the kernel's alpha: only the summation and the bf16 rounding
        R.check('U', _ratio(U[:T, j * H:(j + 1) * H], ref, weighted_sum_bound(ref, ab, dg)))
      covered = torch.zeros(T, dtype=torch.bool, device=DEV)
      covered[tg_p] = True
      R.exact('U of an empty softmax', bool((U[:T][~covered] == 0).all()))
      a.n_iso = getattr(a, 'n_iso', 0) + int((~covered).sum())
      a.mark('attention', l, t)
      continue
    assert L.name == 'hgt_attention_bwd', L.name
    w = al_pre.double()
    dU = L.pre(eng._rel_view(eng.dU, l, t))
    dal = torch.zeros_like(w)
    dabs = torch.zeros_like(w)
    for j, r, hop, slot, tg, sr in ed:
      m = rel_p == j
      V = parts[j][3]
      dal[m], dabs[m] = _heads_dot(dU[tg_p[m], j * H:(j + 1) * H], V[src_p[m], 2 * H:], hd)
    S = torch.zeros(max(T, 1), hd, dtype=torch.float64, device=DEV).index_add_(0, tg_p, w * dal)
    Sab = torch.zeros(max(T, 1), hd, dtype=torch.float64, device=DEV).index_add_(0, tg_p, w * dabs)
    ds = w * (dal - S[tg_p])
    term = w * (dabs + Sab[tg_p])
    # the reference reads the kernel's alpha (arel 0); the sums run over a row's slots (twice: the softmax sum and
    # dqq) and over a source's edges (dK, dV)
    nrow = int(torch.bincount(tg_p).max()) if tg_p.numel() else 0
    ncnt = int(torch.bincount(src_p).max()) if src_p.numel() else 0
    tol = hgt_bwd_tol(D, 2 * nrow + ncnt + 8, 0.0)
    g = ds * pr_all
    tp = term * pr_all.abs()
    dQQ = L.post(eng._rel_view(eng.dQQ, l, t))
    for j, r, hop, slot, tg, sr in ed:
      m = rel_p == j
      s = eng.nt[r]
      K = parts[j][3]
      qq = QQ[tg_p[m], j * H:(j + 1) * H].double()
      Ks = K[src_p[m], :H].double()
      ref = torch.zeros(T, H, dtype=torch.float64, device=DEV).index_add_(0, tg_p[m], _expand(g[m], hd, H) * Ks)
      b_q = torch.zeros_like(ref).index_add_(0, tg_p[m], _expand(tp[m], hd, H) * Ks.abs())
      R.check('dqq', _ratio(dQQ[:T, j * H:(j + 1) * H], ref, bf16_ulp(ref) + tol * b_q + 1e-30))
      dpr = (ds[m] * c_all[m]).sum(0) * scale
      bpr = (tol + int(m.sum()) * EPS32) * (term[m] * cabs_all[m] * scale).sum(0) + 1e-30
      gp = eng._p32(('prior', l, r), True)
      R.exact('dprior start', bool((L.pre(gp) == 0).all()))
      R.check('dprior', _ratio(L.post(gp), dpr, bpr))
      # dK / dV into the source type's fp32 rows, chained over every attention backward of the layer
      nrows = eng.dKV32[s].shape[0]
      dK = torch.zeros(nrows, H, dtype=torch.float64, device=DEV).index_add_(0, src_p[m], _expand(g[m], hd, H) * qq)
      b_k = torch.zeros_like(dK).index_add_(0, src_p[m], _expand(tp[m], hd, H) * qq.abs())
      du = dU[tg_p[m], j * H:(j + 1) * H].double()
      dV = torch.zeros_like(dK).index_add_(0, src_p[m], _expand(w[m], hd, H) * du)
      b_v = torch.zeros_like(dK).index_add_(0, src_p[m], _expand(w[m], hd, H) * du.abs())
      v = kv_chain.setdefault(s, [torch.zeros(nrows, 2 * H, dtype=torch.float64, device=DEV),
                                  torch.zeros(nrows, 2 * H, dtype=torch.float64, device=DEV)])
      new = torch.cat([dK, dV], 1)
      v[1] += tol * torch.cat([b_k, b_v], 1) + EPS32 * (v[0].abs() + new.abs())
      v[0] += new
    R.exact('dQQ tail', bool((dQQ[T:min(n, _round(T, 128))] == 0).all()))
    for s in sorted({eng.nt[r] for r in rels}):
      v = kv_chain[s]
      got = L.post(eng.dKV32[s])
      R.check('dKV32', _ratio(got, v[0], v[1]))
      if a.controls and bool(v[0].any()) and 'dKV32 not re-zeroed' not in a.negatives:
        # not re-zeroed after its use, dKV32 would start the next use from these sums
        a.negative('dKV32 not re-zeroed', _ratio(got.double() * 2, v[0], v[1]))
    a.mark('attention_bwd', l, t)
  return expected


# --------------------------------------------------------------------------- graphs, configurations and the test
def _star(g):
  """A destination type 'hub' with 8 incoming relations from 4 source types (two each), and reverse relations."""
  sizes = {'hub': 1500, 'a': 900, 'b': 800, 'c': 700, 'd': 600}
  e = {}
  for i, s in enumerate('abcd'):
    for k in range(2):
      e[(s, f'r{i}{k}', 'hub')] = torch.stack([torch.randint(0, sizes[s], (5000,), generator=g),
                                               torch.randint(0, sizes['hub'], (5000,), generator=g)])
    e[('hub', f'back{i}', s)] = torch.stack([torch.randint(0, sizes['hub'], (4000,), generator=g),
                                             torch.randint(0, sizes[s], (4000,), generator=g)])
  return e, sizes


CASES = {
    # name: (engine, graph, options, captured, controls)
    'gat-igbh-wd': ('gat', 'igbh', dict(dims={'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128}, hidden=192,
                                       heads=4, fanouts=[4, 3, 2], dropout=0.2, weight_decay=5e-4), False, False),
    'gat-uniform-captured': ('gat', 'igbh', dict(dims=64, hidden=64, heads=4, fanouts=[4, 3, 2], dropout=0.5,
                                                 weight_decay=5e-4), True, True),
    'gat-hidden-1024': ('gat', 'igbh', dict(dims=128, hidden=1024, heads=8, fanouts=[4, 3], bs=128), False, False),
    'gat-mxfp8-2983': ('gat', 'igbh', dict(dims=64, hidden=64, heads=1, num_classes=2983, fanouts=[4, 3],
                                           mxfp8=True), False, False),
    'gat-fanout-zero': ('gat', 'igbh', dict(dims=64, hidden=64, heads=2, fanouts='zero', dropout=0.2), False, False),
    'hgt-mag-captured': ('hgt', 'mag', dict(dims=64, hidden=64, heads=2, fanouts=[4, 3], weight_decay=5e-4), True,
                         True),
    'hgt-igbh-2983': ('hgt', 'igbh', dict(dims={'paper': 1024, 'author': 256, 'institute': 64, 'fos': 128},
                                          hidden=64, heads=2, fanouts=[4, 3, 2], num_classes=2983), False, False),
    'hgt-mag-704': ('hgt', 'mag', dict(dims=64, hidden=704, heads=8, fanouts=[4, 3]), False, False),
    'hgt-hidden-1024': ('hgt', 'mag', dict(dims=128, hidden=1024, heads=8, fanouts=[4, 3], bs=128), False, False),
    'hgt-8-relations': ('hgt', 'star', dict(dims=64, hidden=64, heads=2, fanouts=[3, 2]), False, False),
}


def _build(name):
  from common import synthetic_igbh, synthetic_mag
  kind, schema, opts, captured, controls = CASES[name]
  opts = dict(opts)
  dims, bs, mxfp8 = opts.pop('dims'), opts.pop('bs', 256), opts.pop('mxfp8', False)
  C = opts.pop('num_classes', 19)
  g = torch.Generator().manual_seed(3)
  if schema == 'star':
    edges, sizes = _star(g)
    seed_type, n_old = 'hub', None
  else:
    make = synthetic_igbh if schema == 'igbh' else synthetic_mag
    edges, _, _, sizes = make(3000, 1500, 50, 30, feat_dim=8, num_classes=C, seed=2)
    per_node = {et: 3 for et in edges if et[0] == 'paper'} if kind == 'hgt' else GAT_ISOLATED_EDGES
    n_old = add_isolated_papers(edges, sizes, ISOLATED, g, per_node)
    seed_type = 'paper'
  if opts['fanouts'] == 'zero':
    fan = {et: [3, 3, 2] for et in edges}
    fan[('fos', 'rev_topic', 'paper')] = [4, 0, 2]           # fos feeds paper at hops 0 and 2 only
    fan[('institute', 'rev_affiliated_to', 'author')] = [0, 3, 0]
    opts['fanouts'] = fan
  labels = torch.randint(0, C, (sizes[seed_type],), generator=g).to(DEV)
  widths = dims if isinstance(dims, dict) else {t: dims for t in sizes}
  graphs, tables, keep, feats = {}, {}, [], {}
  for et, ei in edges.items():
    topo = glt.data.Topology(ei.to(DEV), layout='CSC', num_nodes=sizes[et[2]])
    graphs[et] = glt.data.Graph(topo, 'CUDA', 0)
  for t, n in sizes.items():
    x = torch.randn(n, widths[t], generator=g).to(DEV)
    if mxfp8:
      q = quantize_mxfp8(x)
      feats[t] = dequantize_mxfp8(q, widths[t]).to(torch.bfloat16)
      ut = _table(q)
    else:
      feats[t] = x.to(torch.bfloat16)
      ut = _table(feats[t])
    keep.append(ut)
    tables[t] = ut._table()
  Eng = HeteroGatEngine if kind == 'gat' else HeteroHgtEngine
  eng = Eng(graphs, tables, labels, widths, sizes, seed_type, batch_size=bs, num_classes=C, lr=5e-3, seed=1,
            device=DEV, use_cuda_graph=captured, feature_format='mxfp8' if mxfp8 else 'bf16', **opts)
  eng._keep = keep
  return eng, feats, sizes, seed_type, n_old, captured, controls


@pytest.mark.parametrize('name', list(CASES))
def test_attention_step_stages_match_fp64(native, name):
  eng, feats, sizes, seed_type, n_old, captured, controls = _build(name)
  rec = Recorder(eng.nat)
  eng.nat = rec
  if name == 'hgt-8-relations':
    assert max(len(v) for l in range(1, eng.L + 1) for v in eng.in_rel[l].values()) == 8
  if name == 'gat-fanout-zero':
    assert any(0 in f for f in eng.fan)
  if name == 'gat-igbh-wd':
    assert any(k[0] == 'W_dst' for k in eng.param_index)
  if name == 'gat-uniform-captured':
    assert any(eng.Pd[k] is not None and ('W_dst',) + k not in eng.param_index for k in eng.Pd), 'a shared W_src'
  if captured:
    eng.warmup_and_capture(n_eager=1)
    assert eng._graph is not None and rec.graph_log
  fidx = {eng.tid[t]: feats[t] for t in feats}
  g = torch.Generator().manual_seed(11)
  batches = _batches(eng.bs, n_old if n_old is not None else sizes[seed_type], g)
  if n_old is not None:
    batches[2] = torch.tensor([n_old + 5], device=DEV)       # one isolated paper
  audit = _gat_audit if isinstance(eng, HeteroGatEngine) else _hgt_audit
  prev = {}
  n_iso = 0
  for i, seeds in enumerate(batches):
    snap = _snapshot(eng, lambda: None)
    rec.log = []
    eng.train_step(seeds)
    log = rec.graph_log if captured else rec.log
    R = Ratios(f'{name} step {i}')
    a = Audit(R, eng, snap, controls and i == 1)
    a.nat, a.images, a.prev = rec.nat, {}, prev
    expected = audit(a, log, fidx, controls and i == 1)
    _finish(a, expected, controls and i == 1)
    n_iso += getattr(a, 'n_iso', 0)
    R.show()
    if a.controls:
      print(f'{name} controls (error / bound): ' + ', '.join(f'{k} {v:.3g}' for k, v in a.negatives.items()))
    if controls and i == 0:
      # this step's buffers after its launches: the rows a stale tail would leak into the next, smaller step
      prev = {t.data_ptr(): c.clone() for L in log for t, c in zip(L.tensors, L._post) if t.dtype == torch.bfloat16}
  assert n_iso > 0, 'the batches must hold targets without any in-neighbour'
  eng.close()
