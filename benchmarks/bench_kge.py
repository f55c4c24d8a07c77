#!/usr/bin/env python
"""Knowledge-graph embeddings at FB15k-237 and ogbl-wikikg2 shape: KgeEngine against eager torch, D = 128.

  python benchmarks/bench_kge.py [--models transe,distmult,complex,rotate] [--steps 20 --rounds 3] [--record FILE]

Shapes: FB15k-237 (14,541 entities, 237 relations, 272,115 train and 20,466 test triples) and ogbl-wikikg2
(2,500,604 entities, 535 relations); triples come from `synthetic_kg` at those entity and relation counts.

* step arm, per model at K = 1 and K = 64 negatives, batch 1024, at both shapes: the engine's captured step
  (`train_step`) against eager torch that a user writes today: `nn.Embedding(sparse=True)` tables, the same score and
  loss formulas, uniform corruptions drawn with `torch.randint`, `torch.optim.SparseAdam`.
* rank arm, per model: the engine's filtered rank (`rank`, the k_kge_rank kernel) against chunked torch scoring with the
  same filter (`--chunk` queries at a time: the query vectors of the same formulas, the [chunk, N] score matrix by
  `torch.mm` or `torch.cdist`, filtered ids set to -inf by the sorted `kge_filter` keys, then the counts above and
  tied with the true score).  Two workloads: the whole
  FB15k-237 test set in both directions, and 10,000 tail queries at wikikg2 shape.

Arms alternate for --rounds rounds after a warm-up, device-timed with CUDA events.  Per row: ms, and the bytes and
FLOPs of the work computed from shapes (`step_cost`, `rank_cost`) with the kernel's share of the HBM (3.35 TB/s) or
FP32 (67 TFLOP/s) data-sheet bound, whichever is larger.  The rank arm also reports the largest rank difference
between the arms (the torch arm sums in another order, so near-ties may differ).  The card name and power limit are
read in the same run.  One JSON line is printed, and appended to --record on an H100.
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_inference import card  # noqa: E402

PEAK_FP32 = 67e12
PEAK_HBM = 3.35e12
SHAPES = {'fb15k237': dict(N=14541, R=237, train=272115, test=20466),
          'wikikg2': dict(N=2500604, R=535, train=1_000_000, test=10000)}


def widths(model, D):
  return (2 * D if model in ('complex', 'rotate') else D), (2 * D if model == 'complex' else D)


def step_cost(model, D, B, K, N, R):
  """Bytes and FLOPs of one step from shapes: every looked-up entity row (2 + K per positive) read once and its
  gradient red.added (read + write), the relation row likewise, then SparseAdam reading w, g, m, v and writing w, m, v
  and the zeroed g on at most min(lookups, table rows) rows.  FLOPs: a score and its gradient, ~8 per column and
  triple."""
  We, Wr = widths(model, D)
  rows_e, rows_r = B * (2 + K), B
  look = 4 * (rows_e * We * 3 + rows_r * Wr * 3)
  adam = 4 * 8 * (min(rows_e, N) * We + min(rows_r, R) * Wr)
  return look + adam, 8 * B * (1 + K) * We


def rank_cost(model, D, n, N, sms):
  """FLOPs: one multiply-add (dot) or subtract + multiply-add (distance) per query, candidate and column.  Bytes: the
  candidate table once per wave of CTAs (the resident CTAs sweep the same candidate tiles, so L2 serves the rest),
  plus the query vectors."""
  We, _ = widths(model, D)
  per = 2 if model in ('distmult', 'complex') else 3
  tiles = math.ceil(n / 64)
  splits = max(1, math.ceil(2 * sms / tiles))
  waves = math.ceil(tiles * splits / (2 * sms))
  return waves * N * We * 4 + 3 * n * We * 4, per * n * N * We


def bound_share(ms, nbytes, flops):
  t = max(nbytes / PEAK_HBM, flops / PEAK_FP32)
  return {'share': round(t / (ms * 1e-3), 4), 'bound': 'hbm' if nbytes / PEAK_HBM >= flops / PEAK_FP32 else 'fp32'}


class EagerKge:
  """The same formulas in eager torch: sparse embeddings and torch.optim.SparseAdam."""

  def __init__(self, eng):
    import torch
    self.model, self.D, self.margin, self.p = eng.model, eng.hidden_channels, eng.margin, eng.p_norm
    self.N, self.K = eng.num_nodes, eng.num_negatives
    self.ent = torch.nn.Embedding.from_pretrained(eng.ent.clone(), freeze=False, sparse=True)
    self.rel = torch.nn.Embedding.from_pretrained(eng.rel.clone(), freeze=False, sparse=True)
    self.opt = torch.optim.SparseAdam(list(self.ent.parameters()) + list(self.rel.parameters()), lr=eng.lr)

  def score_rows(self, eh, er, et):
    import torch
    import torch.nn.functional as F
    D = self.D
    if self.model == 'transe':
      x = F.normalize(eh, p=self.p, dim=-1) + er - F.normalize(et, p=self.p, dim=-1)
      return -torch.linalg.vector_norm(x, ord=self.p, dim=-1)
    if self.model == 'distmult':
      return (eh * er * et).sum(-1)
    hr, hi, tr, ti = eh[..., :D], eh[..., D:], et[..., :D], et[..., D:]
    if self.model == 'complex':
      rr, ri = er[..., :D], er[..., D:]
      return (hr * rr * tr + hi * rr * ti + hr * ri * ti - hi * ri * tr).sum(-1)
    c, s = torch.cos(er), torch.sin(er)
    a, b = c * hr - s * hi - tr, c * hi + s * hr - ti
    return self.margin - torch.linalg.vector_norm(torch.cat([a, b], -1), dim=-1)

  def step(self, trip):
    import torch
    import torch.nn.functional as F
    h, r, t = trip
    n = h.numel()
    neg = torch.randint(0, self.N, (n, self.K), device=h.device)
    head = (torch.arange(n, device=h.device) < n // 2).unsqueeze(1)
    nh = torch.where(head, neg, h.unsqueeze(1))
    nt = torch.where(head, t.unsqueeze(1), neg)
    s_pos = self.score_rows(self.ent(h), self.rel(r), self.ent(t))
    s_neg = self.score_rows(self.ent(nh), self.rel(r).unsqueeze(1), self.ent(nt))
    if self.model in ('transe', 'distmult'):
      loss = torch.clamp(self.margin - s_pos.unsqueeze(1) + s_neg, min=0).mean()
    else:
      loss = (F.softplus(-s_pos).sum() + F.softplus(s_neg).sum()) / (n + n * self.K)
    self.opt.zero_grad(set_to_none=True)
    loss.backward()
    self.opt.step()
    return loss


def torch_rank(eager, h, r, t, keys, tail, chunk):
  """Filtered ranks from chunked [chunk, N] score matrices: the query vectors of the formulas (h∘r, n(h) + r, ...),
  then `torch.mm` (DistMult, ComplEx) or `torch.cdist` (TransE, RotatE) against every entity row."""
  import torch
  import torch.nn.functional as F
  N, R, D = eager.N, eager.rel.weight.size(0), eager.D
  E, Rl = eager.ent.weight.detach(), eager.rel.weight.detach()
  model = eager.model
  cand = F.normalize(E, p=eager.p, dim=-1) if model == 'transe' else E
  out = []
  for a in range(0, h.numel(), chunk):
    hh, rr, tt = h[a:a + chunk], r[a:a + chunk], t[a:a + chunk]
    m = hh.numel()
    f, truth = (hh, tt) if tail else (tt, hh)
    fe, re_ = E[f], Rl[rr]
    if model == 'transe':
      q = F.normalize(fe, p=eager.p, dim=-1) + (re_ if tail else -re_)
    elif model == 'distmult':
      q = fe * re_
    else:
      if model == 'complex':
        cr, ci = re_[:, :D], re_[:, D:]
      else:
        cr, ci = torch.cos(re_), torch.sin(re_)
      ci = ci if tail else -ci
      q = torch.cat([fe[:, :D] * cr - fe[:, D:] * ci, fe[:, D:] * cr + fe[:, :D] * ci], 1)
    if model in ('distmult', 'complex'):
      s = q @ cand.T
    elif model == 'transe':
      s = -torch.cdist(q, cand, p=eager.p)
    else:
      s = eager.margin - torch.cdist(q, cand)
    base = (f * R + rr) * N
    st = s.gather(1, truth.unsqueeze(1))
    s[torch.arange(m, device=s.device), truth] = float('-inf')
    lo, hi = torch.searchsorted(keys, base), torch.searchsorted(keys, base + N)
    cnt = hi - lo
    row = torch.repeat_interleave(torch.arange(m, device=s.device), cnt)
    pos = torch.arange(int(cnt.sum()), device=s.device) - torch.repeat_interleave(torch.cumsum(cnt, 0) - cnt, cnt)
    col = keys[torch.repeat_interleave(lo, cnt) + pos] - torch.repeat_interleave(base, cnt)
    s[row, col] = float('-inf')
    out.append(1 + (s > st).sum(1).double() + 0.5 * (s == st).sum(1).double())
  return torch.cat(out)


def timed(fn, rounds):
  import torch
  ts = []
  for _ in range(rounds):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
  return ts


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--models', default='transe,distmult,complex,rotate')
  p.add_argument('--shapes', default='fb15k237,wikikg2')
  p.add_argument('--negatives', default='1,64')
  p.add_argument('--dim', type=int, default=128)
  p.add_argument('--batch', type=int, default=1024)
  p.add_argument('--steps', type=int, default=20)
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--chunk', type=int, default=256)
  p.add_argument('--no-rank', action='store_true')
  p.add_argument('--record', default=os.path.join(ROOT, 'profiles', 'bench_kge_h100.json'))
  args = p.parse_args()
  import torch
  from graphlearn_for_pytorch_b200.models import KgeEngine, kge_filter
  from graphlearn_for_pytorch_b200.utils.synthetic import synthetic_kg
  assert torch.cuda.is_available(), 'bench_kge measures on a GPU'
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  sms = torch.cuda.get_device_properties(dev).multi_processor_count
  D, B = args.dim, args.batch
  result = {'bench': 'kge', 'card': card(), 'dim': D, 'batch': B, 'steps': args.steps, 'rounds': args.rounds,
            'step': [], 'rank': []}
  for shape in args.shapes.split(','):
    sh = SHAPES[shape]
    N, R = sh['N'], sh['R']
    train, valid, test = synthetic_kg(N, R, sh['train'] * 10 // 8 + sh['test'] * 2, seed=0)
    test = test[:, :sh['test']].to(dev)
    train = train.to(dev)
    flt = kge_filter(torch.cat([train, valid.to(dev), test], 1), N, R)
    for model in args.models.split(','):
      for K in (int(k) for k in args.negatives.split(',')):
        eng = KgeEngine(N, R, model=model, hidden_channels=D, num_negatives=K, batch_size=B, seed=0, device=dev)
        eng.warmup_and_capture()
        eager = EagerKge(eng)
        batches = [train[:, i * B:(i + 1) * B].contiguous() for i in range(args.steps)]
        run_e = lambda: [eng.train_step(b) for b in batches]           # noqa: E731
        run_t = lambda: [eager.step(b) for b in batches]                # noqa: E731
        run_e(), run_t()
        torch.cuda.synchronize()
        te, tt = [], []
        for _ in range(args.rounds):
          te += timed(run_e, 1)
          tt += timed(run_t, 1)
        ms_e, ms_t = statistics.median(te) / args.steps, statistics.median(tt) / args.steps
        nbytes, flops = step_cost(model, D, B, K, N, R)
        row = {'shape': shape, 'model': model, 'K': K, 'engine_ms': round(ms_e, 4), 'torch_ms': round(ms_t, 4),
               'speedup': round(ms_t / ms_e, 2), 'kernels_per_step': eng.kernels_per_step, 'bytes': nbytes,
               'flops': flops, **bound_share(ms_e, nbytes, flops)}
        result['step'].append(row)
        print(json.dumps(row), flush=True)
        if args.no_rank or K != int(args.negatives.split(',')[0]):
          del eng, eager
          torch.cuda.empty_cache()
          continue
        with torch.no_grad():                       # both arms rank the engine's trained tables
          eager.ent.weight.copy_(eng.ent)
          eager.rel.weight.copy_(eng.rel)
        qs = test if shape == 'fb15k237' else test[:, :10000]
        modes = (True, False) if shape == 'fb15k237' else (True,)
        h, r, t = qs
        run_e = lambda: [eng.rank(h, r, t, mode='tail' if m else 'head', filter=flt) for m in modes]   # noqa: E731
        run_t = lambda: [torch_rank(eager, h, r, t, flt[0] if m else flt[1], m, args.chunk) for m in modes]  # noqa
        ke, kt = run_e(), run_t()
        diff = max(float((a - b).abs().max()) for a, b in zip(ke, kt))
        same = sum(int((a == b).sum()) for a, b in zip(ke, kt)) / sum(a.numel() for a in ke)
        te, tt = [], []
        for _ in range(args.rounds):
          te += timed(run_e, 1)
          tt += timed(run_t, 1)
        ms_e, ms_t = statistics.median(te), statistics.median(tt)
        n = h.numel() * len(modes)
        nbytes, flops = rank_cost(model, D, h.numel(), N, sms)
        nbytes, flops = nbytes * len(modes), flops * len(modes)
        row = {'shape': shape, 'model': model, 'queries': n, 'engine_ms': round(ms_e, 3), 'torch_ms': round(ms_t, 3),
               'speedup': round(ms_t / ms_e, 2), 'max_rank_diff': diff, 'equal_ranks': round(same, 5),
               'bytes': nbytes, 'flops': flops, 'tflops': round(flops / (ms_e * 1e-3) / 1e12, 2),
               **bound_share(ms_e, nbytes, flops)}
        result['rank'].append(row)
        print(json.dumps(row), flush=True)
        del eng, eager
        torch.cuda.empty_cache()
  line = json.dumps(result)
  print(line)
  if args.record and 'H100' in result['card']['name']:
    with open(args.record, 'a') as f:
      f.write(line + '\n')


if __name__ == '__main__':
  main()
