"""Full-neighbourhood layer-wise inference of the heterogeneous engines against a PyTorch arm of the same math, in one
call.

  python benchmarks/bench_hetero_inference.py --model rsage|rgat|hgt

Shapes: --model rsage / rgat use the defaults of bench_hetero_rgnn.py (synthetic IGBH: 200,000 papers, 1024-wide
features, hidden 512, 3 layers, 4 heads for R-GAT); --model hgt those of bench_hgt.py (synthetic ogbn-mag node counts,
128-wide features, hidden 64, 2 heads, 2 layers).  Parameters are the engine's seeded initialisation.

Arms:
  engine  `inference()`: every node of every needed type, layer by layer (CUDA kernels of csrc/cuda/sage_infer.cu,
          hetero_infer.cu and the TcGemm GEMMs)
  torch   the same layers over the CSR with segment mean / segment softmax (`scatter_reduce`, `index_add_`) in fp32
          and bf16 matmuls, no custom kernels

Both are device-timed with CUDA events: the median of --calls calls after --warmup calls.  The engine's per-layer times
(the input layer, each layer, the head) come from events around its layer calls in the last timed call.  Agreement is
the max |engine - torch| and the argmax agreement of the logits on --sample seed-type nodes.  The card name and power
limit are read in the same run.  One JSON line is printed.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'examples'))

MAG = dict(num_papers=736_389, num_authors=1_134_649, num_insts=8_740, num_fields=59_965)


def card():
  try:
    r = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True, timeout=30)
    power = r.stdout.strip() or None
  except Exception as e:  # the number is still reported, without its power limit
    power = f'unavailable: {type(e).__name__}'
  return {'name': torch.cuda.get_device_name(0), 'power_limit': power}


def timed(fn, warmup, calls):
  for _ in range(warmup):
    out = fn()
  torch.cuda.synchronize()
  ms = []
  for _ in range(calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
  return statistics.median(ms), ms, out


# --------------------------------------------------------------------------- PyTorch arm
def bf16_mm(x, w, b=None):
  y = (x.to(torch.bfloat16) @ w.to(torch.bfloat16).t()).float()
  return y + b.float() if b is not None else y


def seg_softmax(e, dst, n):
  heads = e.shape[1]
  m = torch.full((n, heads), -float('inf'), device=e.device).scatter_reduce(
      0, dst.unsqueeze(1).expand(-1, heads), e, 'amax', include_self=True)
  ex = torch.exp(e - m[dst])
  den = torch.zeros(n, heads, device=e.device).index_add_(0, dst, ex)
  return ex / den[dst]


def torch_rsage(eng, csr, feats, n):
  X = {t: feats[eng.ntypes[t]] for t in range(len(eng.ntypes))}
  for l in range(1, eng.L + 1):
    Z = {}
    for t in eng.targets[l]:
      blocks = []
      for r in eng.in_rel[l][t]:
        dst, src, deg = csr[r]
        blocks.append(torch.zeros(n[t], X[eng.nt[r]].shape[1], device=dst.device)
                      .index_add_(0, dst, X[eng.nt[r]][src].float()) / deg)
      z = bf16_mm(torch.cat(blocks + [X[t].float()], 1), eng.param(('W', l, t)), eng.param(('b', l, t)))
      Z[t] = (F.relu(z) if l < eng.L else z).to(torch.bfloat16)
    X = Z
  return X[eng.tid[eng.seed_type]][:, :eng.C]


def torch_rgat(eng, csr, feats, n):
  H, hd = eng.hidden, eng.heads
  C = H // hd
  X = {t: feats[eng.ntypes[t]] for t in range(len(eng.ntypes))}
  for l in range(1, eng.L + 1):
    Z = {}
    for t in eng.targets[l]:
      pre = torch.zeros(n[t], H, device=X[t].device)
      for r in eng.in_rel[l][t]:
        s = eng.nt[r]
        dst, src, _ = csr[r]
        hs = bf16_mm(X[s], eng.param(('W_src', l, r))).to(torch.bfloat16).float()
        gd = hs if s == t else bf16_mm(X[t], eng._w_dst(l, r)).to(torch.bfloat16).float()
        a_s = (hs.view(-1, hd, C) * eng.param(('att_src', l, r)).float().view(hd, C)).sum(-1)
        a_d = (gd.view(-1, hd, C) * eng.param(('att_dst', l, r)).float().view(hd, C)).sum(-1)
        al = seg_softmax(F.leaky_relu(a_s[src] + a_d[dst], 0.2), dst, n[t])
        pre.index_add_(0, dst, (al.unsqueeze(-1) * hs[src].view(-1, hd, C)).view(-1, H))
        pre += eng.param(('bias', l, r)).float()
      Z[t] = (F.leaky_relu(pre, 0.01) if l < eng.L else pre).to(torch.bfloat16)
    X = Z
  return bf16_mm(X[eng.tid[eng.seed_type]], eng.param(('head_W',)), eng.param(('head_b',)))[:, :eng.C]


def torch_hgt(eng, csr, feats, n):
  H, hd = eng.hidden, eng.heads
  D = H // hd
  p = eng.param
  X = {u: F.relu(bf16_mm(feats[eng.ntypes[u]], p(('in_W', u)), p(('in_b', u)))).to(torch.bfloat16)
       for u in eng.in_types}
  for l in range(1, eng.L + 1):
    KQV = {u: bf16_mm(X[u], p(('kqv_W', l, u)), p(('kqv_b', l, u))).to(torch.bfloat16) for u in eng.kqv_types[l]}
    Z = {}
    for t in eng.targets[l]:
      rels = eng.in_rel[l][t]
      Q = KQV[t][:, H:2 * H]
      scores, dsts = [], []
      for r in rels:
        dst, src, _ = csr[r]
        qq = bf16_mm(Q, torch.block_diag(*p(('att', l, r)).float()))
        k = KQV[eng.nt[r]][:, :H].float()
        sc = (qq[dst].view(-1, hd, D) * k[src].view(-1, hd, D)).sum(-1) * eng._p32(('prior', l, r)) / math.sqrt(D)
        scores.append(sc)
        dsts.append(dst)
      al = seg_softmax(torch.cat(scores), torch.cat(dsts), n[t]).split([s.shape[0] for s in scores])
      agg = torch.zeros(n[t], H, device=Q.device)
      for r, a in zip(rels, al):
        dst, src, _ = csr[r]
        v = KQV[eng.nt[r]][:, 2 * H:].float()
        u = torch.zeros(n[t], H, device=Q.device).index_add_(0, dst, (a.unsqueeze(-1) * v[src].view(-1, hd, D))
                                                               .view(-1, H))
        agg += bf16_mm(u, torch.block_diag(*p(('msg', l, r)).float()).t())
      ge = F.gelu(agg.to(torch.bfloat16).float())
      a_ = bf16_mm(ge, p(('a_W', l, t)), p(('a_b', l, t)))
      g = torch.sigmoid(eng._p32(('skip', l, t)))
      Z[t] = (g * a_ + (1 - g) * X[t].float()).to(torch.bfloat16)
    X = Z
  return bf16_mm(X[eng.tid[eng.seed_type]], p(('head_W',)), p(('head_b',)))[:, :eng.C]


ARMS = {'rsage': torch_rsage, 'rgat': torch_rgat, 'hgt': torch_hgt}


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--model', default='rsage', choices=list(ARMS))
  p.add_argument('--calls', type=int, default=5)
  p.add_argument('--warmup', type=int, default=1)
  p.add_argument('--sample', type=int, default=10000)
  p.add_argument('--chunk-rows', type=int, default=None)
  p.add_argument('--feat-format', default='bf16', choices=['bf16', 'mxfp8'],
                 help='feature storage of every node type; with mxfp8 the PyTorch arm reads the de-quantised rows')
  args = p.parse_args()
  import graphlearn_for_pytorch_b200 as glt
  from common import synthetic_igbh, synthetic_mag
  from graphlearn_for_pytorch_b200.models import HeteroGatEngine, HeteroHgtEngine, HeteroSageEngine
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  if args.model == 'hgt':
    feat_dim, hidden, classes, fan, heads = 128, 64, 349, [10, 10], 2
    edges, feats, _, sizes = synthetic_mag(**MAG, feat_dim=feat_dim, num_classes=classes)
  else:
    feat_dim, hidden, classes, fan, heads = 1024, 512, 19, [15, 10, 5], 4
    papers = 200_000
    edges, feats, _, sizes = synthetic_igbh(papers, papers // 2, max(papers // 400, 8), max(papers // 1000, 8),
                                            feat_dim=feat_dim, num_classes=classes)
  graphs, tables, keep, fdev, csr = {}, {}, [], {}, {}
  for et, ei in edges.items():
    graphs[et] = glt.data.Graph(glt.data.Topology(ei.to(dev), layout='CSC', num_nodes=sizes[et[2]]), 'CUDA', 0)
  for t, x in feats.items():
    rows = fdev[t] = x.to(dev).to(torch.bfloat16)
    if args.feat_format == 'mxfp8':
      rows = glt.data.quantize_mxfp8_chunked(rows)
      fdev[t] = glt.data.dequantize_mxfp8(rows, x.shape[1]).to(torch.bfloat16)
    ut = glt.data.UnifiedTensor(0, rows.dtype)
    ut.append_shared_tensor(rows)
    keep.append(ut)
    tables[t] = ut._table()
  y = torch.randint(0, classes, (sizes['paper'],), generator=torch.Generator().manual_seed(5)).to(dev)
  kw = dict(fanouts=fan, batch_size=1024, hidden=hidden, num_classes=classes, edge_dir='in', seed=1, device=dev,
            use_cuda_graph=False, feature_format=args.feat_format)
  if args.model == 'rsage':
    eng = HeteroSageEngine(graphs, tables, y, feat_dim, sizes, 'paper', **kw)
  elif args.model == 'rgat':
    eng = HeteroGatEngine(graphs, tables, y, feat_dim, sizes, 'paper', heads=heads, **kw)
  else:
    eng = HeteroHgtEngine(graphs, tables, y, feat_dim, sizes, 'paper', heads=heads, **kw)
  n = {eng.tid[t]: sizes[t] for t in sizes}
  for r, et in enumerate(eng.edge_types):
    ei = edges[et].to(dev)
    order = torch.argsort(ei[1], stable=True)
    dst, src = ei[1][order], ei[0][order]
    deg = torch.bincount(dst, minlength=sizes[et[2]]).clamp(min=1).unsqueeze(1).float()
    csr[r] = (dst, src, deg)

  # per-layer device times of the engine, from events around its layer calls
  log = []

  def wrap(name, fn):
    def inner(*a):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      out = fn(*a)
      e1.record()
      log.append((name(*a), e0, e1))
      return out
    return inner
  eng._infer_input = wrap(lambda c: 'input', eng._infer_input)
  eng._infer_layer = wrap(lambda l, X, Z, c: f'layer{l}', eng._infer_layer)
  eng._infer_head = wrap(lambda X: 'head', eng._infer_head)

  def engine_call():
    log.clear()
    return eng.inference(args.chunk_rows)
  ms_eng, all_eng, out_eng = timed(engine_call, args.warmup, args.calls)
  layers = {k: round(a.elapsed_time(b), 3) for k, a, b in log}
  torch.cuda.empty_cache()
  ms_torch, all_torch, out_torch = timed(lambda: ARMS[args.model](eng, csr, fdev, n), args.warmup, args.calls)
  sample = torch.randperm(sizes['paper'], generator=torch.Generator().manual_seed(7))[:args.sample].to(dev)
  a, b = out_eng[sample].float(), out_torch[sample].float()
  result = {'metric': f'{args.model} full-neighbourhood inference of every seed-type node (device-timed ms per call, '
                      f'median of {args.calls})',
            'card': card(), 'model': args.model, 'feature_format': args.feat_format, 'nodes': sizes,
            'edges': {'/'.join(k): int(v.shape[1]) for k, v in edges.items()}, 'feat_dim': feat_dim, 'hidden': hidden,
            'heads': heads if args.model != 'rsage' else None, 'layers': len(fan), 'classes': classes,
            'chunk_rows': args.chunk_rows,
            'engine_ms': round(ms_eng, 3), 'engine_ms_all': [round(x, 3) for x in all_eng],
            'engine_layer_ms': layers,
            'torch_ms': round(ms_torch, 3), 'torch_ms_all': [round(x, 3) for x in all_torch],
            'speedup': round(ms_torch / ms_eng, 2),
            'agreement': {'nodes': int(sample.numel()), 'max_abs_diff': float((a - b).abs().max()),
                          'argmax_agreement': float((a.argmax(1) == b.argmax(1)).float().mean())}}
  print(json.dumps(result), flush=True)


if __name__ == '__main__':
  main()
