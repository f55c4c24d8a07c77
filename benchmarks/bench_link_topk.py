#!/usr/bin/env python
"""Exact top-K link retrieval over every node at ogbn-products' shape: the link_topk kernel against chunked torch.

  python benchmarks/bench_link_topk.py [--nodes 2449029 --dim 256 --k 100 --queries 65536,1024 --rounds 3]

Embeddings are random bf16 rows [N, d]; the exclusion graph is the symmetric products-shape RMAT graph (bench.py's
generator, int32 column ids), so every query drops its training neighbours and itself.  Two workloads, one on each side
of the kernel's split choice: 65,536 queries (1,024 query tiles of 64 rows, one candidate split) and 1,024 queries
(16 query tiles, the candidates split so that every SM has a CTA).

* kernel: `models.link_topk` (csrc/cuda/link_topk.cu), the score matrix never leaves the SM;
* torch:  what a user writes today, per chunk of --chunk queries: `torch.mm(q, X.T, out_dtype=torch.float32)` on bf16,
          -inf scattered over the excluded ids and the query itself, then `torch.topk`.

Arms alternate for --rounds rounds after one warm-up call each, device-timed with CUDA events.  Per workload: ms per
call, achieved TFLOP/s (2 n N d / t), and the share of the floor: the larger of the compute floor (2 n N d at the
data-sheet 989 TFLOP/s dense bf16) and the HBM floor of the kernel's schedule (`kernel_hbm_bytes`, at 3.35 TB/s).
Agreement: per query, the id sets of the two arms must be equal except for ids whose kernel score is within fp32
rounding of the k-th score (ties the torch arm's different summation order may break the other way).  The card name
and power limit are read in the same run.  One JSON line is printed, and appended to --record when given.
"""
import argparse
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench_inference import card  # noqa: E402

PEAK_BF16 = 989e12
PEAK_HBM = 3.35e12


def kernel_hbm_bytes(n, N, d, k, E_q, idx_bytes, sms):
  """HBM traffic of the kernel's schedule.  The grid is (query tiles of 64) x (candidate splits) with splits =
  max(1, min(64, SMs // tiles)) and one CTA per SM at d = 256, k = 100 (its shared memory); the CTAs resident at once
  sweep their candidate tiles in the same ascending order, so L2 serves each candidate row to all of them and a wave
  reads the candidate table from HBM once.  Plus: the query rows gathered (read, written, read by TMA), the exclusion
  rows of the queries (E_q column ids and an indptr pair each), the split partial keys written and read, and the
  outputs."""
  tiles = math.ceil(n / 64)
  splits = max(1, min(64, sms // tiles))
  waves = math.ceil(tiles * splits / sms)
  return (waves * N * d * 2 + 3 * n * d * 2 + E_q * idx_bytes + n * 16 + 2 * splits * n * k * 8 + n * k * 12), splits


def torch_topk(emb, queries, k, indptr, indices, chunk):
  import torch
  n = queries.numel()
  ids = torch.empty(n, k, dtype=torch.int64, device=emb.device)
  scores = torch.empty(n, k, dtype=torch.float32, device=emb.device)
  for r0 in range(0, n, chunk):
    q = queries[r0:r0 + chunk]
    m = q.numel()
    s = torch.mm(emb[q], emb.T, out_dtype=torch.float32)
    deg = indptr[q + 1] - indptr[q]
    r = torch.repeat_interleave(torch.arange(m, device=emb.device), deg)
    pos = torch.repeat_interleave(indptr[q] - torch.cumsum(deg, 0) + deg, deg) + \
        torch.arange(r.numel(), device=emb.device)
    s[r, indices[pos].long()] = float('-inf')
    s[torch.arange(m, device=emb.device), q] = float('-inf')
    top = torch.topk(s, k, dim=1)
    scores[r0:r0 + m], ids[r0:r0 + m] = top.values, top.indices
    del s
  return ids, scores


def agreement(ids_k, sc_k, ids_t, sc_t, d):
  """(mismatched ids, mismatches not explained by rounding at the k-th score) over all queries"""
  import torch
  n, k = ids_k.shape
  span = int(max(ids_k.max(), ids_t.max())) + 1
  rows = torch.arange(n, device=ids_k.device).unsqueeze(1) * span
  key_k, key_t = (rows + ids_k).flatten(), (rows + ids_t).flatten()
  only_k = ~torch.isin(key_k, key_t)
  only_t = ~torch.isin(key_t, key_k)
  kth = sc_k[:, -1:].expand(n, k).flatten()
  tol = 1e-5 * sc_k.abs().max() * d / 64 + 1e-6
  bad = (only_k & ((sc_k.flatten() - kth).abs() > tol)).sum() + (only_t & ((sc_t.flatten() - kth).abs() > tol)).sum()
  return int(only_k.sum()), int(bad)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--nodes', type=int, default=2_449_029)
  p.add_argument('--edges', type=int, default=123_718_280, help='directed edges (both directions of each RMAT edge)')
  p.add_argument('--dim', type=int, default=256)
  p.add_argument('--k', type=int, default=100)
  p.add_argument('--queries', default='65536,1024')
  p.add_argument('--chunk', type=int, default=1024, help='torch arm: queries per score block')
  p.add_argument('--rounds', type=int, default=3)
  p.add_argument('--seed', type=int, default=0)
  p.add_argument('--record', default=None, help='append the JSON line to this file')
  a = p.parse_args()
  import torch
  import graphlearn_for_pytorch_b200 as glt
  from graphlearn_for_pytorch_b200.models import link_topk
  from graphlearn_for_pytorch_b200.utils.synthetic import rmat_csr_shard
  assert torch.cuda.is_available(), 'bench_link_topk measures on a GPU'
  assert a.rounds >= 2
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(dev)
  N, d, k = a.nodes, a.dim, a.k
  shard = rmat_csr_shard(N, a.edges // 2, 0, N, seed=a.seed, device=dev, undirected=True)
  graph = glt.data.Graph.from_shards([shard], 0)
  indptr, indices = shard['indptr'], shard['indices']
  g = torch.Generator(device=dev).manual_seed(a.seed + 1)
  emb = torch.randn(N, d, device=dev, generator=g).to(torch.bfloat16)
  sms = torch.cuda.get_device_properties(dev).multi_processor_count

  workloads = []
  for n in (int(x) for x in a.queries.split(',')):
    queries = torch.randint(0, N, (n,), device=dev, generator=g)
    arms = {'kernel': lambda: link_topk(emb, queries, k, exclude=graph),
            'torch': lambda: torch_topk(emb, queries, k, indptr, indices, a.chunk)}

    def timed(name):
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      e0.record()
      out = arms[name]()
      e1.record()
      torch.cuda.synchronize()
      return out, e0.elapsed_time(e1)

    outs, ms = {}, {name: [] for name in arms}
    for name in arms:                    # warm-up: module loads, cuBLAS heuristics, allocator
      timed(name)
    for _ in range(a.rounds):
      for name in arms:
        outs[name], t = timed(name)
        ms[name].append(t)
    mismatched, unexplained = agreement(*outs['kernel'], *outs['torch'], d)
    E_q = int((indptr[queries + 1] - indptr[queries]).sum())
    flops = 2.0 * n * N * d
    hbm, splits = kernel_hbm_bytes(n, N, d, k, E_q, indices.element_size(), sms)
    floor_s = max(flops / PEAK_BF16, hbm / PEAK_HBM)
    w = {'queries': n, 'splits': splits, 'flops': flops, 'kernel_hbm_bytes_model': hbm,
         'kernel_l2_to_sm_bytes_model': math.ceil(n / 64) * N * d * 2,
         'floor_ms': floor_s * 1e3, 'floor_bound': 'compute' if flops / PEAK_BF16 >= hbm / PEAK_HBM else 'HBM',
         'ids_only_in_kernel': mismatched, 'mismatches_beyond_rounding': unexplained}
    for name in arms:
      med = statistics.median(ms[name])
      w[name] = {'ms_median': med, 'ms_all': ms[name], 'TFLOP_per_s': flops / (med * 1e-3) / 1e12,
                 'share_of_floor': floor_s / (med * 1e-3)}
    w['speedup_vs_torch'] = w['torch']['ms_median'] / w['kernel']['ms_median']
    workloads.append(w)
    del outs

  rec = {
    'metric': 'exact top-K link retrieval over all nodes, ms per call, median (first workload)',
    'value': workloads[0]['kernel']['ms_median'], 'unit': 'ms', 'rounds': a.rounds,
    'workloads': workloads,
    'torch_arm': f'per {a.chunk} queries: torch.mm(bf16, out_dtype=fp32), -inf scatter over excluded ids, torch.topk',
    'shape': {'nodes': N, 'dim': d, 'k': k, 'exclusion_edges': int(indices.numel()),
              'column_id_bytes': indices.element_size()},
    'peaks': {'bf16_dense_flops': PEAK_BF16, 'hbm_bytes_per_s': PEAK_HBM, 'source': 'H100 SXM data sheet'},
    'card': card(),
  }
  line = json.dumps(rec)
  print(line, flush=True)
  if a.record:
    os.makedirs(os.path.dirname(os.path.abspath(a.record)), exist_ok=True)
    with open(a.record, 'a') as f:
      f.write(line + '\n')
  bad = [w['queries'] for w in workloads if w['mismatches_beyond_rounding'] > 0]
  if bad:
    sys.exit(f'the arms disagree beyond rounding at {bad} queries')


if __name__ == '__main__':
  main()
