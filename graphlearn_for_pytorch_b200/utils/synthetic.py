"""Synthetic graphs: RMAT generator with named dataset shapes, and the
self-describing "feature = id" fixtures used by the tests (idea from the
reference's test/python/dist_test_utils.py:41-140, re-implemented).
"""
from typing import Dict, Optional, Tuple

import torch

# nodes, directed edges, feature dim, classes (SURVEY.md Appendix D)
DATASET_SHAPES = {
  'products': dict(num_nodes=2_449_029, num_edges=123_718_280, feat_dim=100, num_classes=47),
  'papers100m': dict(num_nodes=111_059_956, num_edges=1_615_685_872, feat_dim=128, num_classes=172),
  'tiny': dict(num_nodes=10_000, num_edges=200_000, feat_dim=32, num_classes=8),
}


def rmat_edges(num_nodes: int, num_edges: int, a=0.57, b=0.19, c=0.19, seed: int = 0,
               device='cpu', chunk: int = 1 << 24) -> torch.Tensor:
  """R-MAT edge list [2, E] (Graph500 parameters by default), generated on `device`."""
  scale = max(1, (num_nodes - 1).bit_length())
  gen = torch.Generator(device=device)
  gen.manual_seed(seed)
  outs = []
  done = 0
  while done < num_edges:
    n = min(chunk, num_edges - done)
    src = torch.zeros(n, dtype=torch.int64, device=device)
    dst = torch.zeros(n, dtype=torch.int64, device=device)
    for _ in range(scale):
      r = torch.rand(n, device=device, generator=gen)
      src_bit = (r >= a + b).to(torch.int64)
      dst_bit = ((r >= a) & (r < a + b) | (r >= a + b + c)).to(torch.int64)
      src = (src << 1) | src_bit
      dst = (dst << 1) | dst_bit
    # fold ids beyond num_nodes back in and permute to kill the RMAT id locality
    src = src % num_nodes
    dst = dst % num_nodes
    outs.append(torch.stack([src, dst]))
    done += n
  ei = torch.cat(outs, dim=1)
  mult = 0x9E3779B1
  ei = (ei * mult + 12345) % num_nodes  # cheap bijection-ish scramble (keeps degree skew)
  return ei


def ring_graph(num_nodes: int = 40, hops=(1, 2)) -> torch.Tensor:
  """v -> v+1, v+2 (mod N): every node has exactly len(hops) out-neighbours."""
  src = torch.arange(num_nodes).repeat_interleave(len(hops))
  off = torch.tensor(list(hops)).repeat(num_nodes)
  return torch.stack([src, (src + off) % num_nodes])


def id_features(num_nodes: int, dim: int = 16, dtype=torch.float32) -> torch.Tensor:
  """Row v == [v] * dim, so any gathered row can be verified against its id."""
  return torch.arange(num_nodes, dtype=dtype).unsqueeze(1).repeat(1, dim)


def multilabel_targets(edge_index: torch.Tensor, x: torch.Tensor, num_tasks: int, seed: int = 0) -> torch.Tensor:
  """Learnable multi-label targets, bool [N, num_tasks]: task t of node v is positive when a random projection w_t of
  the mean feature row of v's neighbours (edge_index[1] of the edges out of v) is in its top r_t fraction, r_t uniform
  in [0.1, 0.5).  A node without neighbours averages to zero."""
  n = x.shape[0]
  g = torch.Generator().manual_seed(seed)
  src, dst = edge_index[0].long(), edge_index[1].long()
  xf = x.float()
  agg = torch.zeros_like(xf).index_add_(0, src, xf[dst])
  deg = torch.bincount(src, minlength=n).clamp(min=1).to(xf.dtype)
  proj = (agg / deg.unsqueeze(1)) @ torch.randn(x.shape[1], num_tasks, generator=g).to(x.device)
  rate = 0.1 + 0.4 * torch.rand(num_tasks, generator=g).to(x.device)
  k = ((1 - rate) * (n - 1)).long()
  thresh = proj.sort(0).values.gather(0, k.unsqueeze(0))
  return proj > thresh


def synthetic_dataset_tensors(name: str = 'tiny', seed: int = 0, device='cpu',
                              feat_dtype=torch.float32, pad_to: Optional[int] = None,
                              scale_edges: float = 1.0):
  """(edge_index, features, labels, shape-dict) of a named RMAT-shaped dataset."""
  shape = dict(DATASET_SHAPES[name])
  n, e = shape['num_nodes'], int(shape['num_edges'] * scale_edges)
  ei = rmat_edges(n, e, seed=seed, device=device)
  f = shape['feat_dim'] if pad_to is None else pad_to
  gen = torch.Generator(device=device)
  gen.manual_seed(seed + 1)
  feats = torch.randn(n, f, device=device, generator=gen, dtype=torch.float32).to(feat_dtype)
  if pad_to is not None and pad_to > shape['feat_dim']:
    feats[:, shape['feat_dim']:] = 0
  labels = torch.randint(0, shape['num_classes'], (n,), device=device, generator=gen)
  return ei, feats, labels, shape


def _rmat_chunks(num_nodes: int, num_edges: int, seed: int, device, a=0.57, b=0.19, c=0.19, chunk: int = 1 << 24):
  """Yields the [2, n] chunks of `rmat_edges(num_nodes, num_edges, seed=seed)` one at a time (identical RNG
  consumption, so concatenating the chunks reproduces `rmat_edges` bit for bit) without ever holding the
  whole edge list: papers100M-shape graphs (1.6 B edges) are generated shard by shard."""
  scale = max(1, (num_nodes - 1).bit_length())
  gen = torch.Generator(device=device)
  gen.manual_seed(seed)
  done = 0
  mult = 0x9E3779B1
  while done < num_edges:
    n = min(chunk, num_edges - done)
    src = torch.zeros(n, dtype=torch.int64, device=device)
    dst = torch.zeros(n, dtype=torch.int64, device=device)
    for _ in range(scale):
      r = torch.rand(n, device=device, generator=gen)
      src = (src << 1) | (r >= a + b).to(torch.int64)
      dst = (dst << 1) | ((r >= a) & (r < a + b) | (r >= a + b + c)).to(torch.int64)
    ei = torch.stack([src % num_nodes, dst % num_nodes])
    yield (ei * mult + 12345) % num_nodes
    done += n


def rmat_degrees(num_nodes: int, num_edges: int, seed: int = 0, device='cpu', undirected: bool = True) -> torch.Tensor:
  """Out-degree of every node of the (optionally symmetrised) RMAT graph, streamed chunk by chunk."""
  deg = torch.zeros(num_nodes, dtype=torch.int64, device=device)
  for ei in _rmat_chunks(num_nodes, num_edges, seed, device):
    deg += torch.bincount(ei[0], minlength=num_nodes)
    if undirected:
      deg += torch.bincount(ei[1], minlength=num_nodes)
  return deg


def rmat_csr_shard(num_nodes: int, num_edges: int, row_begin: int, row_end: int, seed: int = 0, device='cpu',
                   undirected: bool = True, old2new: Optional[torch.Tensor] = None,
                   idx_dtype=torch.int32) -> Dict[str, torch.Tensor]:
  """CSR rows [row_begin, row_end) of the RMAT graph (after the optional id relabelling `old2new`), built
  from streamed chunks: every rank of a partitioned run generates the same edge stream and keeps its own
  row range only.  `num_edges` counts generated (one-direction) edges; `undirected` adds the reverse of each.
  -> {'indptr' int64 [rows+1], 'indices' idx_dtype [nnz] column-sorted, 'row_begin', 'row_end'}."""
  keys = []
  n_rows = row_end - row_begin
  for ei in _rmat_chunks(num_nodes, num_edges, seed, device):
    if old2new is not None:
      ei = old2new[ei]
    for s, d in ((ei[0], ei[1]), (ei[1], ei[0])) if undirected else ((ei[0], ei[1]),):
      m = (s >= row_begin) & (s < row_end)
      keys.append((s[m] - row_begin) * num_nodes + d[m])        # (local row, col) packed: < 2^63 for N < 2^31
    del ei
  key = torch.cat(keys) if keys else torch.zeros(0, dtype=torch.int64, device=device)
  del keys
  key, _ = torch.sort(key)
  rows = torch.div(key, num_nodes, rounding_mode='floor')
  indices = (key - rows * num_nodes).to(idx_dtype)
  del key
  indptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=device)
  if rows.numel():
    torch.cumsum(torch.bincount(rows, minlength=n_rows), 0, out=indptr[1:])
  return {'indptr': indptr, 'indices': indices.contiguous(), 'eids': None, 'weights': None,
          'row_begin': int(row_begin), 'row_end': int(row_end)}


def synthetic_kg(num_nodes: int, num_relations: int, num_triples: int,
                 seed: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
  """A seeded knowledge graph with planted structure: (train, valid, test) int64 [3, m] (head, relation, tail).

  Entity e belongs to cluster e // 8 of C = num_nodes // 8 clusters in a chain; relation r links
  cluster c to cluster c + r + 1 (when it exists), so a triple's tail cluster is a translation of its head cluster.
  TransE, ComplEx and RotatE can represent this exactly; DistMult only up to its symmetry in head and tail.  Triples
  draw r, then a head cluster with a successor, then a uniform head and tail inside the two clusters; duplicates are
  dropped, and the distinct triples are split 80 / 10 / 10 in a seeded order.  Needs C >= num_relations + 1."""
  N, R, M, S = int(num_nodes), int(num_relations), int(num_triples), 8
  C = N // S
  if R < 1 or M < 1 or C < R + 1:
    raise ValueError(f'synthetic_kg needs num_relations, num_triples >= 1 and num_nodes // 8 >= '
                     f'num_relations + 1 (got N={N}, R={R}, triples={M})')
  g = torch.Generator().manual_seed(int(seed))
  r = torch.randint(0, R, (M,), generator=g)
  span = C - r - 1                                   # head clusters with a successor at distance r + 1
  c = (torch.rand(M, generator=g) * span).long().clamp_max(span - 1)
  h = c * S + torch.randint(0, S, (M,), generator=g)
  t = (c + r + 1) * S + torch.randint(0, S, (M,), generator=g)
  trip = torch.unique(torch.stack([h, r, t]), dim=1)
  trip = trip[:, torch.randperm(trip.size(1), generator=g)]
  m = trip.size(1)
  a, b = int(0.8 * m), int(0.9 * m)
  return trip[:, :a].contiguous(), trip[:, a:b].contiguous(), trip[:, b:].contiguous()
