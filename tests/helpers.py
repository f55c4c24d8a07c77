"""Shared fixtures: tiny self-describing graphs (feature row v == [v]*dim)."""
import torch

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.utils.synthetic import id_features, ring_graph, rmat_edges


def ring_dataset(num_nodes=40, dim=16, graph_mode='CPU', edge_dir='out', with_gpu=False, device=None,
                 split_ratio=0.0, weights=False):
  ei = ring_graph(num_nodes)
  ds = glt.data.Dataset(edge_dir=edge_dir)
  w = (torch.arange(ei.shape[1], dtype=torch.float32) % 3 + 1.0) if weights else None
  ds.init_graph(ei, edge_weights=w, graph_mode=graph_mode, device=device, num_nodes=num_nodes)
  ds.init_node_features(id_features(num_nodes, dim), with_gpu=with_gpu, split_ratio=split_ratio, device=device)
  ds.init_edge_features(id_features(ei.shape[1], 4), with_gpu=with_gpu, device=device)
  ds.init_node_labels(torch.arange(num_nodes))
  return ds


def rmat_csr(num_nodes=2000, num_edges=40000, seed=0):
  ei = rmat_edges(num_nodes, num_edges, seed=seed)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=num_nodes)
  return ei, topo


def adjacency_sets(topo):
  ptr, ind = topo.indptr.tolist(), topo.indices.tolist()
  return [set(ind[ptr[i]:ptr[i + 1]]) for i in range(len(ptr) - 1)]


def canonical_edges(out):
  """Set of (global src, global dst) pairs of a SamplerOutput."""
  node = out.node.cpu()
  return set(zip(node[out.row.cpu()].tolist(), node[out.col.cpu()].tolist()))


# --------------------------------------------------------------------------- error bounds of GPU kernels
def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
  """Spacing of bf16 numbers at |x| (float64): 2^(e - 7) for |x| in [2^e, 2^(e+1)); the smallest normal spacing at 0."""
  x = x.double().abs()
  _, e = torch.frexp(x)                     # x = m * 2^e, m in [0.5, 1)
  return torch.where(x > 0, torch.ldexp(torch.ones_like(x), e - 8), torch.full_like(x, 2.0 ** -133))


def gemm_bound(ref: torch.Tensor, absprod: torch.Tensor, k: int, bf16_out: bool = True) -> torch.Tensor:
  """Largest error of a bf16 GEMM with fp32 accumulation over a contraction of length k: k * 2^-22 * (|A| . |W|^T)
  (fp32 summation with margin for truncating adders), plus one bf16 ulp of the result for a bf16 output.  `ref` and
  `absprod` are float64; for a split-K fp32 output (`bf16_out=False`) only the summation term applies."""
  b = float(k) * 2.0 ** -22 * absprod.double()
  return b + bf16_ulp(ref) if bf16_out else b


EPS32 = 2.0 ** -23


def sum_bound(n, abs_sum: torch.Tensor) -> torch.Tensor:
  """Largest error of an fp32 sum of n terms (in any order, each term rounded once): (n + 1) * 2^-23 * sum|terms|."""
  n = n.double() if torch.is_tensor(n) else float(n)
  return (n + 1) * EPS32 * abs_sum.double()


def mean_ref(X: torch.Tensor, tgt: torch.Tensor, src: torch.Tensor, deg: torch.Tensor):
  """float64 mean aggregation sum_{edges t <- s} X[s] / deg[t] over the T = deg.numel() targets, and its error bound:
  one bf16 ulp of the mean, plus the fp32 sum of deg rows and the multiplication by the fp32 1/deg; rows of degree 0
  must be exactly 0."""
  Xd = X.double()
  T, d = deg.numel(), X.shape[1]
  s = torch.zeros(T, d, dtype=torch.float64, device=X.device).index_add_(0, tgt, Xd[src])
  a = torch.zeros(T, d, dtype=torch.float64, device=X.device).index_add_(0, tgt, Xd[src].abs())
  dg = deg.to(X.device).double().unsqueeze(1)
  ref = s / dg.clamp(min=1)
  bound = torch.where(dg > 0, bf16_ulp(ref) + (dg + 2) * EPS32 * a / dg.clamp(min=1), torch.zeros_like(ref))
  return ref, bound


def gather_ref(dA, d, Z, tgt, src, deg, T, S, cap_src, gscale):
  """float64 dPre of sage_gather_bwd (dPre[s] = relu'(Z[s]) * gscale * (dA[s, d:] if s < T + sum_{t <- s} dA[t, :d] /
  deg[t])) and its error bound, from the exact bf16 operands and the edges (tgt, src) of the layer's hops; the bound is
  0 (exact) on masked elements and on rows in [S, cap_src)."""
  dev = dA.device
  keep = (tgt < T) & (src < S)
  tgt, src = tgt[keep], src[keep]
  inv = (1.0 / deg.float()).double()                   # fp32 1/deg, as the kernel computes it
  dAd = dA.double()
  terms = dAd[tgt, :d] * inv[tgt].unsqueeze(1)
  ref = torch.zeros(cap_src, d, dtype=torch.float64, device=dev)
  ab = torch.zeros_like(ref)
  m = min(T, S)
  ref[:m] = dAd[:m, d:]
  ab[:m] = dAd[:m, d:].abs()
  ref.index_add_(0, src, terms)
  ab.index_add_(0, src, terms.abs())
  n = torch.bincount(src, minlength=cap_src).double()
  n[:m] += 1
  g = float(torch.tensor(gscale, dtype=torch.float32))
  live = (torch.arange(cap_src, device=dev) < S).unsqueeze(1)
  mask = live & (Z[:cap_src] > 0) if Z is not None else live.expand(cap_src, d)
  ref = torch.where(mask, ref * g, torch.zeros_like(ref))
  bound = torch.where(mask, bf16_ulp(ref) + g * sum_bound((n + 2).unsqueeze(1), ab),torch.zeros_like(ref))
  return ref, bound


def colsum_ratio(colsum: torch.Tensor, X: torch.Tensor, S: int, init: float = 0.0) -> float:
  """Error / bound of fp32 column sums (bias gradients) of the first S rows of X accumulated onto `init`."""
  x = X[:S].double()
  return bound_ratio(colsum, x.sum(0) + init, sum_bound(S, x.abs().sum(0) + abs(init)))


def bound_ratio(got: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
  """max |got - ref| / bound over all elements (<= 1 when every element lies within its bound; 0-bound elements
  must match exactly)."""
  err = (got.double() - ref.double()).abs()
  if err.numel() == 0:
    return 0.0
  exact = bound <= 0
  if bool((err[exact] > 0).any()):
    return float('inf')
  return float((err[~exact] / bound[~exact]).max()) if bool((~exact).any()) else 0.0
