"""A small link-prediction task shared by the link engine and link trainer tests: a stochastic-block graph whose
features are the block centroid plus noise, with 5 % of its edges held out of the sampling graph."""
import torch

import graphlearn_for_pytorch_b200 as glt


def sbm_link_task(num_nodes=4096, blocks=16, deg_in=10, deg_out=2, dim=64, noise=3.0, holdout=0.05, seed=0):
  """-> dict(topo, train_ei [2, E] (both directions), train_pairs [2, E/2], held [2, H], neg [2, H], x [N, dim]).

  Undirected edges: `deg_in` per node inside its block and `deg_out` to uniform nodes, no self loops or duplicates.
  `held` edges are removed from the graph (both directions); `neg` are as many uniform random pairs."""
  g = torch.Generator().manual_seed(seed)
  block = torch.arange(num_nodes) % blocks
  e_in, e_out = num_nodes * deg_in // 2, num_nodes * deg_out // 2
  src = torch.randint(0, num_nodes, (e_in + e_out,), generator=g)
  dst = torch.cat([block[src[:e_in]] + blocks * torch.randint(0, num_nodes // blocks, (e_in,), generator=g),
                   torch.randint(0, num_nodes, (e_out,), generator=g)])
  keep = src != dst
  und = torch.unique(torch.stack([torch.minimum(src, dst), torch.maximum(src, dst)])[:, keep], dim=1)
  und = und[:, torch.randperm(und.shape[1], generator=g)]
  n_held = int(holdout * und.shape[1])
  held, train = und[:, :n_held], und[:, n_held:]
  train_ei = torch.cat([train, train.flip(0)], 1)
  centroids = torch.randn(blocks, dim, generator=g)
  x = centroids[block] + noise * torch.randn(num_nodes, dim, generator=g)
  neg = torch.randint(0, num_nodes, (2, n_held), generator=g)
  topo = glt.data.Topology(train_ei, layout='CSR', num_nodes=num_nodes)
  return dict(topo=topo, train_ei=train_ei, train_pairs=train, held=held, neg=neg, x=x, num_nodes=num_nodes)


def pair_batches(pairs, batch, steps, seed=1):
  """`steps` batches of `batch` training pairs, consecutive slices of reshuffled epochs."""
  g = torch.Generator().manual_seed(seed)
  out = []
  while len(out) < steps:
    p = pairs[:, torch.randperm(pairs.shape[1], generator=g)]
    out += [p[:, i:i + batch] for i in range(0, p.shape[1] - batch + 1, batch)]
  return out[:steps]
