"""GraphSageLinkEngine: in-graph negatives (k_link_seeds), the fused edge loss (k_link_bce + cast), one full step
against an fp32 recomputation, CUDA-graph replay, checkpoints and learning a block graph."""
import pytest
import torch
import torch.nn.functional as F

import graphlearn_for_pytorch_b200 as glt
from graphlearn_for_pytorch_b200.models import GraphSageLinkEngine, GraphSageLinkTrainer, link_auc
from helpers import rmat_csr
from link_task import pair_batches, sbm_link_task

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def _device_graph(topo):
  g = glt.data.Graph(topo, 'CUDA', 0)
  g.lazy_init()
  return g


def _link_seeds(native, g, pos, N, k, seed=7, step=0):
  B = pos.shape[1]
  seeds = torch.empty(2 * (1 + k) * B, dtype=torch.int64, device=DEV)
  n = torch.zeros(1, dtype=torch.int32, device=DEV)
  native.link_seeds(g.graph_handler, pos.contiguous(), N, k, seed, torch.tensor([step], dtype=torch.int32, device=DEV),
                    seeds, n)
  return seeds, int(n.item())


def _edge_keys(topo, N):
  rows = torch.repeat_interleave(torch.arange(N), topo.indptr[1:] - topo.indptr[:-1])
  return (rows * N + topo.indices.long()).to(DEV)


# --------------------------------------------------------------------------- 1. negatives
def test_negatives_layout_range_strictness_and_keying(native):
  N, k = 20000, 3
  ei, topo = rmat_csr(N, 200000, seed=3)
  g = _device_graph(topo)
  torch.manual_seed(0)
  B, n = 320, 300
  pos = torch.full((2, B), -1, dtype=torch.int64)
  pos[:, :n] = ei[:, torch.randperm(ei.shape[1])[:n]]
  pos = pos.to(DEV)
  P = (1 + k) * B
  seeds, n_pairs = _link_seeds(native, g, pos, N, k)
  src, dst = seeds[:P], seeds[P:]
  assert n_pairs == (1 + k) * n
  assert torch.equal(src[:B], pos[0]) and torch.equal(dst[:B], pos[1])          # positives verbatim
  neg_src, neg_dst = src[B:].view(B, k), dst[B:].view(B, k)
  assert bool((neg_src[n:] == -1).all()) and bool((neg_dst[n:] == -1).all())   # padding propagates
  ns, nd = neg_src[:n].flatten(), neg_dst[:n].flatten()
  assert bool(((ns >= 0) & (ns < N) & (nd >= 0) & (nd < N)).all())
  assert not bool(torch.isin(ns * N + nd, _edge_keys(topo, N)).any())           # strict on a sparse graph
  again, _ = _link_seeds(native, g, pos, N, k)
  nxt, _ = _link_seeds(native, g, pos, N, k, step=1)
  other_seed, _ = _link_seeds(native, g, pos, N, k, seed=8)
  assert torch.equal(again, seeds)                                               # same (seed, step): same draws
  assert not torch.equal(nxt[B:P], seeds[B:P]) and not torch.equal(other_seed[B:P], seeds[B:P])
  assert torch.equal(nxt[:B], seeds[:B])


def test_negatives_on_a_near_complete_graph_keep_the_last_draw(native):
  N = 16
  r, c = torch.meshgrid(torch.arange(N), torch.arange(N), indexing='ij')
  keep = (r != c) | (r < 2)                       # every pair except 14 self loops is an edge
  topo = glt.data.Topology(torch.stack([r[keep], c[keep]]), layout='CSR', num_nodes=N)
  g = _device_graph(topo)
  pos = torch.stack([torch.arange(64) % N, (torch.arange(64) + 1) % N]).to(DEV)
  seeds, n_pairs = _link_seeds(native, g, pos, N, 4)
  P = 5 * 64
  s, d = seeds[64:P], seeds[P + 64:]
  assert n_pairs == P
  assert bool(((s >= 0) & (s < N) & (d >= 0) & (d < N)).all())
  hit = torch.isin(s * N + d, _edge_keys(topo, N))
  assert int(hit.sum()) > 0 and int((~hit).sum()) > 0     # padded draws (edges) and accepted non-edges both occur


def test_negative_node_frequencies_are_uniform(native):
  N = 1000
  ei, topo = rmat_csr(N, 3000, seed=5)
  g = _device_graph(topo)
  B, k = 100000, 10
  pos = ei[:, torch.randint(0, ei.shape[1], (B,))].to(DEV)
  seeds, _ = _link_seeds(native, g, pos, N, k, seed=11)
  P = (1 + k) * B
  for ids in (seeds[B:P], seeds[P + B:]):
    cnt = torch.bincount(ids, minlength=N).float()
    expect = B * k / N                                   # 1000 per node, sd ~ 32
    assert cnt.numel() == N and float((cnt - expect).abs().max()) < 0.2 * expect


# --------------------------------------------------------------------------- 2. loss kernel + cast
@pytest.mark.parametrize('C', [64, 96, 256, 512, 320])
def test_link_bce_and_cast_match_autograd(native, C):
  torch.manual_seed(C)
  n_pad = (C + 63) // 64 * 64
  R, cap, B, k = 200, 256, 60, 2
  P = (1 + k) * B
  Z = torch.zeros(cap, n_pad, device=DEV)
  Z[:, :C] = torch.randn(cap, C, device=DEV) / C ** 0.5 * 2
  Z = Z.to(torch.bfloat16)
  sl = torch.randint(0, R, (2 * P,), device=DEV, dtype=torch.int32)      # duplicate endpoints
  sl[P + 3:P + 10] = sl[3:10]                                              # self-pairs (positives)
  sl[P + B + 5:P + B + 9] = sl[B + 5:B + 9]                                # self-pairs (negatives)
  sl[B - 4:B] = -1                                                          # padded positives ...
  sl[P + B + 20] = -1                                                       # ... and a padded negative
  valid = (sl[:P] >= 0) & (sl[P:] >= 0)
  n_pairs = torch.tensor([int(valid.sum())], dtype=torch.int32, device=DEV)
  counters = torch.zeros(16, dtype=torch.int32, device=DEV)
  counters[1] = R
  loss = torch.zeros(1, device=DEV)
  correct = torch.zeros(1, dtype=torch.int32, device=DEV)
  dZ = torch.zeros(cap, n_pad, device=DEV)
  native.link_bce(Z, C, sl, P, B, n_pairs, loss, correct, dZ)
  dPre = torch.full((cap, n_pad), 7.0, device=DEV).to(torch.bfloat16)
  gb = torch.zeros(n_pad, device=DEV)
  native.relu_bwd_cast(dZ, Z, counters, 1, dPre, gb, True, 1.0, relu=False)
  torch.cuda.synchronize()
  Zf = Z.float().requires_grad_(True)
  ls, lt = sl[:P].long()[valid], sl[P:].long()[valid]
  y = (torch.arange(P, device=DEV) < B).float()[valid]
  s = (Zf[ls, :C] * Zf[lt, :C]).sum(-1)
  ref = F.binary_cross_entropy_with_logits(s, y)
  ref.backward()
  assert abs(loss.item() - ref.item()) < 1e-4 * max(1.0, ref.item())
  assert int(correct.item()) == int(((s > 0).float() == y).sum())
  g_ref = Zf.grad
  assert torch.allclose(dZ[:, :C], g_ref[:, :C], rtol=1e-4, atol=1e-6)
  assert torch.allclose(dPre[:R].float(), g_ref[:R], rtol=1e-2, atol=1e-5)
  assert bool((dPre[R:] == 0).all())                                       # zero rows up to capacity
  assert bool((dPre[:, C:] == 0).all()) and bool((dZ[:, C:] == 0).all()) and bool((gb[C:] == 0).all())
  assert torch.allclose(gb, dPre[:R].float().sum(0), rtol=1e-4, atol=1e-6)
  assert torch.allclose(gb, g_ref.sum(0), rtol=2e-2, atol=1e-4)


# --------------------------------------------------------------------------- 3. one full step
def _engine(task=None, N=6000, E=120000, Fdim=64, fan=(5, 4, 3), bs=128, out=64, k=1, graph=False, **kw):
  if task is None:
    ei, topo = rmat_csr(N, E, seed=3)
    torch.manual_seed(0)
    feats = torch.randn(N, Fdim, device=DEV).to(torch.bfloat16)
  else:
    topo, N = task['topo'], task['num_nodes']
    feats = task['x'].to(DEV, torch.bfloat16)
    Fdim = feats.shape[1]
  g = _device_graph(topo)
  ut = glt.data.UnifiedTensor(0, torch.bfloat16)
  ut.append_shared_tensor(feats)
  eng = GraphSageLinkEngine(g, ut._table(), Fdim, N, fanouts=list(fan), batch_size=bs, hidden=kw.pop('hidden', 128),
                            out_channels=out, neg_ratio=k, device=DEV, use_cuda_graph=graph, seed=5, **kw)
  eng._keep = (ut, feats, topo)
  return eng, feats, topo


def _dense_link_reference(eng, feats):
  """fp32 recomputation of the engine's link step from the sampled structure (cf. test_gpu_engine._dense_reference)."""
  ar = eng.arena
  L = eng.L
  cum = ar.counters.cpu().tolist()[:L + 2]
  nodes = ar.nodes[:cum[L + 1]]
  params = [(eng.W(l).float().clone().requires_grad_(True), eng.b(l).float().clone().requires_grad_(True))
            for l in range(1, L + 1)]
  H = feats[nodes].float()
  for l in range(1, L + 1):
    nh = L - l + 1
    T = cum[nh]
    mean = torch.zeros(T, H.shape[1], device=DEV)
    for h in range(nh):
      k = eng.fanouts[h]
      rows = cum[h + 1] - cum[h]
      if rows == 0:
        continue
      ell = ar.ell[h][:rows * k].view(rows, k).long()
      valid = (ell >= 0).unsqueeze(-1)
      dg = ar.deg[cum[h]:cum[h + 1]].float().clamp(min=1).unsqueeze(1)
      mean[cum[h]:cum[h + 1]] = (H[ell.clamp(min=0)] * valid).sum(1) / dg
    A = torch.cat([mean, H[:T]], dim=1).to(torch.bfloat16).float()
    W, b = params[l - 1]
    Z = A @ W.t() + b
    if l < L:
      Z = F.relu(Z)
      if eng.dropout > 0.0:
        keep = (eng.Z[l][:T] != 0).float()
        Z = Z * keep / (1.0 - eng.dropout)
    H = Z + (Z.to(torch.bfloat16).float() - Z).detach()      # bf16 storage, straight-through gradient
  P, B = eng.P, eng.pos_bs
  sl = ar.seed_local[:2 * P].long()
  valid = (sl[:P] >= 0) & (sl[P:] >= 0)
  s = (H[sl[:P][valid], :eng.C] * H[sl[P:][valid], :eng.C]).sum(-1)
  y = (torch.arange(P, device=DEV) < B).float()[valid]
  loss = F.binary_cross_entropy_with_logits(s, y)
  loss.backward()
  return loss.item(), params


@pytest.mark.parametrize('cfg', [dict(use_fused=False), dict(use_fused=True), dict(use_fused=True, dropout=0.5)],
                         ids=['unfused', 'fused', 'fused-dropout'])
def test_full_step_matches_fp32_recomputation(native, cfg):
  eng, feats, topo = _engine(k=2, **cfg)
  assert eng.fused_ok[1] == cfg['use_fused']
  ei = torch.stack([torch.repeat_interleave(torch.arange(6000), topo.indptr[1:] - topo.indptr[:-1]),
                    topo.indices.long()])
  pairs = ei[:, torch.randperm(ei.shape[1])[:100]].to(DEV)          # a partial batch (100 of 128)
  eng._stage_seeds(eng._seeds[0], pairs)
  eng._sample(); eng._forward(); eng._backward()
  torch.cuda.synchronize()
  assert int(eng._n_pairs[0].item()) == 300
  ref_loss, params = _dense_link_reference(eng, feats)
  assert abs(float(eng.loss.item()) - ref_loss) < 2e-2 * max(1.0, abs(ref_loss))
  for l in range(1, eng.L + 1):
    off, n, k = eng._w_off[l - 1]
    gW = eng.g32[off:off + n * k].view(n, k)
    W, b = params[l - 1]
    err = (gW - W.grad).abs().max().item() / W.grad.abs().max().clamp(min=1e-6).item()
    assert err < 5e-2, (l, err)
    boff, _ = eng._b_off[l - 1]
    gb = eng.g32[boff:boff + n]
    assert (gb - b.grad).abs().max().item() / b.grad.abs().max().clamp(min=1e-6).item() < 5e-2, l
  boff, n = eng._b_off[eng.L - 1]
  assert bool((eng.g32[boff + eng.C:boff + n] == 0).all())          # padding columns of the last layer


# --------------------------------------------------------------------------- 4. CUDA graph, pipelining
def test_graph_replay_draws_fresh_negatives_and_matches_eager(native):
  eng, feats, topo = _engine(graph=True, bs=256, fan=(4, 3), out=96)
  eng.warmup_and_capture(n_eager=1)
  assert eng.library_gemms_per_step == 0 and eng.kernels_per_step > 0
  pairs = torch.randint(0, 6000, (2, 256), device=DEV)
  saved = eng.state_dict()
  eng._stage_seeds(eng._seeds[0], pairs)
  eng._step_eager()
  eager_loss = float(eng.loss.item())
  eager_seeds = eng.seeds_dev.clone()
  eng.load_state_dict(saved)
  replay_loss = float(eng.train_step(pairs).item())
  assert torch.equal(eng.seeds_dev, eager_seeds)
  assert abs(replay_loss - eager_loss) < 1e-3, (replay_loss, eager_loss)
  first = eng.seeds_dev.clone()
  eng.train_step(pairs)
  P = eng.P
  assert torch.equal(eng.seeds_dev[:256], first[:256])
  assert not torch.equal(eng.seeds_dev[256:P], first[256:P])


def test_pipelined_engine_matches_sequential_semantics(native):
  """sample(b+1) || train(b): the loss lags one call, flush trains the tail, and the engine still learns."""
  task = sbm_link_task()
  for use_graph in (False, True):
    eng, _, _ = _engine(task, fan=(10, 5), bs=256, graph=use_graph, pipeline=True, hidden=64, lr=3e-3)
    eng.warmup_and_capture(n_eager=1)
    batches = pair_batches(task['train_pairs'], 256, 81)
    assert eng.train_step(batches[0]) is None                  # priming call
    losses = [float(eng.train_step(b).item()) for b in batches[1:]]
    tail = eng.flush()
    assert tail is not None and eng.flush() is None
    assert sum(losses[-10:]) / 10 < 0.6 * sum(losses[:5]) / 5, (losses[:5], losses[-10:])
    assert eng.overflow_count() == 0
    loss, correct, n = eng.evaluate_batch(task['train_pairs'][:, :256])
    assert n == 512 and correct / n > 0.6


# --------------------------------------------------------------------------- 5. checkpoint
def test_checkpoint_reproduces_the_next_negatives(native):
  eng, _, _ = _engine(graph=True)
  eng.warmup_and_capture(n_eager=1)
  batches = [torch.randint(0, 6000, (2, 128), device=DEV) for _ in range(4)]
  for b in batches[:3]:
    eng.train_step(b)
  state = eng.state_dict()
  eng.train_step(batches[3])
  seeds, loss = eng.seeds_dev.clone(), float(eng.loss.item())
  other, _, _ = _engine(graph=True)
  other.warmup_and_capture(n_eager=1)
  other.load_state_dict(state)
  other.train_step(batches[3])
  assert torch.equal(other.seeds_dev, seeds)
  assert abs(float(other.loss.item()) - loss) < 1e-3
  eng.load_state_dict(state)
  eng.train_step(batches[3])
  assert torch.equal(eng.seeds_dev, seeds)


# --------------------------------------------------------------------------- 6. learning
def test_engine_learns_the_block_graph_like_the_trainer(native):
  task = sbm_link_task()
  batches = pair_batches(task['train_pairs'], 256, 300)
  eng, _, _ = _engine(task, fan=(10, 5), bs=256, graph=True, hidden=64, lr=3e-3)
  eng.warmup_and_capture(n_eager=1)
  for b in batches:
    eng.train_step(b)
  emb = eng.inference()
  assert emb.shape == (task['num_nodes'], 64) and emb.dtype == torch.bfloat16
  auc = link_auc(emb.cpu(), task['held'], task['neg'])
  tr = GraphSageLinkTrainer(glt.data.Graph(task['topo'], 'CPU'), task['x'], 64, fanouts=[10, 5], hidden=64,
                            out_channels=64, lr=3e-3, seed=5)
  for b in batches:
    tr.train_step(b)
  auc_ref = link_auc(tr.inference(), task['held'], task['neg'])
  assert auc >= 0.85 and abs(auc - auc_ref) <= 0.05, (auc, auc_ref)
