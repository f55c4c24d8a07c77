"""GraphSageMultiLabelEngine and its loss kernel on the GPU.

* `sigmoid_bce` on hand-built batches against float64, at every task count T whose bias-gradient sum runs in
  registers (ld <= 256) or in the second column-sum pass, at seed counts around the warp and block sizes, with node ids
  outside the label table and logits of +-80 and exactly 0.  Negative controls show that the bounds reject a gradient
  without the 1 / T, a label bit read one column off and a tail row left unzeroed.
* Every stage of real engine steps against float64, through the stage checks of test_gpu_step_stages with the
  softmax-loss check replaced by the BCE check below (eager, captured, pipelined, fused and unfused, dropout).
* The captured step has the launches of a GraphSageEngine with T classes; the engine learns what
  GraphSageMultiLabelTrainer learns; checkpoints round-trip; binding errors raise.
"""
import pytest
import torch

import graphlearn_for_pytorch_b200 as glt
import test_gpu_step_stages as stages
from graphlearn_for_pytorch_b200.models import (GraphSageEngine, GraphSageMultiLabelEngine,
                                               GraphSageMultiLabelTrainer, multilabel_auc, multilabel_f1,
                                               pack_label_bits)
from graphlearn_for_pytorch_b200.utils.synthetic import multilabel_targets
from helpers import (EPS32, SIG_ERR, Ratios, _batches, _snapshot, _table, bf16_ulp, bound_ratio, colsum_ratio,
                     rmat_csr, sum_bound)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)


def bce_ref(z, y, n0, T, per_row_terms):
  """float64 loss and dlogits of k_sigmoid_bce from the bf16 logits z [n0, T] and 0/1 labels y, with the kernel's fp32
  scale inv = 1 / (n0 T), and their bounds.  dlogits: one bf16 ulp (at least bf16's subnormal spacing 2^-133: a logit of
  -80 with label 0 has a gradient near 1e-40), sigmoid within SIG_ERR relative, the subtraction and the scaling one u
  each.  Loss: each term max(z, 0) - y z + log1p(exp(-|z|)) within 4 u of its parts' magnitude,
  then fp32 sums along the kernel's longest chain: per_row_terms per lane and row, five warp levels, n0 row atomics."""
  inv = float(torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(n0 * T), dtype=torch.float32)) if n0 else 0.
  s = torch.sigmoid(z)
  ref = (s - y) * inv
  bound = bf16_ulp(ref) + 2.0 ** -133 + (SIG_ERR * s + 2 * EPS32 * (s - y).abs()) * inv
  sp = torch.log1p(torch.exp(-z.abs()))
  terms = z.clamp(min=0) - y * z + sp
  mag = (z.clamp(min=0) + (y * z).abs() + sp) * inv
  loss = float(terms.sum()) * inv
  lbound = float(sum_bound(per_row_terms + 5 + n0 + 2, mag.sum())) + 4 * EPS32 * float(mag.sum())
  return loss, ref, bound, lbound


# --------------------------------------------------------------------------- the kernel on hand-built batches
N_TABLE, CAP = 700, 320


def _batch(T, ld, seed):
  g = torch.Generator().manual_seed(seed)
  y = torch.rand(N_TABLE, T, generator=g) < 0.3
  logits = (torch.randn(CAP, ld, generator=g) * 3)
  logits[0, :T] = torch.where(torch.arange(T) % 2 == 0, 80.0, -80.0)
  logits[1, :T] = 0.0
  logits[2, :T] = torch.where(torch.arange(T) % 3 == 0, -80.0, 80.0)
  nodes = torch.randint(0, N_TABLE, (CAP,), generator=g)
  nodes[3], nodes[4], nodes[5], nodes[6] = -1, N_TABLE, N_TABLE + 1000, 1 << 40    # outside the table: all-zero labels
  return y.to(DEV), logits.to(DEV, torch.bfloat16), nodes.to(DEV)


def _labels_of(y, nodes, n0):
  ids = nodes[:n0]
  ok = (ids >= 0) & (ids < y.shape[0])
  Y = torch.zeros(n0, y.shape[1], dtype=torch.float64, device=DEV)
  Y[ok] = y[ids[ok]].double()
  return Y


KERNEL_T = [1, 31, 32, 33, 112, 121, 256, 257, 1000]


@pytest.mark.parametrize('T', KERNEL_T)
def test_sigmoid_bce_matches_fp64(native, T):
  for ld in sorted({(T + 63) // 64 * 64, (T + 7) // 8 * 8}):
    y, logits, nodes = _batch(T, ld, seed=T + ld)
    bits = pack_label_bits(y)
    for n0 in (0, 1, 127, 128, 129, CAP):
      for prezeroed in (False, True):
        ctr = torch.tensor([0, n0, n0 + 5, 0], dtype=torch.int32, device=DEV)
        dl = torch.full((CAP, ld), 7.0, dtype=torch.bfloat16, device=DEV)          # stale values everywhere
        loss0, colsum0 = (0.25, 0.5) if prezeroed else (0.0, 0.0)
        loss = torch.full((1,), 99.0 if not prezeroed else loss0, device=DEV)
        counts = torch.tensor([1, 2, 3] if prezeroed else [9, 9, 9], dtype=torch.int32, device=DEV)
        colsum = torch.full((ld,), 99.0 if not prezeroed else colsum0, device=DEV)
        native.sigmoid_bce(logits, T, bits, nodes, ctr, loss, dl, counts, colsum, prezeroed)
        torch.cuda.synchronize()
        tag = f'T {T} ld {ld} n0 {n0} prezeroed {prezeroed}'
        assert bool((dl[n0:] == 0).all()), f'{tag}: rows past n0 must be zero'
        assert bool((dl[:n0, T:] == 0).all()), f'{tag}: columns past T must be zero'
        if n0 == 0:
          assert float(loss) == loss0 and bool((colsum == colsum0).all()), tag
          assert counts.tolist() == ([1, 2, 3] if prezeroed else [0, 0, 0]), tag
          continue
        z = logits[:n0, :T].double()
        Y = _labels_of(y, nodes, n0)
        ref_loss, ref, bound, lbound = bce_ref(z, Y, n0, T, (ld + 31) // 32)
        r = bound_ratio(dl[:n0, :T], ref, bound)
        assert r <= 1.0, f'{tag}: dlogits error / bound = {r}'
        assert abs(float(loss) - loss0 - ref_loss) <= lbound + 4 * EPS32 * loss0, (tag, float(loss), ref_loss)
        pred = z > 0
        yb = Y > 0
        exp = [int((pred & yb).sum()), int((pred & ~yb).sum()), int((~pred & yb).sum())]
        base = [1, 2, 3] if prezeroed else [0, 0, 0]
        assert counts.tolist() == [a + b for a, b in zip(exp, base)], tag
        r = colsum_ratio(colsum, dl.float(), n0, init=colsum0)
        assert r <= 1.0, f'{tag}: bias gradient error / bound = {r}'
        if T == 112 and n0 == 129 and not prezeroed:
          # negative controls: the same bounds reject a gradient without 1 / T, labels read one column off, and an
          # unzeroed tail row
          no_T = (ref * T).to(torch.bfloat16)
          assert bound_ratio(no_T, ref, bound) > 1.0, 'the dlogits bound must reject a gradient without 1 / T'
          _, ref_off, bound_off, _ = bce_ref(z, torch.roll(Y, 1, dims=1), n0, T, 4)
          assert bound_ratio(dl[:n0, :T], ref_off, bound_off) > 1.0, 'the check must reject labels read one column off'
          bad = dl.clone()
          bad[n0] = 7.0
          assert not bool((bad[n0:] == 0).all()), 'the tail check must reject an unzeroed row'


def test_sigmoid_bce_without_optional_outputs(native):
  T, ld = 112, 128
  y, logits, nodes = _batch(T, ld, seed=1)
  bits = pack_label_bits(y)
  ctr = torch.tensor([0, 200, 250], dtype=torch.int32, device=DEV)
  loss = torch.zeros(1, device=DEV)
  dl = torch.full((CAP, ld), 3.0, dtype=torch.bfloat16, device=DEV)
  native.sigmoid_bce(logits, T, bits, nodes, ctr, loss, dl)
  ref_loss, ref, bound, lbound = bce_ref(logits[:200, :T].double(), _labels_of(y, nodes, 200), 200, T, 4)
  assert bound_ratio(dl[:200, :T], ref, bound) <= 1.0 and abs(float(loss) - ref_loss) <= lbound
  assert bool((dl[200:] == 0).all()) and bool((dl[:, T:] == 0).all())


# --------------------------------------------------------------------------- binding errors
def test_sigmoid_bce_bad_arguments_raise(native):
  from test_gpu_binding_checks import bad_tensor, pinned, probe
  T, ld = 40, 64
  y, logits, nodes = _batch(T, ld, seed=2)
  bits = pack_label_bits(y)
  ctr = torch.tensor([0, 100, 150], dtype=torch.int32, device=DEV)
  loss = torch.zeros(1, device=DEV)
  dl = torch.zeros(CAP, ld, dtype=torch.bfloat16, device=DEV)
  counts = torch.zeros(3, dtype=torch.int32, device=DEV)
  colsum = torch.zeros(ld, device=DEV)
  args = [logits, T, bits, nodes, ctr, loss, dl, counts, colsum, False]
  probe(native.sigmoid_bce, args, {
      0: bad_tensor(logits, logits[:, :56]),
      1: [0, ld + 1],
      2: [pinned(bits), bits.view(torch.int32), bits[:, :1],
          torch.zeros(N_TABLE, 3, dtype=torch.int32, device=DEV).view(torch.uint32)],
      3: [pinned(nodes), nodes.double(), nodes[:CAP - 1]],
      4: [pinned(ctr), ctr.to(torch.int64), ctr[:1]],
      5: [pinned(loss), loss.double(), torch.zeros(0, device=DEV)],
      6: bad_tensor(dl, dl[:CAP - 1]),
      7: [pinned(counts), counts.to(torch.int64), counts[:2]],
      8: [pinned(colsum), colsum.double(), colsum[:ld - 8]]})


# --------------------------------------------------------------------------- every stage of real steps
def _check_bce(R, Z, T, Y, nodes, n0, dPre, bias_grad, loss, correct):
  """Replaces test_gpu_step_stages._check_softmax for the multi-label engine: `labels` is the dense [N, T] 0/1 table."""
  z = Z[:n0, :T].double()
  ref_loss, ref, bound, lbound = bce_ref(z, Y[nodes[:n0]].double(), n0, T, (Z.shape[1] + 31) // 32)
  R.check('loss', abs(float(loss) - ref_loss) / lbound)
  R.check('dlogits', bound_ratio(dPre[:n0, :T], ref, bound))
  R.exact('dlogits pad', bool((dPre[:n0, T:] == 0).all()))
  R.check('db_last', colsum_ratio(bias_grad, dPre, n0))


ML_CASES = {
    'eager-wd': dict(T=112, weight_decay=5e-4),
    'captured-fused-dropout-wd': dict(T=112, graph=True, dropout=0.5, weight_decay=5e-4, controls=True),
    'pipelined-captured-unfused-dropout': dict(T=112, graph=True, pipeline=True, use_fused=False, dropout=0.3),
    'eager-unfused-T300': dict(T=300, use_fused=False, fanouts=[5, 4], bs=128),
}


@pytest.mark.parametrize('name', list(ML_CASES))
def test_multilabel_step_stages_match_fp64(native, monkeypatch, name):
  monkeypatch.setattr(stages, '_check_softmax', _check_bce)
  cfg = dict(ML_CASES[name])
  T, bs, fanouts = cfg.pop('T'), cfg.pop('bs', 256), cfg.pop('fanouts', [5, 4, 3])
  captured, controls = cfg.pop('graph', False), cfg.pop('controls', False)
  N, in_dim = 12000, 128
  topo, graph = stages._sage_graph(N, 120000, seed=len(name))
  g = torch.Generator().manual_seed(7)
  X = torch.randn(N, in_dim, generator=g).to(DEV).to(torch.bfloat16)
  Y = (torch.rand(N, T, generator=g) < 0.3).to(DEV)
  ut = _table(X)
  eng = GraphSageMultiLabelEngine(graph, ut._table(), Y, in_dim=in_dim, num_nodes=N, fanouts=fanouts, batch_size=bs,
                                  hidden=256, device=DEV, use_cuda_graph=captured, seed=3, **cfg)
  assert eng.C == T
  if captured:
    eng.warmup_and_capture(n_eager=1)
  dpre = lambda: [None] + [eng.dPre[l].clone() for l in range(1, eng.L + 1)]
  batches = _batches(bs, N, g)
  run = lambda i, snap, parity: _run_checks(eng, name, i, snap, parity, X, Y, controls)
  if eng.pipeline:
    eng.train_step(batches[0])
    for i in range(1, len(batches) + 1):
      snap = _snapshot(eng, dpre)
      eng.train_step(batches[i]) if i < len(batches) else eng.flush()
      run(i - 1, snap, 1 - eng._cur if i < len(batches) else eng._cur)
  else:
    for i, seeds in enumerate(batches):
      snap = _snapshot(eng, dpre)
      eng.train_step(seeds)
      run(i, snap, 0)


def _run_checks(eng, name, i, snap, parity, X, Y, controls):
  R = Ratios(f'multilabel {name} step {i}')
  stages._sage_stages(R, eng, snap, parity, X, X, Y, controls and i == 1)
  assert 'dlogits' in R.r and 'loss' in R.r, 'the BCE check must have run'
  R.show()


# --------------------------------------------------------------------------- launches, learning, checkpoints
def _engines(T, pipeline, N=6000, Fdim=128, **extra):
  _, topo = rmat_csr(N, 120000, seed=3)
  g = glt.data.Graph(topo, 'CUDA', 0)
  gen = torch.Generator(device=DEV).manual_seed(0)
  feats = torch.randn(N, Fdim, device=DEV, generator=gen).to(torch.bfloat16)
  ut = _table(feats)
  opts = dict(in_dim=Fdim, num_nodes=N, fanouts=[5, 4, 3], batch_size=256, hidden=128, device=DEV, pipeline=pipeline,
              dropout=0.2, **extra)
  base = GraphSageEngine(g, ut._table(), torch.randint(0, T, (N,), device=DEV, generator=gen), num_classes=T, **opts)
  ml = GraphSageMultiLabelEngine(g, ut._table(), torch.rand(N, T, device=DEV, generator=gen) < 0.3, **opts)
  return base, ml, (ut, topo)


@pytest.mark.parametrize('T', [112, 300])
@pytest.mark.parametrize('pipeline', [False, True])
def test_launch_count_matches_the_node_engine(native, T, pipeline):
  base, ml, keep = _engines(T, pipeline)
  base.warmup_and_capture()
  ml.warmup_and_capture()
  assert ml.kernels_per_step == base.kernels_per_step > 0, (ml.kernels_per_step, base.kernels_per_step)


def _task(N=20000, Fdim=64, T=24):
  ei, _ = rmat_csr(N, 200000, seed=3)
  ei = torch.cat([ei, ei.flip(0)], 1)
  topo = glt.data.Topology(ei, layout='CSR', num_nodes=N)
  x = torch.randn(N, Fdim, generator=torch.Generator().manual_seed(0))
  y = multilabel_targets(ei, x, T, seed=1)
  perm = torch.randperm(N, generator=torch.Generator().manual_seed(9))
  return topo, x, y, perm[:N // 2], perm[N // 2:]


def test_engine_learns_what_the_trainer_learns(native):
  topo, x, y, train, held = _task()
  N, Fdim, T = x.shape[0], x.shape[1], y.shape[1]
  g = glt.data.Graph(topo, 'CUDA', 0)
  ut = _table(x.to(DEV, torch.bfloat16))
  eng = GraphSageMultiLabelEngine(g, ut._table(), y.to(DEV), in_dim=Fdim, num_nodes=N, fanouts=[10, 5],
                                  batch_size=256, hidden=128, lr=1e-2, seed=5, device=DEV)
  eng.warmup_and_capture(n_eager=1)
  tr = GraphSageMultiLabelTrainer(g, x.to(DEV), y.to(DEV), in_dim=Fdim, fanouts=[10, 5], hidden=128, lr=1e-2, seed=5,
                                  device=DEV)
  yh = y[held]

  def scores(logits):
    lg = logits.float().cpu()[held]
    return multilabel_auc(lg, yh), multilabel_f1(lg, yh)

  auc0, f10 = scores(eng.inference())
  gen = torch.Generator().manual_seed(11)
  for _ in range(300):
    seeds = train[torch.randperm(train.numel(), generator=gen)[:256]].to(DEV)
    eng.train_step(seeds)
    tr.train_step(seeds)
  (auc_e, f1_e), (auc_t, f1_t) = scores(eng.inference()), scores(tr.inference())
  print(f'untrained AUC {auc0:.4f} F1 {f10:.4f}; engine AUC {auc_e:.4f} F1 {f1_e:.4f}; '
        f'trainer AUC {auc_t:.4f} F1 {f1_t:.4f}')
  assert auc_e > auc0 + 0.2 and f1_e > f10 + 0.2, (auc0, auc_e, f10, f1_e)
  assert abs(auc_e - auc_t) <= 0.02 and abs(f1_e - f1_t) <= 0.02, (auc_e, auc_t, f1_e, f1_t)
  loss, tp, fp, fn, n = eng.evaluate_batch(held[:256].to(DEV))
  assert n == 256 and tp + fn == int(yh[:256].sum()) and loss > 0


def test_state_dict_round_trips(native):
  # deterministic sampling fixes the row order inside a hop, which the dropout mask is keyed by
  _, ml, keep = _engines(112, False, deterministic_sampling=True)
  batches = [torch.randperm(6000, device=DEV)[:256] for _ in range(4)]
  for b in batches[:3]:
    ml.train_step(b)
  state = ml.state_dict()
  ml.train_step(batches[3])
  L = ml.L
  # the restored sampling position draws the same batch (the node buffer past the batch keeps each engine's stale ids)
  batch_nodes = lambda e: (e.arena.counters[:L + 2].tolist(), e.arena.nodes[:int(e.arena.counters[L + 1])].clone())
  (ctr, nodes), loss = batch_nodes(ml), float(ml.loss.item())
  _, other, keep_other = _engines(112, False, deterministic_sampling=True)
  other.warmup_and_capture(n_eager=1)
  other.load_state_dict(state)
  assert torch.equal(other.p32, state['p32'])
  other.train_step(batches[3])
  ctr2, nodes2 = batch_nodes(other)
  assert ctr2 == ctr and torch.equal(nodes2, nodes)
  assert abs(float(other.loss.item()) - loss) < 1e-3 * max(1.0, loss), (float(other.loss.item()), loss)
