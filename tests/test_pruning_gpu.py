"""Gradual magnitude pruning on the GPU (rigl_mask_prune_run, pruning.Pruning, TrainHarness(pruning=...)) against
the NumPy restatement in tests/pruning_oracle.py: masks and thresholds bit for bit."""
import json
import os

import numpy as np
import pytest
import torch

import pruning_oracle as oracle
from rigl_b200 import _cabi, checkpoint, pruning, workloads
from rigl_b200.masks import MaskUpdateEngine, MaskVariable

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FLAGS = _cabi.LAYER_DROP_ONLY | _cabi.LAYER_ALL_ACTIVE
HERE = os.path.dirname(os.path.abspath(__file__))


def _shapes(tag):
  with open(os.path.join(HERE, 'golden', 'sparse_utils_golden.json')) as f:
    return [tuple(sh) for _, sh in [c for c in json.load(f)['cases'] if c['tag'] == tag][0]['layers']]


def _prune(weights_np, sparsities, old_thr, decay):
  """One rigl_mask_prune_run over the layers; returns (masks bool, thresholds float32)."""
  eng = MaskUpdateEngine()
  specs, keep = [], []
  for i, (w, s) in enumerate(zip(weights_np, sparsities)):
    w = np.ascontiguousarray(w, np.float32).reshape(-1)
    mv = MaskVariable('layer%d' % i, (w.size,), DEV)
    t = torch.from_numpy(w).to(DEV)
    specs.append(dict(mask=mv, weights=t, score_grow=t, flags=FLAGS))
    keep.append(pruning.keep_count(w.size, s))
  thr = torch.tensor(np.asarray(old_thr, np.float32), device=DEV)
  eng.prune(specs, keep, thr, decay)
  torch.cuda.synchronize()
  return [sp['mask'].numpy().astype(bool) for sp in specs], thr.cpu().numpy()


def _check(weights_np, sparsities, old_thr=None, decay=0.0):
  old_thr = np.zeros(len(weights_np), np.float32) if old_thr is None else np.asarray(old_thr, np.float32)
  masks, thr = _prune(weights_np, sparsities, old_thr, decay)
  for i, (w, s) in enumerate(zip(weights_np, sparsities)):
    want_mask, want_thr = oracle.prune_layer(w, s, old_thr[i], decay)
    assert thr[i].tobytes() == np.float32(want_thr).tobytes(), (i, thr[i], want_thr)
    assert np.array_equal(masks[i], want_mask), (i, int(masks[i].sum()), int(want_mask.sum()))
  return masks, thr


@pytest.mark.parametrize('s', [0.0, 0.5, 0.9, 0.99])
def test_resnet50_all_layers_one_plan(s):
  rng = np.random.RandomState(int(s * 100))
  shapes = _shapes('r50_erk80')
  assert len(shapes) == 54
  ws = [(rng.standard_normal(sh) * 0.05).astype(np.float32) for sh in shapes]
  _check(ws, [np.float32(s)] * len(ws))


def test_tie_groups_at_the_threshold():
  rng = np.random.RandomState(1)
  n = 200000
  vals = np.array([0.5, -0.5, 0.25, -0.25, 0.0, -0.0, 1.0, -1.0], np.float32)
  repeated = rng.choice(vals, n)
  pairs = rng.standard_normal(n // 2).astype(np.float32)
  pm = np.concatenate([pairs, -pairs])[rng.permutation(n)]
  zeros = np.where(rng.rand(n) < 0.7, np.float32(0), rng.standard_normal(n).astype(np.float32))
  zeros[rng.rand(n) < 0.3] = -0.0
  neg_zero = np.full(n, -0.0, np.float32)
  neg_zero[:10] = 1.0
  for s in (0.3, 0.5, 0.9):
    _check([repeated, pm, zeros, neg_zero], [np.float32(s)] * 4)


@pytest.mark.parametrize('n', [1, 31, 129])
def test_small_layers_and_extreme_k(n):
  rng = np.random.RandomState(n)
  w = rng.standard_normal(n).astype(np.float32)
  for s in (0.0, 0.5, 0.9, 0.99, 1.0):          # k = n ... k = 1 (clamped)
    _check([w, w[::-1].copy(), np.abs(w)], [np.float32(s)] * 3)
  assert pruning.keep_count(n, np.float32(0.0)) == n and pruning.keep_count(n, np.float32(1.0)) == 1


def test_threshold_decay_with_old_threshold():
  rng = np.random.RandomState(2)
  ws = [rng.standard_normal(sh).astype(np.float32) * 0.1 for sh in ((3, 3, 64, 64), (1000,), (129,))]
  _check(ws, [np.float32(0.5), np.float32(0.8), np.float32(0.3)], old_thr=[0.07, 0.5, 0.0], decay=0.5)
  _check(ws, [np.float32(0.9)] * 3, old_thr=[0.2, 0.01, 3.0], decay=0.25)


def test_zero_map_entry_keeps_every_weight():
  torch.manual_seed(0)
  reg = pruning.MaskedLayerRegistry()
  model = workloads.MnistFC(device=DEV, registry=reg)
  hp = pruning.get_pruning_hparams().parse('begin_pruning_step=0,sparsity_function_begin_step=0,'
                                           'end_pruning_step=10,sparsity_function_end_step=10,target_sparsity=0.9')
  hp.set_hparam('weight_sparsity_map', ['layer2:0.81', 'layer3:0.0'])
  from rigl_b200.sparse_optimizers_base import GlobalStep
  p = pruning.Pruning(hp, global_step=GlobalStep(10), registry=reg)
  weights = [l.weight.detach().cpu().numpy().reshape(-1).copy() for l in reg.layers()]
  p.mask_update_op()
  masks = [m.numpy().reshape(-1).astype(bool) for m in reg.get_masks()]
  thr = p.thresholds.cpu().numpy()
  sps = p.layer_sparsities()
  assert sps[0] == np.float32(0.9) and sps[2] == 0
  for i, (w, s) in enumerate(zip(weights, sps)):
    want_mask, want_thr = oracle.prune_layer(w, oracle.layer_sparsity(np.float32(0.9), 'layer%d/weights' % (i + 1),
                                                                      hp.weight_sparsity_map, 0.9), 0.0, 0.0)
    assert thr[i].tobytes() == want_thr.tobytes() and np.array_equal(masks[i], want_mask)
  assert masks[2].all()
  assert [float(t) for t in reg.get_thresholds()] == [float(t) for t in thr]


def test_launch_count_constant_and_weights_untouched():
  rng = np.random.RandomState(3)
  counts = []
  for shapes in (_shapes('r50_erk80')[:3], _shapes('r50_erk80')):
    ws = [rng.standard_normal(sh).astype(np.float32).reshape(-1) for sh in shapes]
    eng = MaskUpdateEngine()
    specs = []
    for i, w in enumerate(ws):
      t = torch.from_numpy(w).to(DEV)
      specs.append(dict(mask=MaskVariable('l%d' % i, (w.size,), DEV), weights=t, score_grow=t, flags=FLAGS))
    thr = torch.zeros(len(ws), device=DEV)
    keep = [pruning.keep_count(w.size, np.float32(0.8)) for w in ws]
    eng.prune(specs, keep, thr, 0.0)            # builds the plan
    torch.cuda.synchronize()
    before = _cabi.launch_count()
    eng.prune(specs, keep, thr, 0.0)
    counts.append(_cabi.launch_count() - before)
    torch.cuda.synchronize()
    for w, sp in zip(ws, specs):
      assert sp['weights'].cpu().numpy().tobytes() == w.tobytes()
  assert counts[0] == counts[1]


def test_weights_and_slots_untouched_in_a_harness():
  torch.manual_seed(1)
  model = workloads.MnistFC(device=DEV)
  from rigl_b200.sparse_optimizers_base import GlobalStep
  p = pruning.Pruning(pruning.get_pruning_hparams(), global_step=GlobalStep(0), registry=model.registry)
  h = workloads.TrainHarness(model, lr=0.1, weight_decay=1e-4, label_smoothing=0.0, optimizer_cls=None, pruning=p)
  x = torch.randn(64, 784, device=DEV)
  y = x[:, :10].argmax(1).long()
  for _ in range(3):
    h.step(x, y)
  snap = lambda: [t.detach().cpu().numpy().tobytes() for t in model.parameters()] + \
      [t.cpu().numpy().tobytes() for q in model.parameters() for t in h.inner.state[q].values() if torch.is_tensor(t)]
  before = snap()
  h.global_step.value = 50
  p.mask_update_op()
  torch.cuda.synchronize()
  assert snap() == before
  assert [m.count_ones() for m in model.registry.get_masks()] == \
      [pruning.keep_count(m.size, p.sparsity(50)) for m in model.registry.get_masks()]


# ---- training under TrainHarness(optimizer_cls=None, pruning=...)
BEGIN, END, FREQ, TARGET, STEPS = 2, 12, 2, 0.9, 14


def _spec():
  return pruning.get_pruning_hparams().parse(
      'begin_pruning_step={0},sparsity_function_begin_step={0},end_pruning_step={1},sparsity_function_end_step={1},'
      'target_sparsity={2},pruning_frequency={3},threshold_decay=0'.format(BEGIN, END, TARGET, FREQ))


def _build(kind, seed, inner='momentum', fused=None, droprate=0.3):
  torch.manual_seed(seed)
  if kind == 'mnist':
    model = workloads.MnistFC(device=DEV)
  else:
    model = workloads.WideResNet(depth=22, width=2, droprate=droprate, device=DEV)
  p = pruning.Pruning(_spec(), registry=model.registry)
  h = workloads.TrainHarness(model, lr=0.05, weight_decay=1e-4, label_smoothing=0.0, optimizer_cls=None, pruning=p,
                             inner_optimizer=inner, fused_optimizer=fused)
  return model, h, p


def _batches(kind):
  gen = torch.Generator(device=DEV)
  gen.manual_seed(11)
  out = []
  for _ in range(STEPS):
    if kind == 'mnist':
      x = torch.randn(128, 784, device=DEV, generator=gen)
      out.append((x, x[:, :10].argmax(1).long()))
    else:
      x = torch.randn(128, 3, 32, 32, device=DEV, generator=gen).bfloat16().contiguous(memory_format=torch.channels_last)
      out.append((x, torch.randint(0, 10, (128,), device=DEV, generator=gen)))
  return out


def _state(model, h, p):
  return [t.detach().cpu().numpy() for t in model.parameters()] + \
      [m.numpy() for m in model.registry.get_masks()] + [p.thresholds.cpu().numpy()]


@pytest.mark.parametrize('kind,inner,fused', [('mnist', 'momentum', True), ('mnist', 'momentum', False),
                                              ('mnist', 'adam', True), ('wrn', 'momentum', True)])
def test_training_teacher_forced(kind, inner, fused):
  model, h, p = _build(kind, 5, inner, fused)
  layers = model.registry.layers()
  updates = []
  for step, (x, y) in enumerate(_batches(kind)):
    old_thr = p.thresholds.cpu().numpy()
    old_masks = [m.numpy() for m in model.registry.get_masks()]
    loss = h.step(x, y)
    assert np.isfinite(float(loss.detach()))
    gs = h.global_step.value
    assert gs == step + 1
    masks = [m.numpy().reshape(-1).astype(bool) for m in model.registry.get_masks()]
    thr = p.thresholds.cpu().numpy()
    if p.last_update_step == gs and gs > 0:
      updates.append(gs)
      s = oracle.sparsity(gs, 0.0, TARGET, BEGIN, END, 3)
      for i, l in enumerate(layers):
        w = l.weight.detach().cpu().numpy()
        want_mask, want_thr = oracle.prune_layer(w, s, old_thr[i], 0.0)
        assert thr[i].tobytes() == want_thr.tobytes(), (gs, l.scope)
        assert np.array_equal(masks[i], want_mask), (gs, l.scope)
    else:
      assert thr.tobytes() == old_thr.tobytes()
      assert all(np.array_equal(a.reshape(-1).astype(bool), b) for a, b in zip(old_masks, masks))
  assert updates == oracle.update_steps(range(1, STEPS + 1), BEGIN, END, FREQ) == [2, 4, 6, 8, 10, 12]
  s = p.sparsity(STEPS)
  assert s == np.float32(TARGET)
  ones = [m.count_ones() for m in model.registry.get_masks()]
  sizes = [m.size for m in model.registry.get_masks()]
  assert ones == [pruning.keep_count(n, s) for n in sizes]
  global_sparsity = 1.0 - sum(ones) / float(sum(sizes))
  assert abs(global_sparsity - float(s)) <= len(sizes) / float(sum(sizes))
  zero_fracs = model.registry.get_weight_sparsity()
  assert all(abs(z - (1 - o / float(n))) < 1e-6 for z, o, n in zip(zero_fracs, ones, sizes))


@pytest.fixture
def deterministic_cudnn():
  """WRN's dense first conv runs on cuDNN; its deterministic mode makes that conv reproducible to the bit."""
  old = torch.backends.cudnn.deterministic
  torch.backends.cudnn.deterministic = True
  yield
  torch.backends.cudnn.deterministic = old


def _build_reproducible(kind, seed):
  # dropout off: graph warm-up / capture and a resumed process draw the dropout masks from different generator
  # states, which would change the trajectory rather than test the pruning
  return _build(kind, seed, droprate=0.0)


def _assert_same(la, lb, sa, sb):
  assert np.asarray(la, np.float64).tobytes() == np.asarray(lb, np.float64).tobytes()
  assert len(sa) == len(sb) and all(a.tobytes() == b.tobytes() for a, b in zip(sa, sb))


@pytest.mark.parametrize('kind', ['mnist', 'wrn'])
def test_graphed_equals_eager(kind, deterministic_cudnn):
  """Loss, weights, masks and thresholds of the CUDA-graph harness equal the eager harness bit for bit."""
  batches = _batches(kind)

  def run(graph):
    model, h, p = _build_reproducible(kind, 6)
    if graph:
      assert h.enable_cuda_graph(*batches[0])
    losses = [float(h.step(x, y).detach()) for x, y in batches]
    return losses, _state(model, h, p), h.global_step.value, p.last_update_step
  le, se, ge, ue = run(False)
  lg, sg, gg, ug = run(True)
  assert (ge, ue) == (gg, ug) == (STEPS, END)
  _assert_same(le, lg, se, sg)


@pytest.mark.parametrize('kind', ['mnist', 'wrn'])
def test_checkpoint_resume_is_bit_identical(kind, tmp_path, deterministic_cudnn):
  """Save at step 7, restore into a freshly built model and harness: steps 8-14 equal the uninterrupted run."""
  batches = _batches(kind)
  model, h, p = _build_reproducible(kind, 7)
  losses = []
  for i, (x, y) in enumerate(batches):
    losses.append(float(h.step(x, y).detach()))
    if i + 1 == 7:
      variables = checkpoint.variables_of(model, h.inner, pruning=p)
      assert 'model_pruning/last_mask_update_step' in variables
      assert all(l.scope + '/threshold' in variables for l in model.registry.layers())
      path = checkpoint.save(str(tmp_path / 'run'), variables, h.global_step.value)
      saved = _state(model, h, p)
  want = _state(model, h, p)

  model2, h2, p2 = _build_reproducible(kind, 8)
  h2.global_step.value = checkpoint.restore(path, checkpoint.variables_of(model2, h2.inner, pruning=p2,
                                                                          ckpt_path=path))
  assert h2.global_step.value == 7 and p2.last_update_step == 6
  restored = _state(model2, h2, p2)
  assert len(restored) == len(saved) and all(a.tobytes() == b.tobytes() for a, b in zip(restored, saved))
  assert np.count_nonzero(p2.thresholds.cpu().numpy()) == len(model2.registry.layers())
  losses2 = [float(h2.step(x, y).detach()) for x, y in batches[7:]]
  assert (h2.global_step.value, p2.last_update_step) == (h.global_step.value, p.last_update_step) == (STEPS, END)
  _assert_same(losses2, losses[7:], _state(model2, h2, p2), want)


def test_prune_run_does_not_wait_for_the_device():
  """rigl_mask_prune_run only enqueues: behind a ~1 s device sleep, the call returns long before the sleep ends."""
  import time
  rng = np.random.RandomState(4)
  eng = MaskUpdateEngine()
  specs = []
  for i, sh in enumerate(_shapes('r50_erk80')):
    w = torch.from_numpy(rng.standard_normal(sh).astype(np.float32).reshape(-1)).to(DEV)
    specs.append(dict(mask=MaskVariable('l%d' % i, (w.numel(),), DEV), weights=w, score_grow=w, flags=FLAGS))
  keep = [pruning.keep_count(sp['mask'].size, np.float32(0.8)) for sp in specs]
  thr = torch.zeros(len(specs), device=DEV)
  eng.prune(specs, keep, thr, 0.0)              # builds the plan and the workspace
  torch.cuda.synchronize()
  torch.cuda._sleep(2 * 10 ** 9)                # ~1 s of device time at H100 clocks
  t0 = time.perf_counter()
  eng.prune(specs, keep, thr, 0.5)
  dt = time.perf_counter() - t0
  torch.cuda.synchronize()
  assert dt < 0.25, dt


def test_variables_of_without_pruning_is_unchanged():
  model, h, p = _build('mnist', 9)
  plain = checkpoint.variables_of(model, h.inner)
  assert not any(k.endswith('threshold') or 'last_mask_update_step' in k for k in plain)
