"""optim.FusedAdam on the H100: the batched kernel against the numpy restatement of tf.train.AdamOptimizer bit for
bit, CUDA-graph replay, RigL mask updates resetting both moments, the train harness and checkpoints."""
import ctypes as C

import numpy as np
import pytest
import torch

import adam_oracle as ao
from oracle import rigl_oracle as orc
from rigl_b200 import _cabi, checkpoint, pruning, sparse_optimizers, workloads
from rigl_b200.layers import SparseLinear
from rigl_b200.masks import MaskVariable
from rigl_b200.optim import FusedAdam
from rigl_b200.sparse_optimizers_base import GlobalStep

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32 = np.float32


def _np(t):
  return t.detach().cpu().numpy().copy()


def _same(a, b):
  """Bit-equal, except that any NaN equals any NaN (the device and numpy write different NaN payloads)."""
  nan = np.isnan(a)
  return np.array_equal(nan, np.isnan(b)) and a[~nan].tobytes() == b[~nan].tobytes()


def test_kernel_matches_oracle_bit_for_bit():
  """Every size class of the chunked task table (one element, scalar tails, chunk edges, a ResNet-50 3x3x512x512
  layer), masked and dense, a pointer one float off 16-byte alignment (the scalar path), grad_scale != 1,
  weight decay, non-zero initial moments, five steps with an lr change: weights, m, v and both powers exact."""
  rng = np.random.RandomState(0)
  lib = _cabi.lib()
  b1, b2, eps = 0.9, 0.999, 1e-8
  params = []
  for n in (1, 3, 5, 31, 33, 8191, 8193, 2359296):
    for masked, offset in ((False, 0), (True, 0), (True, 1)):
      if offset and n > 8193:
        continue
      base = [torch.empty(n + offset, device=DEV) for _ in range(4)]
      w, m, v, g = (b[offset:] for b in base)
      w.copy_(torch.from_numpy(rng.standard_normal(n).astype(F32)))
      m.copy_(torch.from_numpy((0.1 * rng.standard_normal(n)).astype(F32)))
      v.copy_(torch.from_numpy((1e-3 * rng.rand(n)).astype(F32)))
      mask = None
      if masked:
        on = (rng.rand(n) < 0.3).astype(F32)
        mask = MaskVariable('p%d_%d' % (n, offset), (n,), DEV).assign(on)
      params.append(dict(w=w, m=m, v=v, g=g, mask=mask, on=None if mask is None else on.astype(bool),
                         wd=float(F32(1e-2 * (1 + len(params) % 3))), scale=0.25 if masked else 0.5, base=base))
  descs = (_cabi.AdamDesc * len(params))()
  for d, p in zip(descs, params):
    d.param, d.m, d.v, d.grad = p['w'].data_ptr(), p['m'].data_ptr(), p['v'].data_ptr(), p['g'].data_ptr()
    d.mask_bits = None if p['mask'] is None else p['mask'].bits.data_ptr()
    d.n, d.weight_decay, d.grad_scale = p['w'].numel(), p['wd'], p['scale']
  plan = C.c_void_p(None)
  _cabi.check(lib.rigl_adam_plan_create(descs, len(params), C.byref(plan)), 'rigl_adam_plan_create')
  lr_dev = torch.zeros(1, device=DEV)
  powers = torch.tensor([b1, b2], dtype=torch.float32, device=DEV)
  want = [dict(w=_np(p['w']), m=_np(p['m']), v=_np(p['v'])) for p in params]
  p1, p2 = F32(b1), F32(b2)
  try:
    for step in range(5):
      lr = 1e-3 if step < 3 else 2.5e-4
      lr_dev.fill_(lr)
      for p, s in zip(params, want):
        g = rng.standard_normal(p['w'].numel()).astype(F32)
        p['g'].copy_(torch.from_numpy(g))
        ge = ao.optimizer_grad(s['w'], g, p['on'], p['scale'], p['wd'])
        s['w'], s['m'], s['v'] = ao.adam_step(s['w'], s['m'], s['v'], ge, F32(lr), b1, b2, eps, p1, p2)
      _cabi.check(lib.rigl_adam_plan_run(plan, lr_dev.data_ptr(), powers.data_ptr(), b1, b2, eps,
                                         _cabi.stream_ptr()), 'rigl_adam_plan_run')
      p1, p2 = ao.advance_powers(p1, p2, b1, b2)
      for i, (p, s) in enumerate(zip(params, want)):
        for k in ('w', 'm', 'v'):
          assert _np(p[k]).tobytes() == s[k].tobytes(), (step, i, p['w'].numel(), k)
      assert _np(powers).tobytes() == np.array([p1, p2], F32).tobytes(), step
  finally:
    lib.rigl_adam_plan_destroy(plan)


def _two_layers(seed):
  pruning.reset_default_registry()
  torch.manual_seed(seed)
  la = SparseLinear(130, 77, name='a', device=DEV)       # 10010 weights: not a multiple of 4
  rng = np.random.RandomState(seed)
  la.mask.assign((rng.rand(130, 77) > 0.7).astype(F32))
  return la


def test_graph_replay_equals_eager_steps():
  """step() captured once and replayed with set_lr between replays == the same number of eager steps."""
  def run(graph, n=6):
    la = _two_layers(11)
    opt = FusedAdam(la.parameters(), lr=1e-2, weight_decay=1e-3)
    opt.attach_masked_layers([la], grad_scale=0.5)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(5)
    la.masked_weights.dense_grad.copy_(torch.randn(la.weight.numel(), device=DEV, generator=gen))
    la.bias.grad = torch.randn(la.bias.shape, device=DEV, generator=gen)
    if graph:
      opt.prepare()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        opt.step()
    for i in range(n):
      opt.set_lr(1e-2 / (1 + i))
      if graph:
        g.replay()
      else:
        opt.step()
    torch.cuda.synchronize()
    st = [opt.state[p] for p in (la.weight, la.bias)]
    return [_np(la.weight), _np(la.bias)] + [_np(s[k]) for s in st for k in ('exp_avg', 'exp_avg_sq')] + \
        [_np(opt._powers)]
  eager, graphed = run(False), run(True)
  for a, b in zip(eager, graphed):
    assert a.tobytes() == b.tobytes()
  p1, p2 = F32(0.9), F32(0.999)
  for _ in range(6):
    p1, p2 = ao.advance_powers(p1, p2, 0.9, 0.999)
  assert eager[-1].tobytes() == np.array([p1, p2], F32).tobytes()


def _mnist_layers(rng):
  layers = [SparseLinear(784, 300, name='layer1', device=DEV), SparseLinear(300, 100, name='layer2', device=DEV),
            SparseLinear(100, 10, name='layer3', device=DEV, out_dtype=torch.float32)]
  for l, s in zip(layers, (0.9, 0.81, 0.5)):
    l.mask.assign(orc.get_mask_random_numpy(tuple(l.weight.shape), s, rng))
  return layers


@pytest.mark.parametrize('acc_scale', [0.0, 0.5])
def test_rigl_over_adam_resets_both_moments_and_freezes_the_powers(acc_scale):
  """SparseRigLOptimizer over FusedAdam: the first update at global_step 0 resets exp_avg AND exp_avg_sq (created
  with the optimizer) to dense_grad * initial_acc_scale at new connections; update iterations do not advance the
  powers; inner steps equal the oracle bit for bit.
  With initial_acc_scale > 0 the reset writes negative values into exp_avg_sq wherever the dense gradient is
  negative (base.py:555-564 resets every slot alike), and sqrt(v) makes those weights NaN at the next step, as in
  the reference; that case stops after the first inner step, which must reproduce the NaNs exactly."""
  pruning.reset_default_registry()
  torch.manual_seed(1)
  rng = np.random.RandomState(1)
  layers = _mnist_layers(rng)
  params = [p for l in layers for p in l.parameters()]
  lr, wd = 1e-3, 1e-4
  inner = FusedAdam(params, lr=lr, weight_decay=wd)
  assert list(inner.state[layers[0].weight]) == ['exp_avg', 'exp_avg_sq']
  so = sparse_optimizers.SparseRigLOptimizer(inner, 0, 50000, 3, drop_fraction=0.3,
                                             drop_fraction_anneal='cosine', initial_acc_scale=acc_scale)
  assert so.get_slot_names() == ['exp_avg', 'exp_avg_sq']
  gs = GlobalStep(0)
  x = torch.randn(100, 784, device=DEV)
  target = torch.randint(0, 10, (100,), device=DEV)

  def loss_fn():
    h = torch.relu(layers[0](x))
    h = torch.relu(layers[1](h))
    return torch.nn.functional.cross_entropy(layers[2](h).float(), target)

  p1, p2 = F32(0.9), F32(0.999)
  iters = 8 if acc_scale == 0 else 2
  inner_steps = 0
  for it in range(iters):
    loss = loss_fn()
    gv = so.compute_gradients(loss)
    snap = [dict(mask=l.mask.numpy(), w=_np(l.weight), g=_np(l.masked_weights.dense_grad).reshape(l.weight.shape),
                 m=_np(inner.state[l.weight]['exp_avg']), v=_np(inner.state[l.weight]['exp_avg_sq']))
            for l in layers]
    before = {id(p): (_np(p), None if p.grad is None else _np(p.grad), _np(inner.state[p]['exp_avg']),
                      _np(inner.state[p]['exp_avg_sq'])) for p in params}
    step_before = gs.value
    so.apply_gradients(gv, gs)
    torch.cuda.synchronize()
    if it in (0, 4):          # gs 0 and gs 3 (the step counter is frozen on update iterations)
      assert so.last_update_was_mask_update and gs.value == step_before
      frac = orc.get_drop_fraction('cosine', 0.3, step_before, 0, 50000, True)
      grown = 0
      for l, s in zip(layers, snap):
        noise = so.last_update_noise(l.weight)
        noise = None if noise is None else _np(noise).reshape(s['w'].shape)
        want = orc.rigl_mask_update(s['mask'], s['w'], s['g'], frac, noise=noise, initial_acc_scale=acc_scale,
                                    slots=[s['m'], s['v']])
        assert np.array_equal(l.mask.numpy(), want['mask'])
        assert _np(l.weight).tobytes() == want['weights'].tobytes()
        assert _np(inner.state[l.weight]['exp_avg']).tobytes() == want['slots'][0].tobytes()
        assert _np(inner.state[l.weight]['exp_avg_sq']).tobytes() == want['slots'][1].tobytes()
        grown += int(want['new_connections'].sum())
      assert grown > 0
    else:
      assert not so.last_update_was_mask_update and gs.value == step_before + 1
      for p in params:
        w0, g0, m0, v0 = before[id(p)]
        ge = ao.optimizer_grad(w0, g0, weight_decay=wd)
        w1, m1, v1 = ao.adam_step(w0, m0, v0, ge, lr, 0.9, 0.999, 1e-8, p1, p2)
        assert _same(_np(p), w1)
        assert _np(inner.state[p]['exp_avg']).tobytes() == m1.tobytes()
        assert _same(_np(inner.state[p]['exp_avg_sq']), v1)
      if acc_scale:
        assert np.isnan(_np(layers[0].weight)).any()
      p1, p2 = ao.advance_powers(p1, p2, 0.9, 0.999)
      inner_steps += 1
    assert _np(inner._powers).tobytes() == np.array([p1, p2], F32).tobytes(), it
  # mask updates at iterations 0 and 4: powers = beta^(1 + inner steps) in float32
  assert inner_steps == (6 if acc_scale == 0 else 1)
  q1, q2 = F32(0.9), F32(0.999)
  for _ in range(inner_steps):
    q1, q2 = ao.advance_powers(q1, q2, 0.9, 0.999)
  assert (p1, p2) == (q1, q2)


def test_set_over_adam_advances_the_powers_every_step():
  pruning.reset_default_registry()
  torch.manual_seed(2)
  layers = _mnist_layers(np.random.RandomState(2))
  inner = FusedAdam([p for l in layers for p in l.parameters()], lr=1e-3)
  so = sparse_optimizers.SparseSETOptimizer(inner, 0, 100, 2, drop_fraction=0.3)
  gs = GlobalStep(0)
  x = torch.randn(64, 784, device=DEV)
  p1, p2 = F32(0.9), F32(0.999)
  updates = 0
  for _ in range(5):
    h = torch.relu(layers[1](torch.relu(layers[0](x))))
    so.minimize(layers[2](h).float().square().mean(), gs)
    updates += bool(so.last_update_was_mask_update)
    p1, p2 = ao.advance_powers(p1, p2, 0.9, 0.999)
    assert _np(inner._powers).tobytes() == np.array([p1, p2], F32).tobytes()
  assert updates >= 2 and gs.value == 5


def _harness(kind, graph, seed=7, steps=12):
  torch.manual_seed(seed)
  if kind == 'mnist':
    model = workloads.MnistFC(device=DEV)
    workloads.init_masks(model, 'random', 0.9, {'layer2': 0.81, 'layer3': 0.0}, seed=seed)
    h = workloads.TrainHarness(model, lr=1e-3, weight_decay=0.0, label_smoothing=0.0, frequency=4, end_step=1000,
                               inner_optimizer='adam')
    x = torch.randn(100, 784, device=DEV)
    y = (x[:, :10].argmax(1)).long()
  else:
    model = workloads.ResNet50(num_classes=10, device=DEV)
    workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=seed)
    h = workloads.TrainHarness(model, lr=1e-3, frequency=4, end_step=1000, inner_optimizer='adam')
    x = torch.randn(8, 3, 64, 64, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (8,), device=DEV)
  assert isinstance(h.inner, FusedAdam) and h.fused
  h.step(x, y)
  h.step(x, y)
  if graph:
    assert h.enable_cuda_graph(x, y)
  losses = [float(h.step(x, y).detach()) for _ in range(steps)]
  counts = [m.count_ones() for m in model.registry.get_masks()]
  return losses, h.global_step.value, _np(h.inner._powers), counts


@pytest.mark.parametrize('kind', ['mnist', 'resnet50'])
def test_train_step_with_adam_eager_and_graph(kind):
  le, ge, pe, ce = _harness(kind, False)
  lg, gg, pg, cg = _harness(kind, True)
  assert ge == gg and pe.tobytes() == pg.tobytes() and ce == cg
  assert ge == 11              # 14 steps; at gs 0, 4 and 8 a mask update ran instead of the inner step
  for losses in (le, lg):
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
  assert np.allclose(le, lg, rtol=2e-2, atol=2e-3)


def test_checkpoint_resume_is_bit_identical(tmp_path):
  """Save mid-run with variables_of(model, inner, sparse_opt), restore into a freshly built harness and continue:
  the same weights, moments, powers and masks as the uninterrupted run."""
  def build(seed=3):
    torch.manual_seed(seed)
    model = workloads.MnistFC(device=DEV)
    workloads.init_masks(model, 'random', 0.9, {'layer2': 0.81, 'layer3': 0.0}, seed=seed)
    h = workloads.TrainHarness(model, lr=1e-3, weight_decay=1e-4, label_smoothing=0.0, frequency=4,
                               end_step=1000, inner_optimizer='adam')
    return model, h

  gen = torch.Generator(device=DEV)
  gen.manual_seed(0)
  data = [torch.randn(100, 784, device=DEV, generator=gen) for _ in range(12)]
  batches = [(x, x[:, :10].argmax(1).long()) for x in data]

  def state(model, h):
    return [_np(t) for t in model.parameters()] + [m.numpy() for m in model.registry.get_masks()] + \
        [_np(t) for p in model.parameters() for t in h.inner.state[p].values()] + [_np(h.inner._powers)]

  model, h = build()
  for x, y in batches[:6]:
    h.step(x, y)
  variables = checkpoint.variables_of(model, h.inner, h.opt)
  for l in model.registry.layers():
    assert l.scope + '/weights/exp_avg' in variables and l.scope + '/weights/exp_avg_sq' in variables
  assert 'beta1_power' in variables and 'beta2_power' in variables
  path = checkpoint.save(str(tmp_path / 'run'), variables, h.global_step.value)
  saved_step = h.global_step.value
  for x, y in batches[6:]:
    h.step(x, y)
  want = state(model, h)

  model2, h2 = build(seed=4)                   # different initial weights and masks: all of it comes from the file
  h2.global_step.value = checkpoint.restore(path, checkpoint.variables_of(model2, h2.inner, h2.opt, ckpt_path=path))
  assert h2.global_step.value == saved_step
  for x, y in batches[6:]:
    h2.step(x, y)
  got = state(model2, h2)
  assert len(got) == len(want)
  for a, b in zip(got, want):
    assert a.tobytes() == b.tobytes()
