"""optim.FusedMomentumSGD on the H100: k_sgd_nesterov_batched against the numpy restatement of sgd_one
(sgd_oracle) bit for bit -- every size class of the chunked task table, the scalar path, both update forms, the
whole ResNet-50 parameter set and a CUDA-graph replay."""
import ctypes as C

import numpy as np
import pytest
import torch

import sgd_oracle as so
from rigl_b200 import _cabi, pruning, workloads
from rigl_b200.layers import SparseLinear
from rigl_b200.masks import MaskVariable
from rigl_b200.optim import FusedMomentumSGD

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
F32 = np.float32
SIZES = (1, 3, 5, 31, 33, 8191, 8192, 8193, 2359296)     # scalar tails, the 8192-element chunk edges, a 3x3x512x512


def _np(t):
  return t.detach().cpu().numpy().copy()


def _bits(a):
  return np.ascontiguousarray(a, F32).view(np.uint32)


@pytest.mark.parametrize('momentum', [0.0, 0.9])
@pytest.mark.parametrize('nesterov', [True, False], ids=['nesterov', 'plain'])
def test_kernel_matches_oracle_bit_for_bit(nesterov, momentum):
  """rigl_sgd_plan_* directly: every size masked and dense, a parameter one float off 16-byte alignment (the scalar
  path) for the sizes up to a chunk and one more, weight decay 0 and 1e-4, grad scales 0.5 (masked) and 0.25
  (dense), nonzero initial momentum, five steps with an lr change.  The masked-out gradients are NaN: a masked-out
  weight only decays, so none may reach the result."""
  rng = np.random.RandomState(1 + int(nesterov) + int(10 * momentum))
  lib = _cabi.lib()
  params = []
  for n in SIZES:
    for masked, offset in ((False, 0), (True, 0), (True, 1), (False, 1)):
      if offset and n > 8193:
        continue
      base = [torch.empty(n + offset, device=DEV) for _ in range(3)]
      w, m, g = (b[offset:] for b in base)
      w.copy_(torch.from_numpy(rng.standard_normal(n).astype(F32)))
      m.copy_(torch.from_numpy((0.1 * rng.standard_normal(n)).astype(F32)))
      on = mask = None
      if masked:
        on = rng.rand(n) < 0.3
        mask = MaskVariable('p%d_%d' % (n, offset), (n,), DEV).assign(on.astype(F32))
      params.append(dict(w=w, m=m, g=g, mask=mask, on=on, base=base, wd=0.0 if len(params) % 2 else 1e-4,
                         scale=0.5 if masked else 0.25))
  assert any(p['w'].data_ptr() % 16 for p in params) and any(p['w'].data_ptr() % 16 == 0 for p in params)
  descs = (_cabi.SgdDesc * len(params))()
  for d, p in zip(descs, params):
    d.param, d.momentum, d.grad = p['w'].data_ptr(), p['m'].data_ptr(), p['g'].data_ptr()
    d.mask_bits = None if p['mask'] is None else p['mask'].bits.data_ptr()
    d.n, d.weight_decay, d.grad_scale = p['w'].numel(), p['wd'], p['scale']
  plan = C.c_void_p(None)
  _cabi.check(lib.rigl_sgd_plan_create(descs, len(params), C.byref(plan)), 'rigl_sgd_plan_create')
  lr_dev = torch.zeros(1, device=DEV)
  want = [dict(w=_np(p['w']), m=_np(p['m'])) for p in params]
  try:
    for step in range(5):
      lr = 0.1 if step < 3 else 0.025
      lr_dev.fill_(lr)
      for p, s in zip(params, want):
        g = rng.standard_normal(p['w'].numel()).astype(F32)
        if p['on'] is not None:
          g[~p['on']] = np.nan
        p['g'].copy_(torch.from_numpy(g))
        s['w'], s['m'] = so.sgd_step(s['w'], s['m'], g, p['on'], p['scale'], p['wd'], lr, momentum, nesterov)
      _cabi.check(lib.rigl_sgd_plan_run(plan, lr_dev.data_ptr(), momentum, int(nesterov), _cabi.stream_ptr()),
                  'rigl_sgd_plan_run')
      for i, (p, s) in enumerate(zip(params, want)):
        what = (step, i, p['w'].numel(), p['on'] is not None, p['w'].data_ptr() % 16)
        got_w = _np(p['w'])
        assert np.isfinite(got_w).all(), what
        assert _bits(got_w).tobytes() == _bits(s['w']).tobytes(), what + ('w',)
        assert _bits(_np(p['m'])).tobytes() == _bits(s['m']).tobytes(), what + ('m',)
  finally:
    lib.rigl_sgd_plan_destroy(plan)


def _resnet50_optimizer(seed):
  pruning.reset_default_registry()
  torch.manual_seed(seed)
  model = workloads.ResNet50(num_classes=1000, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=seed)
  layers = model.registry.layers()
  opt = FusedMomentumSGD(model.parameters(), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-4)
  opt.attach_masked_layers(layers, grad_scale=0.5, other_grad_scale=0.25)
  return model, layers, opt


def test_resnet50_parameter_set_bit_for_bit():
  """FusedMomentumSGD over every ResNet-50 parameter -- the 54 masked tensors (25.5 M weights, mask * dense_grad
  formed in the kernel), the 53 batch norms' gamma and beta and the classifier bias -- for three steps with an lr
  change through set_lr, against the restatement: weights and momentum slots bit for bit."""
  model, layers, opt = _resnet50_optimizer(5)
  masked = {id(l.weight): l for l in layers}
  params = list(model.parameters())
  others = [p for p in params if id(p) not in masked]
  assert len(layers) == 54 and sum(l.weight.numel() for l in layers) > 25_000_000
  assert len(others) == 2 * 53 + 1 and any(p is model.final_dense.bias for p in others)
  gen = torch.Generator(device=DEV)
  gen.manual_seed(5)
  want = {id(p): (_np(p), np.zeros(p.numel(), F32).reshape(p.shape)) for p in params}
  for step in range(3):
    if step == 2:
      opt.set_lr(0.05)
    lr = opt.param_groups[0]['lr']
    for p in params:
      l = masked.get(id(p))
      if l is not None:
        l.masked_weights.dense_grad.copy_(torch.randn(p.numel(), device=DEV, generator=gen))
        g, on, scale = _np(l.masked_weights.dense_grad).reshape(p.shape), l.mask.numpy().astype(bool), 0.5
      else:
        p.grad = torch.randn(p.shape, device=DEV, generator=gen)
        g, on, scale = _np(p.grad), None, 0.25
      w0, m0 = want[id(p)]
      want[id(p)] = so.sgd_step(w0, m0, g, on, scale, 1e-4, lr, 0.9, True)
    opt.step()
    torch.cuda.synchronize()
    for i, p in enumerate(params):
      w1, m1 = want[id(p)]
      assert _bits(_np(p)).tobytes() == _bits(w1).tobytes(), (step, i, tuple(p.shape), 'weights')
      assert _bits(_np(opt.state[p]['momentum_buffer'])).tobytes() == _bits(m1).tobytes(), (step, i, 'momentum')
  for l in layers:
    assert l.weight.grad is None                    # the masked gradient is formed in the kernel, never stored
  del model, opt
  torch.cuda.empty_cache()


def test_graph_replay_equals_eager_steps():
  """step() captured once and replayed with set_lr between replays == the same number of eager steps == the
  restatement, bit for bit (a masked 130 x 77 layer: 10010 weights, not a multiple of 4, and its bias)."""
  def run(graph, n=6):
    pruning.reset_default_registry()
    torch.manual_seed(11)
    la = SparseLinear(130, 77, name='a', device=DEV)
    on = np.random.RandomState(11).rand(130, 77) > 0.7
    la.mask.assign(on.astype(F32))
    opt = FusedMomentumSGD(la.parameters(), lr=0.1, momentum=0.9, nesterov=True, weight_decay=1e-3)
    opt.attach_masked_layers([la], grad_scale=0.5, other_grad_scale=0.25)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(5)
    la.masked_weights.dense_grad.copy_(torch.randn(la.weight.numel(), device=DEV, generator=gen))
    la.bias.grad = torch.randn(la.bias.shape, device=DEV, generator=gen)
    start = (_np(la.weight), _np(la.bias), _np(la.masked_weights.dense_grad).reshape(130, 77), _np(la.bias.grad), on)
    if graph:
      opt.prepare()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        opt.step()
    for i in range(n):
      opt.set_lr(0.1 / (1 + i))
      if graph:
        g.replay()
      else:
        opt.step()
    torch.cuda.synchronize()
    st = [opt.state[p]['momentum_buffer'] for p in (la.weight, la.bias)]
    return [_np(la.weight), _np(la.bias)] + [_np(s) for s in st], start
  eager, start = run(False)
  graphed, _ = run(True)
  for a, b in zip(eager, graphed):
    assert _bits(a).tobytes() == _bits(b).tobytes()
  w, b, gw, gb, on = start
  mw, mb = np.zeros_like(w), np.zeros_like(b)
  for i in range(6):
    lr = 0.1 / (1 + i)
    w, mw = so.sgd_step(w, mw, gw, on, 0.5, 1e-3, lr, 0.9, True)
    b, mb = so.sgd_step(b, mb, gb, None, 0.25, 1e-3, lr, 0.9, True)
  for got, want in zip(eager, (w, b, mw, mb)):
    assert _bits(got).tobytes() == _bits(want).tobytes()
