"""MobileNet-v2 on the CUDA hot path: the linear-bottleneck batch-norm forms of csrc/bn.cu, the conv and depthwise
shapes the network runs, and the whole model (layer table, forward, train step against the CPU restatement, CUDA
graph replay).  Whole-step figures are recorded like the other models' (test_whole_step_parity_gpu._record)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mobilenet_v2_oracle as mo
import test_conv_gpu as tcg
import test_whole_step_parity_gpu as wsp
from isolated import assert_not_ran, assert_ran, run_isolated
from oracle import rigl_oracle as orc
from rigl_b200 import pruning, sparse_utils, workloads
from rigl_b200.layers import SparseConv2d
from rigl_b200.norm import FusedBatchNormReLU

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ---------------------------------------------------------------------------------------------------------------
# Batch norm without ReLU (the contraction BN): residual with one / two output gradients, plain with two.
# ---------------------------------------------------------------------------------------------------------------
def _dev_bf16(shape, seed, scale=1.0, shift=0.0):
  g = torch.Generator(device=DEV).manual_seed(seed)
  t = torch.randn(shape, device=DEV, generator=g) * scale + shift
  return t.to(torch.bfloat16).permute(0, 3, 1, 2)          # logical NCHW, channels_last storage


def _close_bf16(got, want, what):
  """Within one bf16 ulp of the float64 result (+ a little absolute slack), as tests/test_bn_gpu.py."""
  got = got.double()
  scale = float(want.abs().max()) + 1e-30
  tol = want.abs() * 2.0 ** -7 + scale * 2.0 ** -9
  bad = (got - want).abs() > tol
  assert not bool(bad.any()), '%s: max err %g at scale %g (%d bad)' % (what, float((got - want).abs().max()), scale,
                                                                     int(bad.sum()))


def _run_linear_bn(shape, form, fork=True):
  """form: 'res1' residual, one consumer; 'res2' residual, output forked to two consumers; 'plain2' no residual,
  forked.  fork=False feeds the un-forked BN the pre-added bf16 gradient instead.  Returns the module, the
  inputs, the output and every gradient."""
  n, h, w, c = shape
  bn = FusedBatchNormReLU(c, relu=False, device=DEV)
  with torch.no_grad():
    bn.weight.copy_(torch.linspace(0.5, 1.5, c))
    bn.bias.copy_(torch.linspace(-0.3, 0.3, c))
  y = _dev_bf16(shape, c + n, 1.4, 0.2).requires_grad_(True)
  r = _dev_bf16(shape, c + 1).requires_grad_(True) if form != 'plain2' else None
  g1 = _dev_bf16(shape, c + 2)
  g2 = _dev_bf16(shape, c + 3, 0.5) if form != 'res1' else None
  if g2 is not None and fork:
    a1, a2 = bn(y, residual=r, fork=True)
    assert a1.data_ptr() == a2.data_ptr()
  else:
    a1 = bn(y, residual=r)
  assert a1.grad_fn.saved_tensors[1] is None          # (y, ReLU bitmap, statistics): no bitmap without a ReLU
  if g2 is not None and fork:
    torch.autograd.backward([a1, a2], [g1, g2])
  else:
    a1.backward(g1 if g2 is None else g1 + g2)           # bf16 add: the separate elementwise pass
  return bn, y, r, g1, g2, a1


def bn_linear_form_vs_fp64(shape, form):
  bn, y, r, g1, g2, out = _run_linear_bn(shape, form)
  n, h, w, c = shape
  m = n * h * w
  yd = y.detach().permute(0, 2, 3, 1).reshape(m, c).double()
  mean = yd.mean(0)
  var = yd.var(0, unbiased=False)
  rstd = 1.0 / torch.sqrt(var + 1e-5)
  xhat = (yd - mean) * rstd
  gamma, beta = bn.weight.detach().double(), bn.bias.detach().double()
  z = gamma * xhat + beta
  if r is not None:
    z = z + r.detach().permute(0, 2, 3, 1).reshape(m, c).double()
  _close_bf16(out.detach().permute(0, 2, 3, 1).reshape(m, c), z, 'forward %s %s' % (form, shape))
  g = g1.permute(0, 2, 3, 1).reshape(m, c)
  if g2 is not None:       # the two consumers' gradients, summed and rounded to bf16 like the add it replaces
    g = g + g2.permute(0, 2, 3, 1).reshape(m, c)
  g = g.double()
  dbeta, dgamma = g.sum(0), (g * xhat).sum(0)
  dy = gamma * rstd * (g - dbeta / m - xhat * dgamma / m)
  _close_bf16(y.grad.permute(0, 2, 3, 1).reshape(m, c), dy, 'dy %s %s' % (form, shape))
  red = float(g.abs().sum(0).max()) + 1e-30
  assert float((bn.bias.grad.double() - dbeta).abs().max()) <= 2e-3 * red
  assert float((bn.weight.grad.double() - dgamma).abs().max()) <= 6e-3 * red
  if r is not None:
    assert torch.equal(r.grad.permute(0, 2, 3, 1).reshape(m, c).double(), g), 'dresidual %s %s' % (form, shape)
  assert torch.allclose(bn.running_mean, 0.1 * mean.float(), rtol=1e-3, atol=1e-4)


# C in {16, 24, 96, 160, 320} at MobileNet-v2's spatial sizes, small batches; the last shape (102 MB) is above the
# single-launch kernels' 64 MB and takes the three-kernel path by default.
_BN_SHAPES = [(4, 28, 28, 16), (3, 14, 14, 24), (2, 14, 14, 96), (4, 7, 7, 160), (8, 7, 7, 320), (2, 9, 5, 24),
              (256, 112, 112, 16)]


@pytest.mark.parametrize('form', ['res1', 'res2', 'plain2'])
@pytest.mark.parametrize('shape', _BN_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_bn_linear_forms_vs_fp64(shape, form):
  bn_linear_form_vs_fp64(shape, form)


def bn_forked_equals_pre_added(shape, form):
  """The in-kernel gradient sum is bit-identical to the un-forked BN fed the pre-added bf16 gradient; the residual
  form with one consumer hands its output gradient back as the shortcut's, unchanged; no ReLU bitmap exists."""
  res = {}
  for fork in (True, False):
    torch.manual_seed(0)
    bn, y, r, g1, g2, a1 = _run_linear_bn(shape, form, fork=fork)
    res[fork] = [a1.detach().clone(), y.grad.clone(), bn.weight.grad.clone(), bn.bias.grad.clone()] + \
        ([r.grad.clone()] if r is not None else [])
    if form == 'res1':
      assert torch.equal(r.grad, g1)
  for got, want, what in zip(res[True], res[False], ('out', 'dy', 'dgamma', 'dbeta', 'dresidual')):
    assert torch.equal(got, want), (what, form, shape)


_PATH_SHAPES = [(4, 8, 8, 64), (3, 14, 14, 24), (2, 7, 7, 320), (4, 28, 28, 16)]


@pytest.mark.parametrize('path', ['single_launch', 'three_kernel'])
def test_bn_linear_forms_on_both_bn_paths(path):
  env = {'RIGL_BN_FUSED': '0'} if path == 'three_kernel' else {}
  calls = []
  for shape in _PATH_SHAPES:
    for form in ('res1', 'res2', 'plain2'):
      calls += [('bn_forked_equals_pre_added', (shape, form)), ('bn_linear_form_vs_fp64', (shape, form))]
  ran = run_isolated('test_mobilenet_v2_gpu', calls, env)
  for (fn, (shape, form)), names in zip(calls, ran):
    what = '%s %s %s' % (fn, form, shape)
    if form != 'res1':                # two gradients: the no-ReLU residual-form kernels sum them
      assert_ran(names, r'k_bn_(colsum|bwd_fused)<3>', what)
    assert_not_ran(names, r'k_bn_(colsum|bwd_fused)<2>', what)
    if path == 'three_kernel':
      assert_not_ran(names, r'k_bn_(fwd|bwd)_fused', what)
    elif form != 'res1':
      assert_ran(names, r'k_bn_bwd_fused<3>', what)


# ---------------------------------------------------------------------------------------------------------------
# Conv and depthwise shapes
# ---------------------------------------------------------------------------------------------------------------
def _conv_shapes(batch):
  sp = mo.erk_sparsities(0.8)
  seen, out = set(), []
  for name, sh, _, hw in mo.masked_layers():
    if len(sh) != 4 or (hw, sh[2], sh[3]) in seen:
      continue
    seen.add((hw, sh[2], sh[3]))
    out.append((batch, hw, hw, sh[2], sh[3], 1, 1, round(float(sp[name + '/mask:0']), 3)))
  return out


_IDS = lambda c: 'h%d_c%d_%d' % (c[1], c[3], c[4])


@pytest.mark.parametrize('case', _conv_shapes(2), ids=_IDS)
def test_every_mobilenet_v2_conv_shape_vs_fp64(case):
  tcg._conv_case(case, force_simt=False)


@pytest.mark.parametrize('case', [c for c in _conv_shapes(256) if {16, 24} & {c[3], c[4]}], ids=_IDS)
def test_narrow_conv_shapes_b256_tensor_core_vs_cuda_core(case):
  """GEMM N or K of 16 / 24 (narrower than one 64-wide tile) at the two largest spatial sizes, batch 256."""
  n, h, w, cin, cout, k, stride, sparsity = case
  rng = np.random.RandomState(cin * 7 + cout)
  pruning.reset_default_registry()
  layer = SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', name='t', device=DEV)
  layer.mask.assign(orc.get_mask_random_numpy((k, k, cin, cout), sparsity, rng).astype(np.float32))
  g = torch.Generator(device=DEV).manual_seed(cin + cout)
  x = torch.randn((n, cin, h, w), device=DEV, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  dy = torch.randn((n, cout, h, w), device=DEV, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  y1, dx1, dw1 = tcg._run_both(layer, x, dy, force_simt=False)
  y0, dx0, dw0 = tcg._run_both(layer, x, dy, force_simt=True)
  for got, want, what in ((y1, y0, 'fprop'), (dx1, dx0, 'dgrad')):
    scale = float(want.abs().max())
    bad = (got - want).abs() > want.abs() * 2.0 ** -7 + scale * 2e-5
    assert not bool(bad.any()), '%s %s: %d elements off, max err %g (scale %g)' % (
        what, case, int(bad.sum()), float((got - want).abs().max()), scale)
  scale = float(dw0.abs().max())
  assert float((dw1 - dw0).abs().max()) <= 5e-5 * scale, 'wgrad %s' % (case,)


_DW = sorted({(hw, c, s) for _, c, s, hw, _ in mo.depthwise_layers()}, reverse=True)


@pytest.mark.parametrize('hw,c,stride', _DW, ids=lambda v: str(v))
def test_native_depthwise_on_mobilenet_v2_shapes_vs_fp64(hw, c, stride):
  tcg.test_depthwise3x3_vs_fp64((2, hw, hw, c, stride))


# ---------------------------------------------------------------------------------------------------------------
# The model
# ---------------------------------------------------------------------------------------------------------------
def test_registry_equals_the_layer_table_and_erk_counts():
  import json
  import os
  with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden',
                         'mobilenet_v2_sparsities_golden.json')) as f:
    golden = {c['tag']: c for c in json.load(f)['cases']}
  for prune_last in (True, False):
    torch.manual_seed(0)
    model = workloads.MobileNetV2(prune_last_layer=prune_last, device=DEV)
    want = [(n + '/mask:0', list(sh)) for n, sh, _, _ in mo.masked_layers(1000, prune_last)]
    assert [(m.name, list(m.shape)) for m in model.registry.get_masks()] == want
    for s in (0.8, 0.9):
      case = golden['mobilenet_v2_erdos_renyi_kernel%g_%s' % (s, 'prune_last' if prune_last else 'dense_last')]
      sp = workloads.init_masks(model, 'erdos_renyi_kernel', s, seed=1)
      for m in model.registry.get_masks():
        size = int(np.prod(m.shape))
        assert float(sp[m.name]).hex() == case['sparsities_hex'][m.name], m.name
        assert m.count_ones() == size - sparse_utils.get_n_zeros(size, sp[m.name]) == case['nnz'][m.name], m.name
    assert len([m for m in model.modules() if isinstance(m, workloads.DepthwiseConv2d)]) == 17


def _q(t):
  return t.to(torch.bfloat16)


def _stock_forward(model, x, training):
  """The same network on stock torch: cuDNN convs on bf16(mask * W), torch batch norm (fp32 arithmetic on the bf16
  activations, rounded to bf16 where the CUDA path stores), with copies of the running statistics."""
  def conv(layer, t):
    w = (layer.weight.detach() * layer.mask.to_dense()).to(torch.bfloat16).permute(3, 2, 0, 1).contiguous()
    return F.conv2d(t, w)

  def bn(mod, t, residual=None):
    o = F.batch_norm(t.float(), mod.running_mean.clone(), mod.running_var.clone(), mod.weight.detach(),
                     mod.bias.detach(), training=training, momentum=mod.momentum, eps=mod.eps)
    if residual is not None:
      o = o + residual.float()
    return _q(torch.relu(o) if mod.relu else o)
  t = bn(model.initial_bn, F.conv2d(x, model.initial_conv.weight.detach().to(torch.bfloat16), stride=2, padding=1))
  for blk in model.blocks:
    h = t
    if blk.expand is not None:
      h = bn(blk.bn_expand, conv(blk.expand, h))
    h = bn(blk.bn_dw, F.conv2d(h, blk.depthwise.weight.detach().to(torch.bfloat16), None, blk.depthwise.stride, 1, 1,
                               h.shape[1]))
    t = bn(blk.bn_contraction, conv(blk.contraction, h), residual=t if blk.shortcut else None)
  t = bn(model.final_bn, conv(model.final_conv, t)).mean(dim=(2, 3))
  fc = model.final_dense
  return t.float() @ (fc.weight.detach() * fc.mask.to_dense()).to(torch.bfloat16).float() + fc.bias.detach()


def test_forward_matches_stock_torch_in_train_and_eval_mode():
  torch.manual_seed(1)
  model = workloads.MobileNetV2(device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=1)
  x = torch.randn(8, 3, 64, 64, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  errs = {}
  for mode in ('train', 'eval'):
    model.train(mode == 'train')
    with torch.no_grad():
      want = _stock_forward(model, x, mode == 'train')
      got = model(x)
    assert got.shape == (8, 1000) and got.dtype == torch.float32 and torch.isfinite(got).all()
    errs[mode] = (float((got - want).abs().max()) / float(want.abs().max()),
                  float((got - want).norm()) / float(want.norm()))
  wsp._record('mobilenet_v2_forward', errs)
  # Eval mode (fixed statistics): the two builds agree to fp32 noise (measured on an H100: max 2.6e-7 of the largest
  # logit).  Train mode: each of the 52 BNs normalises with statistics summed in a different order (conv epilogue /
  # stats pass vs torch), and the rare bf16 rounding flips that causes grow ~1.2x per BN (DESIGN.md 5): measured
  # rel L2 0.13 at batch 8, 64x64 (0.07 at 128x128); bounded at about 3x that.
  assert errs['eval'][0] <= 1e-3, errs
  assert errs['train'][1] <= 0.4, errs


def _oracle_and_model(seed):
  net = mo.CpuMobileNetV2(sparsity=0.9, seed=seed, bf16_weights=True)
  net.bn_init, net.bf16_act = wsp._bn_init(seed), True
  model = workloads.MobileNetV2(device=DEV)
  with torch.no_grad():
    model.initial_conv.weight.copy_(net.p['initial_conv'].detach().permute(3, 2, 0, 1).to(DEV))
    for i, blk in enumerate(model.blocks):
      blk.depthwise.weight.copy_(net.p['depthwise_%d' % i].detach().to(DEV))
  return net, model


def test_mobilenet_v2_step_vs_cpu_oracle():
  """Teacher-forced bounds on all 35 masked layers (fprop / dgrad 1e-3, dense wgrad 2e-5), the free-running step
  bounded at about 3x the measured figure of the last layers, then bit-exact drop / grow over 4 steps.
  Measured on an H100 (seed below): teacher-forced worst fprop 1.2e-5, dgrad 3.5e-5, dense wgrad 5e-7; loss
  6.88972 vs 6.88986; free-running dense-gradient rel L2 median 0.38 / max 0.47 over the 35 layers, like
  MobileNet-v1 a BN stack that amplifies rounding flips from the classifier down, and 0.24 (`final_1x1_conv`) /
  0.025 (`final_dense`) on the last two, which are bounded at 0.7."""
  torch.manual_seed(3)
  net, model = _oracle_and_model(14)
  images = torch.randn(8, 3, 64, 64).to(torch.bfloat16)
  labels = torch.randint(0, 1000, (8,))
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  rel = wsp._compare_step('mobilenet_v2', model, net, images, labels, h, loss_tol=2e-2, grad_tol=0.7,
                          label_smoothing=0.1, last_layers=2)
  assert len(rel) == 35
  wsp._check_update_steps(model, h, images, labels, 4, [0, 2])


def _train(graph, inner, steps=5):
  torch.manual_seed(5)
  model = workloads.MobileNetV2(num_classes=100, device=DEV)
  for m in model.modules():
    if isinstance(m, workloads.DepthwiseConv2d):
      m.native = True                # the project's depthwise kernels: deterministic weight gradients
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=5)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100, inner_optimizer=inner)
  x = torch.randn(16, 3, 64, 64, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  y = torch.randint(0, 100, (16,), device=DEV)
  if graph:
    assert h.enable_cuda_graph(x, y)
  losses, masks = [], []
  for _ in range(steps):
    losses.append(h.step(x, y).detach().clone())
    masks.append([m.numpy().copy() for m in model.registry.get_masks()])
  torch.cuda.synchronize()
  weights = [l.weight.detach().clone() for l in model.registry.layers()]
  return torch.stack(losses), masks, weights, h.global_step.value


@pytest.mark.parametrize('inner', ['momentum', 'adam'])
def test_cuda_graph_replay_bit_identical_to_eager(inner):
  """Five steps with mask updates at global steps 0 and 2: graph replay and the eager step give the same losses,
  masks and weights bit for bit (the initial conv's cuDNN kernels run in deterministic mode)."""
  old = torch.backends.cudnn.deterministic
  torch.backends.cudnn.deterministic = True
  try:
    le, me, we, ge = _train(False, inner)
    lg, mg, wg, gg = _train(True, inner)
  finally:
    torch.backends.cudnn.deterministic = old
  assert ge == gg == 3
  assert torch.isfinite(le).all()
  assert torch.equal(le, lg), (le.tolist(), lg.tolist())
  for a, b in zip(me, mg):
    assert all(np.array_equal(p, q) for p, q in zip(a, b))
  for a, b in zip(we, wg):
    assert torch.equal(a, b)
