"""Fused BN(+ReLU,+residual) kernels vs a float64 restatement of batch_norm_relu
(rigl/imagenet_resnet/resnet_model.py:41-80) on the same bf16-rounded inputs.
Tolerances: bf16 outputs within 1 bf16 ulp of the fp64 result (+ tiny absolute slack);
fp32 reductions (dgamma, dbeta, running stats) rel 2e-3 of the reduction scale."""
import numpy as np
import pytest
import torch

from rigl_b200.norm import FusedBatchNormReLU

from isolated import assert_not_ran, assert_ran, run_isolated

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _bf(a):
  return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16)


def _nhwc_to_dev(a):
  return _bf(a).permute(0, 3, 1, 2).to(DEV).contiguous(memory_format=torch.channels_last)


def _close_bf16(got, want, what):
  got = got.detach().float().cpu().numpy().astype(np.float64)
  scale = np.abs(want).max() + 1e-30
  tol = np.abs(want) * 2.0 ** -7 + scale * 2.0 ** -9
  err = np.abs(got - want)
  assert (err <= tol).all(), '%s: max err %g at scale %g (%d bad)' % (what, err.max(), scale, (err > tol).sum())


@pytest.mark.parametrize('shape', [(4, 8, 8, 64), (2, 7, 7, 2048), (3, 5, 9, 24), (16, 28, 28, 128), (2, 3, 3, 8)])
@pytest.mark.parametrize('relu,residual', [(True, False), (False, False), (True, True)])
def test_bn_forward_backward(shape, relu, residual):
  n, h, w, c = shape
  rng = np.random.RandomState(c + n)
  y_np = _bf(rng.standard_normal(shape) * 1.7 + 0.3).float().numpy().astype(np.float64)
  r_np = _bf(rng.standard_normal(shape)).float().numpy().astype(np.float64) if residual else None
  da_np = _bf(rng.standard_normal(shape)).float().numpy().astype(np.float64)
  gamma = rng.rand(c) + 0.5
  beta = rng.standard_normal(c) * 0.2
  bn = FusedBatchNormReLU(c, relu=relu, device=DEV)
  with torch.no_grad():
    bn.weight.copy_(torch.from_numpy(gamma.astype(np.float32)))
    bn.bias.copy_(torch.from_numpy(beta.astype(np.float32)))
  gamma, beta = bn.weight.detach().cpu().double().numpy(), bn.bias.detach().cpu().double().numpy()
  y = _nhwc_to_dev(y_np).requires_grad_(True)
  r = _nhwc_to_dev(r_np).requires_grad_(True) if residual else None
  out = bn(y, residual=r)
  out.backward(_nhwc_to_dev(da_np))
  # ---- float64 reference
  m = n * h * w
  mean = y_np.reshape(m, c).mean(0)
  var = y_np.reshape(m, c).var(0)
  rstd = 1.0 / np.sqrt(var + 1e-5)
  xhat = (y_np - mean) * rstd
  z = gamma * xhat + beta + (r_np if residual else 0.0)
  want = np.maximum(z, 0) if relu else z
  _close_bf16(out.permute(0, 2, 3, 1), want, 'forward')
  # relu mask from the kernel's own (bf16) output avoids counting sign flips at |z| ~ 0 as errors
  a_got = out.detach().permute(0, 2, 3, 1).float().cpu().numpy()
  g = da_np * ((a_got > 0) if relu else 1.0)
  dbeta = g.reshape(m, c).sum(0)
  dgamma = (g * xhat).reshape(m, c).sum(0)
  dy = gamma * rstd * (g - dbeta / m - xhat * dgamma / m)
  _close_bf16(y.grad.permute(0, 2, 3, 1), dy, 'dy')
  red_scale = np.abs(g).sum(axis=(0, 1, 2)).max() + 1e-30
  assert np.abs(bn.bias.grad.cpu().double().numpy() - dbeta).max() <= 2e-3 * red_scale
  assert np.abs(bn.weight.grad.cpu().double().numpy() - dgamma).max() <= 2e-3 * red_scale * 3
  if residual:
    _close_bf16(r.grad.permute(0, 2, 3, 1), g, 'dresidual')
  assert np.allclose(bn.running_mean.cpu().numpy(), 0.1 * mean, rtol=1e-3, atol=1e-4)
  assert np.allclose(bn.running_var.cpu().numpy(), 0.9 + 0.1 * var * m / (m - 1), rtol=1e-3, atol=1e-4)


@pytest.mark.parametrize('shape', [(4, 8, 8, 64), (2, 7, 7, 2048), (3, 5, 9, 24)])
def test_bn_three_kernel_path(shape):
  """Small tensors take the single-launch (grid-barrier) kernels by default; RIGL_BN_FUSED=0 keeps the
  3-kernel path (the only one large tensors use) covered at oracle-checkable sizes."""
  calls = [('test_bn_forward_backward', (shape, relu, res)) for relu, res in ((True, False), (False, False), (True, True))]
  for ran in run_isolated('test_bn_gpu', calls, {'RIGL_BN_FUSED': '0'}):
    assert_ran(ran, r'k_bn_', shape)
    assert_not_ran(ran, r'k_bn_(fwd|bwd)_fused', shape)


@pytest.mark.parametrize('shape', [(4, 8, 8, 64), (2, 14, 14, 256), (3, 5, 9, 24)])
def test_bn_forked_output_sums_two_gradients_in_kernel(shape):
  """fork=True hands the block output out twice; the two incoming gradients are summed inside the
  backward column-sum pass (rigl_bn_backward), rounded to bf16 exactly like the elementwise add
  (tf AddN / autograd accumulation) it replaces: results are bit-identical to the un-forked BN fed
  with the pre-added gradient."""
  n, h, w, c = shape
  rng = np.random.RandomState(7 + c)
  y_np = rng.standard_normal(shape) * 1.3
  r_np = rng.standard_normal(shape)
  g1_np, g2_np = rng.standard_normal(shape), rng.standard_normal(shape) * 0.5
  res = {}
  for fork in (True, False):
    torch.manual_seed(0)
    bn = FusedBatchNormReLU(c, relu=True, device=DEV)
    with torch.no_grad():
      bn.weight.copy_(torch.linspace(0.5, 1.5, c))
      bn.bias.copy_(torch.linspace(-0.2, 0.2, c))
    y = _nhwc_to_dev(y_np).requires_grad_(True)
    r = _nhwc_to_dev(r_np).requires_grad_(True)
    g1, g2 = _nhwc_to_dev(g1_np), _nhwc_to_dev(g2_np)
    if fork:
      a1, a2 = bn(y, residual=r, fork=True)
      assert a1.data_ptr() == a2.data_ptr()
      torch.autograd.backward([a1, a2], [g1, g2])
    else:
      a1 = bn(y, residual=r)
      a1.backward(g1 + g2)                       # bf16 add: the separate elementwise pass
    res[fork] = (a1.detach().clone(), y.grad.clone(), r.grad.clone(), bn.weight.grad.clone(), bn.bias.grad.clone())
  for got, want, what in zip(res[True], res[False], ('out', 'dy', 'dresidual', 'dgamma', 'dbeta')):
    assert torch.equal(got, want), what
  # only one consumer used: the other gradient is absent, not zero-filled
  bn = FusedBatchNormReLU(c, relu=True, device=DEV)
  y = _nhwc_to_dev(y_np).requires_grad_(True)
  r = _nhwc_to_dev(r_np).requires_grad_(True)
  a1, a2 = bn(y, residual=r, fork=True)
  a2.backward(_nhwc_to_dev(g2_np))
  assert y.grad is not None and torch.isfinite(y.grad.float()).all()


def test_bn_eval_mode_and_errors():
  bn = FusedBatchNormReLU(16, relu=True, device=DEV)
  with torch.no_grad():
    bn.running_mean.normal_()
    bn.running_var.uniform_(0.5, 2.0)
    bn.weight.uniform_(0.5, 1.5)
    bn.bias.normal_()
  bn.eval()
  x = torch.randn(2, 16, 5, 5, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  got = bn(x).float()
  want = torch.relu((x.float() - bn.running_mean[None, :, None, None]) *
                    torch.rsqrt(bn.running_var + 1e-5)[None, :, None, None] * bn.weight[None, :, None, None] +
                    bn.bias[None, :, None, None])
  assert float((got - want).abs().max()) <= 2 ** -7 * float(want.abs().max()) + 1e-3
  with pytest.raises(ValueError):
    FusedBatchNormReLU(12, device=DEV)
  with pytest.raises(ValueError):
    bn(torch.zeros(2, 8, 5, 5, device=DEV))


@pytest.mark.parametrize('shape', [(2, 12, 12, 16), (3, 9, 7, 8), (2, 112, 112, 64)])
def test_maxpool_same_forward_backward(shape):
  from rigl_b200.norm import max_pool_same
  import torch.nn.functional as F
  n, h, w, c = shape
  torch.manual_seed(h)
  x = torch.randn(n, c, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  x.requires_grad_(True)
  y = max_pool_same(x, 3, 2)
  oh, ow = (h + 1) // 2, (w + 1) // 2
  ph, pw = max((oh - 1) * 2 + 3 - h, 0), max((ow - 1) * 2 + 3 - w, 0)
  xr = x.detach().float().clone().requires_grad_(True)
  yr = F.max_pool2d(F.pad(xr, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float('-inf')), 3, 2, 0)
  assert tuple(y.shape) == tuple(yr.shape) and torch.equal(y.float(), yr)
  dy = torch.randn_like(yr).to(torch.bfloat16).float()
  y.backward(dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
  yr.backward(dy)
  # each pixel gets the fp32 sum of the gradients of the windows whose FIRST maximum it is (tied maxima included),
  # windows in (oh, ow) order, rounded once to bf16
  from test_streaming_b256_gpu import maxpool_backward_reference, maxpool_reference
  want = maxpool_backward_reference(maxpool_reference(x.detach().float())[1], dy, h, w)
  assert torch.equal(x.grad, want)
  assert abs(float(x.grad.float().sum()) - float(dy.sum())) <= 1e-2 * float(dy.abs().sum())


# (n, h, w, cin, cout, k, stride, epilogue statistics expected): the halo kernels (3x3/s1, <= 64 channels) and the
# space-to-depth stem have no statistics epilogue and fall back to the stats pass; the rest covers the K-major
# kernel with both tile widths, several N tiles (cout 512 / 1024), pixel grids that do not fill their boxes (7x7, 13x9) and
# problems with many tiles per CTA, and ragged output widths (200 = a 128-wide tile + 72 channels, 72 = a partially
# valid second slab).
_BN_STATS_CASES = [(4, 56, 56, 64, 64, 3, 1, None), (4, 16, 16, 64, 128, 3, 1, True), (2, 28, 28, 128, 256, 1, 1, True),
                   (8, 14, 14, 64, 64, 3, 2, True), (3, 32, 32, 3, 64, 7, 2, False),
                   (1, 8, 8, 64, 64, 1, 1, True), (16, 7, 7, 256, 1024, 1, 1, True),
                   (5, 13, 9, 128, 512, 1, 1, True), (64, 56, 56, 64, 256, 1, 1, True),
                   (32, 28, 28, 128, 128, 3, 1, True), (6, 14, 14, 256, 256, 3, 2, True),
                   (4, 16, 16, 128, 200, 3, 1, True), (4, 14, 14, 256, 72, 1, 1, True)]


@pytest.mark.parametrize('case', _BN_STATS_CASES)
def test_conv_epilogue_bn_stats_match_stats_pass(case):
  """BN fed by the conv epilogue's statistics == BN with its own stats pass: both sum the bf16-ROUNDED
  outputs, in different orders (fp32 partials, fp64 combine)."""
  from rigl_b200 import layers, pruning
  n, h, w, cin, cout, k, stride, expect_epilogue = case
  torch.manual_seed(cout + k)
  pruning.reset_default_registry()
  conv = layers.SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', name='c', device=DEV)
  conv.mask.assign((torch.rand(k, k, cin, cout, device=DEV) > 0.5).float())
  conv.collect_bn_stats = True
  x = torch.randn(n, cin, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  outs = []
  old = layers.FUSE_BN_STATS
  from rigl_b200 import _cabi
  _cabi.lib().rigl_set_bn_stats_always(1)        # every supported shape, not only the profitable ones
  for fused in (True, False):
    layers.FUSE_BN_STATS = fused
    try:
      bn = FusedBatchNormReLU(cout, relu=True, device=DEV)
      y = conv(x)
      if expect_epilogue is not None:       # (None: halo-kernel eligibility decides; either way the results must agree)
        assert (conv.bn_partial is not None) == (fused and expect_epilogue)
      outs.append((bn(y, producer=conv).float(), bn.running_mean.clone(), bn.running_var.clone()))
    finally:
      layers.FUSE_BN_STATS = old
      if not fused:
        _cabi.lib().rigl_set_bn_stats_always(0)
  (a, ma, va), (b, mb, vb) = outs
  # same bf16 values summed in a different order: the statistics agree to fp32 summation noise
  assert float((ma - mb).abs().max()) <= 1e-5 * float(vb.sqrt().max()) * 10 + 1e-6
  assert torch.allclose(va, vb, rtol=1e-4, atol=1e-6)
  assert float((a - b).abs().max()) <= 2 ** -7 * float(b.abs().max()) + 1e-3


def test_conv_epilogue_bn_stats_only_where_profitable():
  """Default policy: short reductions with wide outputs (epilogue-bound layers) keep the separate stats pass."""
  from rigl_b200 import layers, pruning
  pruning.reset_default_registry()
  old, layers.FUSE_BN_STATS = layers.FUSE_BN_STATS, True
  try:
    for cin, cout, k, expect in ((64, 256, 1, False), (128, 512, 1, False), (256, 512, 1, False), (256, 64, 1, True),
                                (512, 128, 1, True), (128, 128, 3, True)):
      conv = layers.SparseConv2d(cin, cout, k, padding='FIXED', name='c%d_%d' % (cin, cout), device=DEV)
      conv.collect_bn_stats = True
      x = torch.randn(4, cin, 14, 14, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
      conv(x)
      assert (conv.bn_partial is not None) == expect, (cin, cout, k)
  finally:
    layers.FUSE_BN_STATS = old


@pytest.mark.parametrize('shape', [(4, 8, 8, 64), (2, 7, 7, 2048), (16, 28, 28, 128), (64, 56, 56, 64), (3, 5, 9, 24)])
@pytest.mark.parametrize('two_grads', [False, True])
def test_bn_residual_relu_bitmap_is_the_sign_of_the_output(shape, two_grads):
  """Residual form: the forward writes one bit per output element, out > 0 (k_bn_apply for C < 512, k_bn_fwd_fused
  for C = 2048), and the backward reads nothing else of the output.  So the bitmap must be exactly the output's ReLU
  mask; the backward, with one or two incoming gradients, runs on it."""
  from rigl_b200 import _cabi
  lib = _cabi.lib()
  n, h, w, c = shape
  rows = n * h * w
  rng = np.random.RandomState(c * 3 + n)
  y, r, da, db = (_bf(rng.standard_normal((rows, c)) * s).to(DEV) for s in (1.3, 1.0, 1.0, 1.0))
  gamma, beta = torch.linspace(0.5, 1.5, c, device=DEV), torch.linspace(-0.3, 0.3, c, device=DEV)
  save = torch.empty((4, c), dtype=torch.float32, device=DEV)
  out = torch.empty_like(y)
  bits = torch.full((rows * c // 8,), 0xFF, dtype=torch.uint8, device=DEV)
  ws = torch.empty(lib.rigl_bn_workspace_bytes(rows, c) + 8 * c + 256, dtype=torch.uint8, device=DEV)
  _cabi.check(lib.rigl_bn_forward_train(
      y.data_ptr(), r.data_ptr(), gamma.data_ptr(), beta.data_ptr(), rows, c, 1e-5, 0.1, 1, None, None,
      save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(), out.data_ptr(), ws.data_ptr(),
      ws.numel(), bits.data_ptr(), _cabi.stream_ptr()), 'rigl_bn_forward_train')
  want = np.packbits(out.float().cpu().numpy().reshape(-1) > 0, bitorder='little')
  assert np.array_equal(bits.cpu().numpy(), want)
  dy, dres = torch.empty_like(y), torch.empty_like(y)
  dgb = torch.empty((2, c), dtype=torch.float32, device=DEV)
  _cabi.check(lib.rigl_bn_backward(
      da.data_ptr(), db.data_ptr() if two_grads else None, y.data_ptr(), save[0].data_ptr(), save[1].data_ptr(),
      save[2].data_ptr(), save[3].data_ptr(), rows, c, 1, dy.data_ptr(), dres.data_ptr(), dgb[0].data_ptr(),
      dgb[1].data_ptr(), ws.data_ptr(), ws.numel(), bits.data_ptr(), _cabi.stream_ptr()), 'rigl_bn_backward')
  for t, what in ((dy, 'dy'), (dres, 'dresidual'), (dgb, 'dgamma/dbeta')):
    assert torch.isfinite(t.float()).all(), what
