"""Masked conv / linear fprop, dgrad and dense wgrad vs the float64 CPU oracle.

Tolerance (floating point, north_star: 1e-5 rel on fp32 accumulators): inputs are
rounded to bf16 ONCE on the host and fed identically to both sides, so the only
differences are fp32 accumulation order (checked at rtol 2e-5 of the output scale
on the fp32 outputs) and the single final rounding to bf16 (<= 1 bf16 ulp =
2^-8 relative, checked on the bf16 outputs).
"""
import numpy as np
import pytest
import torch

from oracle import rigl_oracle as orc
from rigl_b200 import _cabi
from rigl_b200.layers import SparseConv2d, SparseLinear
from rigl_b200 import pruning

from isolated import assert_not_ran, assert_ran, run_isolated
from tile_masks import STRUCTURED_CONV_CASES, STRUCTURED_LINEAR_CASES, tile_counts, tile_mask

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _bf16(a):
  return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16)


def _check_bf16(got, want, what):
  got = got.detach().float().cpu().numpy().astype(np.float64)
  scale = np.abs(want).max() + 1e-30
  err = np.abs(got - want)
  tol = np.maximum(np.abs(want) * 2.0 ** -8, scale * 2.0 ** -16) * 1.01 + scale * 2e-5
  assert (err <= tol).all(), '%s: max err %g (scale %g) at %d positions' % (
      what, err.max(), scale, int((err > tol).sum()))


def _check_f32(got, want, what, rtol=2e-5):
  got = got.detach().float().cpu().numpy().astype(np.float64)
  scale = np.abs(want).max() + 1e-30
  assert np.abs(got - want).max() <= rtol * scale, '%s: max err %g scale %g' % (
      what, np.abs(got - want).max(), scale)


CONV_CASES = [
    # n, h, w, cin, cout, k, stride, sparsity
    (2, 8, 8, 16, 32, 3, 1, 0.5),
    (2, 9, 7, 8, 16, 3, 2, 0.8),
    (3, 8, 8, 64, 64, 1, 1, 0.0),
    (2, 14, 14, 64, 128, 1, 2, 0.4),
    (2, 12, 12, 3, 8, 7, 2, 0.14),      # stem-like: cin=3 (space-to-depth stem / SIMT)
    (3, 32, 32, 3, 64, 7, 2, 0.14),
    (2, 17, 17, 3, 16, 3, 1, 0.3),
    (4, 16, 16, 64, 64, 3, 1, 0.64),
    (8, 14, 14, 128, 128, 3, 1, 0.82),
    (4, 28, 28, 128, 128, 3, 2, 0.82),
    (16, 7, 7, 256, 256, 3, 1, 0.95),
    (32, 7, 7, 512, 128, 1, 1, 0.7),
    # TensorFlow 'SAME' incl. the asymmetric stride-2 case (WRN, cifar_resnet/resnet_model.py:158-181)
    (4, 32, 32, 16, 32, 3, 2, 0.8, 'SAME'),
    (2, 16, 16, 64, 128, 3, 2, 0.9, 'SAME'),
    (2, 15, 15, 32, 64, 3, 2, 0.5, 'SAME'),
    (2, 16, 16, 32, 64, 1, 2, 0.2, 'VALID'),
    (2, 9, 9, 16, 16, 3, 1, 0.3, 'VALID'),
    # ragged channel counts above 64: partially valid second 64-channel slab of a 128-wide N tile (fprop cout,
    # dgrad cin), N tiles that start at channel 128 with a few channels valid, ragged K blocks; two or more M tiles
    # in fprop and in every dgrad parity class
    (4, 8, 8, 72, 136, 1, 1, 0.5),
    (4, 16, 16, 96, 200, 1, 2, 0.6),
    (4, 8, 8, 200, 72, 3, 1, 0.7),
    (4, 16, 16, 136, 200, 3, 2, 0.8),
    (3, 7, 7, 72, 72, 3, 1, 0.5),
    (4, 11, 11, 200, 136, 3, 2, 0.6, 'SAME'),
]


def _conv_case(case, force_simt, mask=None):
  """`mask`: None (uniformly random at the case's sparsity) or a tile_masks pattern name (dead 64x64 weight tiles;
  the sparsity then applies inside the live tiles)."""
  n, h, w, cin, cout, k, stride, sparsity = case[:8]
  padding = case[8] if len(case) > 8 else 'FIXED'
  rng = np.random.RandomState(abs(hash(case[:8])) % (2 ** 31))
  pruning.reset_default_registry()
  _cabi.lib().rigl_set_force_simt(1 if force_simt else 0)
  try:
    layer = SparseConv2d(cin, cout, k, strides=stride, padding=padding, name='t', device=DEV)
    w_np = _bf16(rng.standard_normal((k, k, cin, cout)) / np.sqrt(k * k * cin)).float().numpy()
    if mask is None:
      m_np = orc.get_mask_random_numpy((k, k, cin, cout), sparsity, rng).astype(np.float32)
    else:
      m_np = tile_mask(mask, (k, k, cin, cout), rng, sparsity)
    with torch.no_grad():
      layer.weight.copy_(torch.from_numpy(w_np))
    layer.mask.assign(m_np)
    x_np = _bf16(rng.standard_normal((n, h, w, cin))).float().numpy()
    x = torch.from_numpy(x_np).permute(0, 3, 1, 2).to(DEV).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last).requires_grad_(True)
    y = layer(x)
    wm = (w_np * m_np).astype(np.float64)
    (ho, pad), (wo, _) = layer.out_size(h), layer.out_size(w)
    if padding == 'SAME':
      assert (ho, pad) == orc.tf_same_padding(h, k, stride)[:2]
    y_want = orc.conv2d_nhwc_general(x_np.astype(np.float64), wm, stride, pad, (ho, wo))
    assert tuple(y.shape) == (n, cout, y_want.shape[1], y_want.shape[2])
    _check_bf16(y.permute(0, 2, 3, 1), y_want, 'fprop %s' % (case,))
    dy_np = _bf16(rng.standard_normal(y_want.shape)).float().numpy()
    dy = torch.from_numpy(dy_np).permute(0, 3, 1, 2).to(DEV).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last)
    y.backward(dy)
    dx_want, dw_want = orc.conv2d_nhwc_general_bwd(x_np.astype(np.float64), wm, dy_np.astype(np.float64), stride, pad)
    _check_bf16(x.grad.permute(0, 2, 3, 1), dx_want, 'dgrad %s' % (case,))
    # dense wgrad: every position, including masked-out ones (RigL grow scores)
    _check_f32(layer.masked_weights.dense_grad.view(k, k, cin, cout), dw_want, 'wgrad %s' % (case,))
    # dL/dweights = mask * dense
    _check_f32(layer.weight.grad, dw_want * m_np, 'masked wgrad %s' % (case,))
    assert (layer.weight.grad.detach().cpu().numpy()[m_np == 0] == 0).all()
  finally:
    _cabi.lib().rigl_set_force_simt(0)


@pytest.mark.parametrize('case', CONV_CASES[:6])
def test_conv_simt_path(case):
  _conv_case(case, force_simt=True)


@pytest.mark.parametrize('case', CONV_CASES)
def test_conv_default_path(case):
  _conv_case(case, force_simt=False)


LINEAR_CASES = [(1, 3, 5, 0.5), (100, 784, 300, 0.9), (100, 300, 100, 0.81), (100, 100, 10, 0.0),
                (256, 2048, 1000, 0.85), (37, 64, 64, 0.3), (130, 200, 200, 0.6), (64, 136, 72, 0.5)]


def _linear_case(case, force_simt, out='f32', use_bias=True, mask=None):
  """`out`: 'f32' or 'bf16' output; `mask` as in _conv_case.  bf16 output without a bias takes the TMA-store
  epilogue, fp32 output or a bias the per-thread stores."""
  m_rows, n_in, n_out, sparsity = case
  out_dtype = {'f32': torch.float32, 'bf16': torch.bfloat16}[out]
  rng = np.random.RandomState(m_rows + n_in)
  pruning.reset_default_registry()
  _cabi.lib().rigl_set_force_simt(1 if force_simt else 0)
  try:
    layer = SparseLinear(n_in, n_out, use_bias=use_bias, name='fc', device=DEV, out_dtype=out_dtype)
    w_np = _bf16(rng.standard_normal((n_in, n_out)) / np.sqrt(n_in)).float().numpy()
    if mask is None:
      m_np = orc.get_mask_random_numpy((n_in, n_out), sparsity, rng).astype(np.float32)
    else:
      m_np = tile_mask(mask, (n_in, n_out), rng, sparsity)
    b_np = rng.standard_normal(n_out).astype(np.float32) if use_bias else None
    with torch.no_grad():
      layer.weight.copy_(torch.from_numpy(w_np))
      if use_bias:
        layer.bias.copy_(torch.from_numpy(b_np))
    layer.mask.assign(m_np)
    x_np = _bf16(rng.standard_normal((m_rows, n_in))).float().numpy()
    x = torch.from_numpy(x_np).to(DEV).to(torch.bfloat16).requires_grad_(True)
    y = layer(x)
    assert y.dtype == out_dtype
    y_want = orc.masked_linear_fwd(x_np, w_np, m_np, b_np)
    (_check_f32 if out_dtype == torch.float32 else _check_bf16)(y, y_want, 'linear fprop %s' % (case,))
    dy_np = _bf16(rng.standard_normal(y_want.shape)).float().numpy()
    y.backward(torch.from_numpy(dy_np).to(DEV).to(out_dtype))
    dx_want, dw_dense, dw_masked = orc.masked_linear_bwd(x_np, w_np, m_np, dy_np)
    _check_bf16(x.grad, dx_want, 'linear dgrad %s' % (case,))
    _check_f32(layer.masked_weights.dense_grad.view(n_in, n_out), dw_dense, 'linear dense wgrad %s' % (case,))
    _check_f32(layer.weight.grad, dw_masked, 'linear masked wgrad %s' % (case,))
    if use_bias:
      _check_f32(layer.bias.grad, dy_np.astype(np.float64).sum(0), 'bias grad')
  finally:
    _cabi.lib().rigl_set_force_simt(0)


@pytest.mark.parametrize('case', LINEAR_CASES)
@pytest.mark.parametrize('force_simt', [True, False])
def test_linear(case, force_simt):
  _linear_case(case, force_simt)


@pytest.mark.parametrize('case', [c for c in LINEAR_CASES if c[2] in (1000, 200, 72)])
@pytest.mark.parametrize('use_bias', [False, True])
def test_linear_bf16_output(case, use_bias):
  """The default bf16 output: without a bias through the TMA-store epilogue (ragged last N tiles of 1000, 200 and
  72 units), with one through the per-thread bf16 stores."""
  _linear_case(case, False, 'bf16', use_bias)


def test_rank_and_channel_errors():
  pruning.reset_default_registry()
  layer = SparseConv2d(8, 8, 3, name='e', device=DEV)
  with pytest.raises(ValueError):
    layer(torch.zeros(2, 8, 4, device=DEV))
  with pytest.raises(ValueError):
    layer(torch.zeros(2, 4, 4, 4, device=DEV))


@pytest.mark.parametrize('case', [(2, 16, 16, 3, 64, 7, 2, 0.14), (3, 32, 32, 3, 64, 7, 2, 0.14),
                                  (2, 64, 48, 3, 16, 7, 2, 0.5), (2, 224, 224, 3, 64, 7, 2, 0.14)])
def test_conv_stem_s2d_path(case):
  """The space-to-depth stem (layers.STEM_S2D_PATH, the default): same oracle, same tolerances."""
  from rigl_b200 import layers
  old, layers.STEM_S2D_PATH = layers.STEM_S2D_PATH, True
  try:
    _conv_case(case, force_simt=False)
  finally:
    layers.STEM_S2D_PATH = old


@pytest.mark.parametrize('case', [(3, 32, 32, 3, 64, 7, 2, 0.14), (2, 64, 48, 3, 16, 7, 2, 0.5)])
def test_conv_stem_patch_matrix_path(case):
  """RIGL_STEM_S2D=0 fallback: the im2col patch-matrix stem."""
  from rigl_b200 import layers
  old, layers.STEM_S2D_PATH = layers.STEM_S2D_PATH, False
  try:
    _conv_case(case, force_simt=False)
  finally:
    layers.STEM_S2D_PATH = old


_KMAJOR = r'k_igemm_kmajor<'


def _isolated(calls, env, timeout=300):
  """run_isolated over this module's case functions."""
  return run_isolated('test_conv_gpu', calls, env, timeout)


# 3x3 / stride 1 / pad 1 layers with <= 64 reduction channels run on the halo kernels (one halo tile in
# shared memory feeds all nine taps): full and partial channel blocks, H not a multiple of the strip,
# H smaller than a strip, several N tiles, every halo pitch (8 / 16 / 32 / 64 / 128).  At pitch 128 (W = 96..126) the
# shared memory only fits one-row strips with two halo tiles in flight.
HALO_CASES = [
    (2, 14, 14, 64, 64, 3, 1, 0.6),
    (3, 56, 56, 64, 64, 3, 1, 0.64),
    (2, 28, 28, 32, 128, 3, 1, 0.8),
    (2, 13, 27, 64, 24, 3, 1, 0.5),
    (5, 6, 14, 16, 64, 3, 1, 0.3),
    (2, 28, 28, 64, 64, 3, 1, 0.9, 'SAME'),
    (2, 37, 6, 64, 64, 3, 1, 0.5),          # pitch 8
    (1, 45, 112, 32, 64, 3, 1, 0.6),        # pitch 128
]


@pytest.mark.parametrize('case', HALO_CASES)
def test_conv_halo_path(case):
  _conv_case(case, force_simt=False)


def test_conv_halo_pitches_run_the_halo_kernels():
  """The pitch-8 and pitch-128 cases really run on the halo kernels (fprop, dgrad and wgrad)."""
  for case, ran in zip(HALO_CASES[-2:], _isolated([('_conv_case', (c, False)) for c in HALO_CASES[-2:]], {})):
    assert_ran(ran, r'k_halo3x3_kmajor', case)
    assert_ran(ran, r'k_halo3x3_wgrad', case)
    assert_not_ran(ran, _KMAJOR, case)


@pytest.mark.parametrize('case', [HALO_CASES[1], HALO_CASES[3]])
def test_conv_halo_disabled_matches(case):
  """RIGL_HALO3X3=0 routes the same layers through the generic per-tap kernels."""
  ran, = _isolated([('_conv_case', (case, False))], {'RIGL_HALO3X3': '0'})
  assert_ran(ran, _KMAJOR, case)
  assert_not_ran(ran, r'k_halo3x3', case)


# ---- BASELINE-size problems (C2: ResNet-50, batch 256, 224x224): many more tiles than CTAs, so the persistent
# tile loops, smem-ring wrap and split-K schedules run for many tiles per CTA.
def _r50_erk80_sparsity():
  layers = orc.resnet50_masked_layers()
  sp = orc.get_sparsities([orc.FakeMask(n + '/mask:0', sh) for n, sh, _, _ in layers], 'erdos_renyi_kernel', 0.8, {})
  return layers, sp


def _r50_b256_shapes():
  """Distinct (n,h,w,cin,cout,k,stride,sparsity) of the 53 ResNet-50 convs at batch 256."""
  layers, sp = _r50_erk80_sparsity()
  seen, out = set(), []
  for name, sh, stride, out_hw in layers:
    if len(sh) != 4:
      continue
    k, _, cin, cout = sh
    key = (out_hw * stride, cin, cout, k, stride)
    if key in seen:
      continue
    seen.add(key)
    out.append((256, out_hw * stride, out_hw * stride, cin, cout, k, stride, round(float(sp[name + '/mask:0']), 3)))
  return out


# the four shapes VERDICT r1 asked for: 56^2 64->256 1x1, 56^2->28^2 128 3x3 s2, 14^2 256 3x3, 7^2 512 3x3
_B256_ORACLE = [c for c in _r50_b256_shapes() if (c[1], c[3], c[4], c[5], c[6]) in
                ((56, 64, 256, 1, 1), (56, 128, 128, 3, 2), (14, 256, 256, 3, 1), (7, 512, 512, 3, 1))]


@pytest.mark.parametrize('case', _B256_ORACLE, ids=lambda c: 'h%d_c%d_%d_k%d_s%d' % (c[1], c[3], c[4], c[5], c[6]))
def test_conv_b256_baseline_shapes_vs_fp64_oracle(case):
  assert len(_B256_ORACLE) == 4
  _conv_case(case, force_simt=False)


def _run_both(layer, x, dy, force_simt):
  _cabi.lib().rigl_set_force_simt(1 if force_simt else 0)
  try:
    xx = x.detach().clone().requires_grad_(True)
    layer.masked_weights.fresh = False
    layer.weight.grad = None
    y = layer(xx)
    y.backward(dy)
    torch.cuda.synchronize()
    return y.detach().float(), xx.grad.detach().float() if xx.grad is not None else None, \
        layer.masked_weights.dense_grad.clone()
  finally:
    _cabi.lib().rigl_set_force_simt(0)


@pytest.mark.parametrize('case', _r50_b256_shapes(), ids=lambda c: 'h%d_c%d_%d_k%d_s%d' % (c[1], c[3], c[4], c[5], c[6]))
def test_conv_b256_every_r50_shape_tensor_core_vs_cuda_core(case):
  """Every distinct ResNet-50 conv shape at batch 256: the tensor-core kernels against the shape-agnostic CUDA-core
  kernels on the SAME device inputs and packed operands (fp32 accumulation on both sides; bf16 outputs may differ
  by one rounding)."""
  n, h, w, cin, cout, k, stride, sparsity = case
  rng = np.random.RandomState(cin * 7 + cout + k)
  pruning.reset_default_registry()
  layer = SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', name='t', device=DEV)
  layer.mask.assign(orc.get_mask_random_numpy((k, k, cin, cout), sparsity, rng).astype(np.float32))
  g = torch.Generator(device=DEV).manual_seed(cin + cout)
  x = torch.randn((n, cin, h, w), device=DEV, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  ho = layer.out_size(h)[0]
  dy = torch.randn((n, cout, ho, ho), device=DEV, generator=g).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  y1, dx1, dw1 = _run_both(layer, x, dy, force_simt=False)
  y0, dx0, dw0 = _run_both(layer, x, dy, force_simt=True)
  for got, want, what in ((y1, y0, 'fprop'), (dx1, dx0, 'dgrad')):
    scale = float(want.abs().max())
    bad = (got - want).abs() > want.abs() * 2.0 ** -7 + scale * 2e-5
    assert not bool(bad.any()), '%s %s: %d elements off, max err %g (scale %g)' % (
        what, case, int(bad.sum()), float((got - want).abs().max()), scale)
  scale = float(dw0.abs().max())
  assert float((dw1 - dw0).abs().max()) <= 5e-5 * scale, 'wgrad %s: %g vs scale %g' % (
      case, float((dw1 - dw0).abs().max()), scale)


def test_batched_pack_equals_per_layer_pack():
  """layers.pack_all (ONE launch over a tile table) writes byte-identical operand blobs -- both K-major layouts and
  the 64x64 survivor counts -- to the per-layer rigl_pack_masked_weights calls, incl. ragged channel counts, the
  stem's patch-matrix form and a linear layer."""
  from rigl_b200 import layers
  pruning.reset_default_registry()
  rng = np.random.RandomState(5)
  ls = [SparseConv2d(3, 64, 7, strides=2, padding='FIXED', name='stem', device=DEV),
        SparseConv2d(64, 256, 1, name='a', device=DEV), SparseConv2d(72, 40, 3, name='ragged', device=DEV),
        SparseConv2d(128, 128, 3, strides=2, name='b', device=DEV), SparseLinear(300, 100, name='fc', device=DEV),
        SparseConv2d(5, 3, 3, name='tiny', device=DEV)]
  for l in ls:
    l.mask.assign(orc.get_mask_random_numpy(tuple(l.weight.shape), 0.8, rng).astype(np.float32))
  blobs = lambda l: [b for b in (getattr(l, 'packed_patch', None), l.packed, getattr(l, 'packed_s2d', None)) if b is not None]
  want = []
  for l in ls:
    for b in blobs(l):
      b.fill_(0x5a)          # (alignment padding between the blob's sections is never written: same filler twice)
    l.pack()
    want.append([b.clone() for b in blobs(l)])
  for l in ls:
    for b in blobs(l):
      b.fill_(0x5a)
  layers.pack_all(ls)
  torch.cuda.synchronize()
  for l, ws in zip(ls, want):
    got = blobs(l)
    if getattr(l, 'patch_mode', False):       # patch-mode layers only pack their patch / special forms
      got, ws = [got[0]] + got[2:], [ws[0]] + ws[2:]
    for g, w in zip(got, ws):
      assert torch.equal(g, w), l.scope
  layers._PACKED_AHEAD.clear()


def test_conv_wgrad_accumulates_over_backward_passes():
  """beta = 1: a second backward before the gradients are consumed ADDS to the dense gradient (k_splitk_reduce
  reads dw back and adds the split-K partials to it in split order)."""
  pruning.reset_default_registry()
  torch.manual_seed(3)
  layer = SparseConv2d(128, 256, 3, padding='FIXED', name='acc', device=DEV)
  x = torch.randn(8, 128, 14, 14, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  dy = torch.randn(8, 256, 14, 14, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  layer.masked_weights.fresh = False
  layer(x).backward(dy)
  once = layer.masked_weights.dense_grad.clone()
  layer(x).backward(dy)                       # fresh is still True: accumulates
  assert torch.allclose(layer.masked_weights.dense_grad, once + once, rtol=1e-5, atol=1e-5 * float(once.abs().max()))


@pytest.mark.parametrize('case', [(2, 16, 16, 32, 1), (2, 17, 13, 64, 2), (3, 14, 14, 256, 1), (2, 8, 8, 1024, 2),
                                  (4, 112, 112, 32, 1), (2, 56, 56, 128, 2), (1, 5, 7, 24, 1)])
def test_depthwise3x3_vs_fp64(case):
  """Native depthwise 3x3 (csrc/depthwise.cu; MobileNet-v1's depthwise_conv2d_fixed_padding, mobilenetv1_model.py:
  120-153) forward, input gradient and weight gradient against a float64 grouped convolution on the same
  bf16-rounded operands."""
  from rigl_b200.workloads import DepthwiseConv2d
  n, h, w, c, stride = case
  torch.manual_seed(c + h)
  dw = DepthwiseConv2d(c, stride=stride, device=DEV)
  dw.native = True                       # the csrc/depthwise.cu kernels (the default path is cuDNN)
  with torch.no_grad():
    dw.weight.copy_(dw.weight.to(torch.bfloat16).float() * 3)
    dw.weight.copy_(dw.weight.to(torch.bfloat16).float())
  x = torch.randn(n, c, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
  y = dw(x)
  x64 = x.detach().double().cpu().requires_grad_(True)
  w64 = dw.weight.detach().double().cpu().requires_grad_(True)
  y64 = torch.nn.functional.conv2d(x64, w64, None, stride, 1, 1, c)
  assert tuple(y.shape) == tuple(y64.shape)
  dy = torch.randn_like(y64).to(torch.bfloat16)
  y.backward(dy.to(DEV).contiguous(memory_format=torch.channels_last))
  y64.backward(dy.double())
  _check_bf16(y.permute(0, 2, 3, 1), y64.detach().permute(0, 2, 3, 1).numpy(), 'depthwise fprop %s' % (case,))
  _check_bf16(x.grad.permute(0, 2, 3, 1), x64.grad.permute(0, 2, 3, 1).numpy(), 'depthwise dgrad %s' % (case,))
  _check_f32(dw.weight.grad, w64.grad.numpy(), 'depthwise wgrad %s' % (case,))


# ---- dead weight tiles (tile_masks.py): the survivor-table lookups that let the K-major kernels skip the load and
# the MMA of an all-zero 64x64 weight tile.  Run in a child process with a time limit, because a producer and
# consumers that disagree on which K blocks are live would wait on each other forever.
@pytest.mark.parametrize('env', [{}], ids=['default'])
def test_conv_dead_weight_tiles(env):
  ran = _isolated([('_conv_case', (case, False, pattern)) for case, pattern in STRUCTURED_CONV_CASES], env, 600)
  for (case, pattern), names in zip(STRUCTURED_CONV_CASES, ran):
    if case[3] <= 64 and case[6] == 1:      # the halo case: its kernels keep all nine taps' weights resident
      assert_ran(names, r'k_halo3x3_kmajor', (case, pattern))
    else:
      assert_ran(names, _KMAJOR, (case, pattern))


@pytest.mark.parametrize('env', [{}], ids=['default'])
def test_linear_dead_weight_tiles_at_the_liveness_cap(env):
  """K = 320 blocks (dead blocks skipped) and 321 blocks (every block loaded) in fprop and in dgrad."""
  calls = [('_linear_case', (case, False, 'f32', True, pattern)) for case, pattern in STRUCTURED_LINEAR_CASES]
  for (case, pattern), names in zip(STRUCTURED_LINEAR_CASES, _isolated(calls, env, 600)):
    assert_ran(names, _KMAJOR, (case, pattern))


def _packed_layout(taps, cin, cout):
  """Mirror of packed_layout() in rigl_b200/csrc/conv_common.cuh: (off_fprop, off_dgrad, off_nnz, total, cin_pad,
  cout_pad, n_tiles, k_tiles) of the packed operand blob."""
  up = lambda v: (v + 255) // 256 * 256
  cin_pad, cout_pad = (cin + 7) // 8 * 8, (cout + 7) // 8 * 8
  n_tiles, k_tiles = (cout + 63) // 64, (cin + 63) // 64
  off_dgrad = up(taps * cout * cin_pad * 2)
  off_nnz = off_dgrad + up(taps * cin * cout_pad * 2)
  return 0, off_dgrad, off_nnz, off_nnz + up(taps * n_tiles * k_tiles * 4), cin_pad, cout_pad, n_tiles, k_tiles


def _bf16_bits(a):
  return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).view(torch.int16).numpy()


_PACK_LAYERS = [((64, 256, 1), None), ((128, 128, 3), None), ((72, 200, 3), None), ((300, 100, None), None)] + \
    [((c[3], c[4], c[5]), p) for c, p in STRUCTURED_CONV_CASES]


@pytest.mark.parametrize('spec,pattern', _PACK_LAYERS)
def test_pack_matches_numpy_reference(spec, pattern):
  """rigl_pack_masked_weights against numpy: the survivor count of every 64x64 tile, both bf16 K-major operands
  (mask * W, exactly) and zeros in the channel padding of each."""
  cin, cout, k = spec
  rng = np.random.RandomState(cin + cout)
  pruning.reset_default_registry()
  shape = (cin, cout) if k is None else (k, k, cin, cout)
  layer = SparseLinear(cin, cout, name='fc', device=DEV) if k is None else \
      SparseConv2d(cin, cout, k, padding='FIXED', name='c', device=DEV)
  w_np = _bf16(rng.standard_normal(shape)).float().numpy()
  m_np = orc.get_mask_random_numpy(shape, 0.7, rng).astype(np.float32) if pattern is None else \
      tile_mask(pattern, shape, rng)
  with torch.no_grad():
    layer.weight.copy_(torch.from_numpy(w_np))
  layer.mask.assign(m_np)
  layer.packed.fill_(0x5a)                    # padding that is never written would show up as 0x5a5a
  layer.pack()
  blob = layer.packed.cpu().numpy()
  taps = 1 if k is None else k * k
  off_f, off_d, off_n, total, cin_pad, cout_pad, n_tiles, k_tiles = _packed_layout(taps, cin, cout)
  assert blob.size == total
  wm = np.where(m_np != 0, w_np, 0).reshape(taps, cin, cout)          # (no -0.0 from masked negative weights)
  want_f = np.zeros((taps, cout, cin_pad), np.int16)
  want_f[:, :, :cin] = _bf16_bits(wm.transpose(0, 2, 1))
  got_f = blob[off_f:off_f + taps * cout * cin_pad * 2].view(np.int16).reshape(taps, cout, cin_pad)
  assert np.array_equal(got_f, want_f), 'fprop operand [tap][cout][cin_pad]'
  want_d = np.zeros((taps, cin, cout_pad), np.int16)
  want_d[:, :, :cout] = _bf16_bits(wm)
  got_d = blob[off_d:off_d + taps * cin * cout_pad * 2].view(np.int16).reshape(taps, cin, cout_pad)
  assert np.array_equal(got_d, want_d), 'dgrad operand [tap][cin][cout_pad]'
  got_n = blob[off_n:off_n + taps * n_tiles * k_tiles * 4].view(np.uint32).reshape(taps, n_tiles, k_tiles)
  assert np.array_equal(got_n, tile_counts(m_np)), 'survivor counts [tap][cout tile][cin tile]'
