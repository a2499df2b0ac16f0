"""The streaming kernels between the masked convs -- batch norm (csrc/bn.cu), the batch-norm statistics epilogue of
the conv (csrc/igemm_tc.cu) and the 3x3/2 max pool (csrc/pool.cu) -- against float64 at the sizes ResNet-50 and
MobileNet-v1 run them at batch 256, 224 x 224, where they switch code paths.

The float64 reference runs on the device in row chunks of CHUNK_ELEMS elements, so no float64 copy of a whole
activation (up to 411 MB in bf16) is ever made.

Statistics bound.  The kernels sum bf16 values exactly converted to fp32: sequentially per thread over at most
~130 rows (3.2 M rows / 792 CTAs / 32 row-threads on the three-kernel path; fewer on the others), then over the
rpi row-threads of a block (or ~50 slab atomics per CTA in the conv epilogue) in fp32, then across CTAs in fp64.
The worst-case error of such a sum is (130 + rpi + 2) * 2^-24 of the sum of the magnitudes it adds.  rpi = 512 /
(C / 8) on the 512-thread grid-barrier kernels (the larger of the two paths), at most 64 for C >= 64, which gives
STAT_TOL = 2^-16 (1.5e-5 > 196 * 2^-24); the narrow edge cases (C = 8: rpi = 512, C = 24: rpi = 170) get the
larger bound of _stat_tol.  The tolerance applies to sum |y| (mean), sum y^2 (variance), sum |g| (dbeta) and
sum |g * xhat| (dgamma).  Each check is paired with a control: the same check against a reference that leaves
out one CTA's share of the rows (a lost or double-counted partial) must fail.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from isolated import assert_not_ran, run_isolated

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
EPS, MOMENTUM = 1e-5, 0.1
STAT_TOL = 2.0 ** -16
CHUNK_ELEMS = 1 << 25                 # elements per float64 chunk: 256 MB per temporary
FUSED_MAX_BYTES = 64 << 20            # bn.cu: tensors up to this size take the grid-barrier kernels
THREE_KERNEL_CTAS = 132 * 6           # bn.cu colsum_blocks: ~6 CTAs per SM of the column-sum pass


def _lib():
  from rigl_b200 import _cabi
  return _cabi


def _chunks(rows, c):
  step = max(1, CHUNK_ELEMS // c)
  return [(a, min(a + step, rows)) for a in range(0, rows, step)]


def _bf16_tol(want, cancelled=None):
  """Per-element bound of _close_bf16 for the float64 values `want`."""
  scale = float(want.abs().max()) + 1e-30
  tol = want.abs() * 2.0 ** -7 + scale * 2.0 ** -9
  if cancelled is not None:
    tol = tol + cancelled * 2.0 ** -22
  return tol


def _close_bf16(got, want, what, cancelled=None):
  """bf16 result within 1 bf16 ulp (2^-7 relative) of the float64 value, plus 2^-9 of the chunk's largest
  magnitude for cancellation (the bound of test_bn_gpu._close_bf16, on device tensors).  `cancelled`: the summed
  magnitude of the fp32 terms the kernel adds to form each element; 2^-22 of it is added (fp32 rounding of those
  terms, which matters where they cancel to a result near zero)."""
  got = got.double()
  scale = float(want.abs().max()) + 1e-30
  tol = _bf16_tol(want, cancelled)
  err = (got - want).abs()
  bad = int((err > tol).sum())
  assert bad == 0, '%s: max err %g at scale %g (%d bad)' % (what, float(err.max()), scale, bad)


def _within(got, want, tol):
  """Per-channel |got - want| <= tol (all float64 device tensors)."""
  return bool(((got.double() - want).abs() <= tol).all())


# ---------------------------------------------------------------------------------------------------------------
# Batch norm through the C entry points (rigl_bn_forward_train / rigl_bn_backward), so the saved mean / rstd can
# be read.  Forms: 'relu' (stem, conv1, conv2: BN+ReLU), 'plain' (projection: no ReLU), 'residual2' (conv3:
# relu(BN + shortcut) whose output is forked, two incoming gradients), 'residual1' (the last block: one gradient).
# ---------------------------------------------------------------------------------------------------------------

def _fill(rows, c, mean, sd, gen):
  """bf16 [rows, c] = mean + sd * N(0, 1), generated in chunks (no full-size fp32 temporary)."""
  t = torch.empty((rows, c), dtype=torch.bfloat16, device=DEV)
  for a, b in _chunks(rows, c):
    t[a:b] = (torch.randn((b - a, c), generator=gen, device=DEV) * sd + mean).to(torch.bfloat16)
  return t


def _channel_spread(c, lo, hi, gen):
  """Clearly nonzero per-channel values in +-[lo, hi], in a shuffled order."""
  mag = torch.linspace(lo, hi, c, device=DEV)
  sign = torch.where(torch.arange(c, device=DEV) % 2 == 0, 1.0, -1.0)
  return (mag * sign)[torch.randperm(c, generator=gen, device=DEV)]


def _predict_fused(rows, c, enabled=None):
  """(forward, backward) take the grid-barrier kernels: bn.cu fused_plan.  RIGL_BN_FUSED=0 disables them."""
  if enabled is None:
    enabled = os.environ.get('RIGL_BN_FUSED', '1')[:1] != '0'
  small = enabled and c <= 4096 and rows * c * 2 <= FUSED_MAX_BYTES
  return small and c >= 512, small


def _stat_sums(t, rows, c, drop=0):
  """float64 statistics of t [rows, c]: (mean, variance, E|t|, E[t^2]).  drop > 0 leaves rows [0, drop) out of the
  sums but still divides by `rows`: the statistics a kernel would produce if it lost one CTA's partial sums."""
  s = torch.zeros(c, dtype=torch.float64, device=DEV)
  a = torch.zeros_like(s)
  for lo, hi in _chunks(rows, c):
    x = t[max(lo, drop):hi].double()
    s += x.sum(0)
    a += x.abs().sum(0)
  m = rows
  mean = s / m
  d = torch.zeros_like(s)
  q = torch.zeros_like(s)
  for lo, hi in _chunks(rows, c):
    x = t[max(lo, drop):hi].double()
    d += ((x - mean) ** 2).sum(0)
    q += (x * x).sum(0)
  return mean, d / m, a / m, q / m


def _stat_tol(c):
  """Relative bound of the batch-norm column sums at C channels (module docstring)."""
  rpi = 512 // min(c // 8, 512)
  return max(STAT_TOL, (130 + rpi + 2) * 2.0 ** -24)


def _stats_ok(mean_got, rstd_got, ref, tol=STAT_TOL):
  """Saved mean / rstd against the float64 statistics `ref` = (mean, var, E|y|, E[y^2]) to `tol` of the summed
  magnitudes.  rstd = 1/sqrt(var + eps) with var = E[y^2] - mean^2: its relative error is half that of var + eps."""
  mean, var, abs_mean, sq_mean = ref
  rstd = 1.0 / torch.sqrt(var + EPS)
  tol_var = tol * 2 * sq_mean
  rstd_tol = (0.5 * tol_var / (var + EPS) + 2.0 ** -23) * rstd
  return _within(mean_got, mean, tol * abs_mean + 1e-30) and _within(rstd_got, rstd, rstd_tol)


def _bn_case(rows, c, form, special=False, seed=0):
  """Forward and backward of one BN against float64; returns nothing, asserts.

  It first checks that each direction took the path fused_plan's size rules predict (grid-barrier kernels up to
  64 MB, the forward only for C >= 512; RIGL_BN_FUSED=0 disables them), so a moved threshold cannot silently drop a
  path from the coverage.  The witness is the library's own launch counter (rigl_launch_count): a grid-barrier
  direction is one launch, the three-kernel path three (column sums, finalize, apply).  torch.profiler was tried
  for this and lost kernel records now and then, whole windows included, both in the test process and in fresh
  ones."""
  cabi = _lib()
  lib = cabi.lib()
  gen = torch.Generator(device=DEV)
  gen.manual_seed(seed * 7919 + rows * 3 + c)
  relu = form != 'plain'
  residual = form.startswith('residual')
  mu = _channel_spread(c, 0.5, 3.0, gen)
  sd = torch.linspace(0.6, 1.8, c, device=DEV)
  if special and c >= 16:
    mu[0], sd[0] = 1.5, 0.0                # a constant channel: variance 0
    mu[1], sd[1] = 64.0 * 0.25, 0.25       # |mean| / std = 64
  y = _fill(rows, c, mu, sd, gen)
  r = _fill(rows, c, 0.2, 1.0, gen) if residual else None
  gmu = _channel_spread(c, 0.2, 0.8, gen)
  da = _fill(rows, c, gmu, 1.0, gen)
  db = _fill(rows, c, -0.3 * gmu, 0.7, gen) if form == 'residual2' else None
  gamma = torch.linspace(0.5, 1.5, c, device=DEV)[torch.randperm(c, generator=gen, device=DEV)].contiguous()
  beta = torch.linspace(-0.4, 0.4, c, device=DEV)
  rm0 = torch.linspace(-0.3, 0.3, c, device=DEV)
  rv0 = torch.linspace(0.8, 1.2, c, device=DEV)
  rm, rv = rm0.clone(), rv0.clone()
  save = torch.empty((4, c), dtype=torch.float32, device=DEV)
  out = torch.empty_like(y)
  bits = torch.empty(rows * c // 8, dtype=torch.uint8, device=DEV) if residual else None
  ws = torch.empty(lib.rigl_bn_workspace_bytes(rows, c) + 8 * c + 256, dtype=torch.uint8, device=DEV)
  p = lambda t: None if t is None else t.data_ptr()

  def fwd():
    cabi.check(lib.rigl_bn_forward_train(
        y.data_ptr(), p(r), gamma.data_ptr(), beta.data_ptr(), rows, c, EPS, MOMENTUM, int(relu), rm.data_ptr(),
        rv.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(),
        out.data_ptr(), ws.data_ptr(), ws.numel(), p(bits), cabi.stream_ptr()), 'rigl_bn_forward_train')

  dy = torch.empty_like(y)
  dres = torch.empty_like(y) if residual else None
  dgb = torch.empty((2, c), dtype=torch.float32, device=DEV)

  def bwd():
    cabi.check(lib.rigl_bn_backward(
        da.data_ptr(), p(db), y.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(),
        save[3].data_ptr(), rows, c, int(relu), dy.data_ptr(), p(dres), dgb[0].data_ptr(), dgb[1].data_ptr(),
        ws.data_ptr(), ws.numel(), p(bits), cabi.stream_ptr()), 'rigl_bn_backward')

  fused_fwd, fused_bwd = _predict_fused(rows, c)
  n0 = cabi.launch_count()
  fwd()
  n1 = cabi.launch_count()
  bwd()
  n2 = cabi.launch_count()
  torch.cuda.synchronize()
  assert n1 - n0 == (1 if fused_fwd else 3), 'forward: %d launches, expected the %s path' % (
      n1 - n0, 'grid-barrier' if fused_fwd else 'three-kernel')
  assert n2 - n1 == (1 if fused_bwd else 3), 'backward: %d launches, expected the %s path' % (
      n2 - n1, 'grid-barrier' if fused_bwd else 'three-kernel')
  tol = _stat_tol(c)

  # ---- forward statistics and running statistics
  ref = _stat_sums(y, rows, c)
  mean, var = ref[0], ref[1]
  assert _stats_ok(save[0], save[1], ref, tol), 'saved mean / rstd'
  drop = rows // THREE_KERNEL_CTAS            # less than one CTA's share of the rows on either path
  if drop > 0:
    assert not _stats_ok(save[0], save[1], _stat_sums(y, rows, c, drop), tol), 'statistics control: rows left out'
  if special and c >= 16:
    # constant channel: every sum is exact, so the variance is exactly 0
    assert float(save[1][0]) == pytest.approx(1.0 / np.sqrt(np.float64(np.float32(EPS))), rel=1e-6)
    # |mean| / std = 64: the worst-case bound above is ~6 % of rstd there (E[y^2] ~ 4097 var).  The values, multiples
    # of 2^-3 near 16, have squares of <= 15 significant bits, so at these sizes (< ~960 rows per CTA) the fp32 sums
    # are exact and only the fp64 finalize rounds (a CPU emulation of the summation order puts the error below 1e-4
    # even at batch-256 sizes).  A variance formed in fp32 from E[y^2] and mean^2 would be off by up to
    # 2^-24 * 4097 / 2 ~ 1.2e-4 of rstd on its own.
    assert abs(float(save[1][1]) / float(1.0 / torch.sqrt(var[1] + EPS)) - 1.0) <= 1e-4, 'rstd at |mean|/std = 64'
  unbiased = var * rows / (rows - 1) if rows > 1 else var
  rm_want = (1 - MOMENTUM) * rm0.double() + MOMENTUM * mean
  rv_want = (1 - MOMENTUM) * rv0.double() + MOMENTUM * unbiased
  assert _within(rm, rm_want, MOMENTUM * tol * ref[2] + 2.0 ** -22 * rm_want.abs()), 'running mean'
  assert _within(rv, rv_want, MOMENTUM * tol * 2 * ref[3] * max(1.0, rows / max(rows - 1, 1)) +
                 2.0 ** -22 * rv_want.abs()), 'running variance'
  if rows == 2:                # the unbiased factor M / (M - 1) = 2 is not hidden under the tolerance
    assert not _within(rv, (1 - MOMENTUM) * rv0.double() + MOMENTUM * var, 2.0 ** -20 * rv_want.abs() + 1e-12)

  # ---- forward output, against the float64 statistics
  rstd = 1.0 / torch.sqrt(var + EPS)
  g64, b64 = gamma.double(), beta.double()
  for lo, hi in _chunks(rows, c):
    z = (y[lo:hi].double() - mean) * rstd * g64 + b64
    if residual:
      z = z + r[lo:hi].double()
    _close_bf16(out[lo:hi], z.clamp_min(0) if relu else z, 'forward rows %d:%d' % (lo, hi))
  if residual:
    assert torch.equal(bits, _pack_sign(out)), 'ReLU bitmap'

  # ---- backward, with the saved (fp32) mean / rstd as the kernel used them
  m_k, r_k = save[0].double(), save[1].double()

  def grad_in(lo, hi):
    g = da[lo:hi]
    if db is not None:
      g = (g.float() + db[lo:hi].float()).to(torch.bfloat16)       # the gradient sum is rounded to bf16
    g = g.double()
    return g * (out[lo:hi] > 0) if relu else g

  def bwd_sums(drop=0):
    s0 = torch.zeros(c, dtype=torch.float64, device=DEV)
    s1, a0, a1 = torch.zeros_like(s0), torch.zeros_like(s0), torch.zeros_like(s0)
    for lo, hi in _chunks(rows, c):
      lo = max(lo, drop)
      g = grad_in(lo, hi)
      gx = g * ((y[lo:hi].double() - m_k) * r_k)
      s0 += g.sum(0); s1 += gx.sum(0); a0 += g.abs().sum(0); a1 += gx.abs().sum(0)
    return s0, s1, a0, a1

  def dgb_ok(sums):
    s0, s1, a0, a1 = sums
    return _within(dgb[1], s0, tol * a0 + 1e-30) and _within(dgb[0], s1, tol * a1 + 1e-30)

  sums = bwd_sums()
  assert dgb_ok(sums), 'dgamma / dbeta'
  if drop > 0:
    assert not dgb_ok(bwd_sums(drop)), 'dgamma / dbeta control: rows left out'
  dbeta, dgamma = sums[0], sums[1]
  for lo, hi in _chunks(rows, c):
    g = grad_in(lo, hi)
    xhat = (y[lo:hi].double() - m_k) * r_k
    # the kernel forms dy = scale*g + P*y + Q (bn.cu finalize_bwd_channel) in fp32
    sc = g64 * r_k
    terms = (sc * g).abs() + (sc * r_k * dgamma / rows * y[lo:hi].double()).abs() + \
        (sc * (r_k * m_k * dgamma / rows - dbeta / rows)).abs()
    _close_bf16(dy[lo:hi], sc * (g - dbeta / rows - xhat * dgamma / rows), 'dy rows %d:%d' % (lo, hi), terms)
    if residual:
      assert torch.equal(dres[lo:hi], g.to(torch.bfloat16)), 'dresidual rows %d:%d' % (lo, hi)


def _pack_sign(out):
  """Bit k of byte i = out.flat[8i + k] > 0 (the residual form's ReLU bitmap)."""
  b = (out.reshape(-1, 8) > 0).to(torch.uint8)
  w = torch.tensor([1, 2, 4, 8, 16, 32, 64, 128], dtype=torch.uint8, device=out.device)
  return (b * w).sum(1, dtype=torch.uint8)


# Every distinct batch-256 BN shape of ResNet-50 (r50) and MobileNet-v1 (mbv1, all BN+ReLU), with the forms each
# has in the model.
_B = 256
_BN_SHAPES = [
    ('r50-mbv1', 112, 64, ('relu',)), ('mbv1', 112, 32, ('relu',)),
    ('r50-mbv1', 56, 64, ('relu',)), ('r50-mbv1', 56, 128, ('relu',)), ('r50', 56, 256, ('plain', 'residual2')),
    ('r50-mbv1', 28, 128, ('relu',)), ('r50-mbv1', 28, 256, ('relu',)), ('r50', 28, 512, ('plain', 'residual2')),
    ('r50-mbv1', 14, 256, ('relu',)), ('r50-mbv1', 14, 512, ('relu',)), ('r50', 14, 1024, ('plain', 'residual2')),
    ('r50-mbv1', 7, 512, ('relu',)), ('mbv1', 7, 1024, ('relu',)),
    ('r50', 7, 2048, ('plain', 'residual2', 'residual1')),
]
_BN_CASES = [pytest.param(_B * hw * hw, c, form, id='%s-%dx%dx%d-%s' % (tag, hw, hw, c, form))
             for tag, hw, c, forms in _BN_SHAPES for form in forms]
# the shapes that take the grid-barrier kernels by default (<= 64 MB), as plain (rows, c, form) literals
_FUSED_CASES = [tuple(p.values) for p in _BN_CASES if _predict_fused(p.values[0], p.values[1], enabled=True)[1]]


@pytest.mark.parametrize('rows,c,form', _BN_CASES)
def test_bn_b256_against_float64(rows, c, form):
  _bn_case(rows, c, form)


def test_bn_b256_fused_shapes_on_the_three_kernel_path():
  """The shapes that take the grid-barrier kernels by default, once more on the three-kernel path."""
  assert len({(r, c) for r, c, _ in _FUSED_CASES}) == 6      # 5 ResNet-50 shapes + MobileNet-v1's 7x7x1024
  calls = [('_bn_case', (rows, c, form)) for rows, c, form in _FUSED_CASES]     # (each asserts its path)
  torch.cuda.empty_cache()                   # the child allocates the same sizes
  for case, ran in zip(_FUSED_CASES, run_isolated('test_streaming_b256_gpu', calls, {'RIGL_BN_FUSED': '0'},
                                                  timeout=600)):
    assert_not_ran(ran, r'k_bn_(fwd|bwd)_fused', case)


# rows, c: single rows, one vector per row (C = 8) and three (C = 24), the widest fused layers and beyond the
# fused limit (C = 2560 / 3072 / 4104: V = C / 8 is not a multiple of the 256 column-sum threads, so those threads
# own different numbers of vectors), exactly 64 MiB and one row more, and a last CTA with a single row on each
# path (C = 64: 791 full CTAs of 32 rows; C = 2048: 2-row CTAs on a 132- or 264-CTA grid).
_EDGE_CASES = [(1, 64), (2, 64), (1, 2048), (2, 24), (1000, 8), (777, 24), (300, 2048), (96, 2560), (64, 3072),
               (50, 4096), (40, 4104), (65536, 512), (65537, 512), (791 * 32 + 1, 64), (263, 2048)]


_EDGE_FORMS = ('relu', 'residual2')


@pytest.mark.parametrize('rows,c', _EDGE_CASES)
@pytest.mark.parametrize('form', _EDGE_FORMS)
def test_bn_edge_shapes_against_float64(rows, c, form):
  _bn_case(rows, c, form, special=True)


def test_bn_edge_shapes_on_the_three_kernel_path():
  calls = [('_bn_case', (rows, c, form, True)) for rows, c in _EDGE_CASES for form in ('relu', 'residual2')]
  torch.cuda.empty_cache()
  for (fn, args), ran in zip(calls, run_isolated('test_streaming_b256_gpu', calls, {'RIGL_BN_FUSED': '0'})):
    assert_not_ran(ran, r'k_bn_(fwd|bwd)_fused', args)      # (each call asserts its path by launch count)


# ---------------------------------------------------------------------------------------------------------------
# Batch-norm statistics from the conv epilogue (rigl_masked_conv2d_fprop_bnstats), default policy, against the
# float64 statistics of the conv's own bf16 output.
# ---------------------------------------------------------------------------------------------------------------

# every distinct batch-256 ResNet-50 conv shape that has a statistics epilogue candidate: (cin, cout, k, stride, hw)
_CONV_SHAPES = [(256, 64, 1, 1, 56), (64, 256, 1, 1, 56), (64, 64, 1, 1, 56),
                (256, 512, 1, 2, 56), (256, 128, 1, 1, 56), (128, 128, 3, 2, 56), (128, 512, 1, 1, 28),
                (512, 128, 1, 1, 28), (128, 128, 3, 1, 28),
                (512, 1024, 1, 2, 28), (512, 256, 1, 1, 28), (256, 256, 3, 2, 28), (256, 1024, 1, 1, 14),
                (1024, 256, 1, 1, 14), (256, 256, 3, 1, 14),
                (1024, 2048, 1, 2, 14), (1024, 512, 1, 1, 14), (512, 512, 3, 2, 14), (512, 2048, 1, 1, 7),
                (2048, 512, 1, 1, 7), (512, 512, 3, 1, 7)]


def _conv_stats_case(cin, cout, k, stride, hw):
  from rigl_b200 import layers, pruning
  cabi = _lib()
  lib = cabi.lib()
  torch.manual_seed(cin * 7 + cout + k)
  pruning.reset_default_registry()
  conv = layers.SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', name='c', device=DEV)
  conv.mask.assign((torch.rand(k, k, cin, cout, device=DEV) < 0.3).float())
  conv.collect_bn_stats = True
  x = torch.empty((_B, cin, hw, hw), dtype=torch.bfloat16, device=DEV, memory_format=torch.channels_last)
  x.copy_((torch.rand((_B, cin, hw, hw), device=DEV) * 2.0 - 0.5).to(torch.bfloat16))   # mean 0.5: nonzero outputs
  old = layers.FUSE_BN_STATS
  layers.FUSE_BN_STATS = True
  try:
    yt = conv(x).detach()
  finally:
    layers.FUSE_BN_STATS = old
  del x
  if conv.bn_partial is None:
    pytest.skip('the default policy keeps the separate stats pass for this shape')
  part, nrows, ptr = conv.bn_partial
  assert ptr == yt.data_ptr() and 0 < nrows <= lib.rigl_bn_partial_rows()
  n, _, oh, ow = yt.shape
  rows = n * oh * ow
  y = yt.permute(0, 2, 3, 1).reshape(rows, cout)         # channels_last storage: a view
  save = torch.empty((4, cout), dtype=torch.float32, device=DEV)
  out = torch.empty_like(y)
  gamma, beta = torch.ones(cout, device=DEV), torch.zeros(cout, device=DEV)
  cabi.check(lib.rigl_bn_forward_train_partials(
      y.data_ptr(), None, gamma.data_ptr(), beta.data_ptr(), part.data_ptr(), nrows, rows, cout, EPS, MOMENTUM, 1,
      None, None, save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(), out.data_ptr(),
      None, cabi.stream_ptr()), 'rigl_bn_forward_train_partials')
  torch.cuda.synchronize()
  assert _stats_ok(save[0], save[1], _stat_sums(y, rows, cout)), 'statistics from the epilogue partials'
  assert not _stats_ok(save[0], save[1], _stat_sums(y, rows, cout, rows // nrows)), 'control: one CTA left out'


@pytest.mark.parametrize('cin,cout,k,stride,hw', _CONV_SHAPES,
                         ids=['%dx%dx%d-k%ds%d-%d' % (hw, hw, cin, k, s, cout) for cin, cout, k, s, hw in _CONV_SHAPES])
def test_conv_epilogue_bn_stats_b256_against_float64(cin, cout, k, stride, hw):
  _conv_stats_case(cin, cout, k, stride, hw)


# ---------------------------------------------------------------------------------------------------------------
# Max pool 3x3/2 'SAME'
# ---------------------------------------------------------------------------------------------------------------

def _pool_geom(h, w):
  oh, ow = (h + 1) // 2, (w + 1) // 2
  ph, pw = max((oh - 1) * 2 + 3 - h, 0), max((ow - 1) * 2 + 3 - w, 0)
  return oh, ow, ph // 2, pw // 2, ph - ph // 2, pw - pw // 2


def maxpool_reference(x, first=True):
  """float [N,C,H,W] -> (max, window-relative argmax [N,OH,OW,C] uint8) of TF 'SAME' 3x3/2 pooling, the argmax
  being the first maximum in (kh, kw) order (the last with first=False)."""
  n, c, h, w = x.shape
  oh, ow, pt, pl, pb, pr = _pool_geom(h, w)
  xp = F.pad(x, (pl, pr, pt, pb), value=float('-inf'))
  win = torch.stack([xp[:, :, kh:kh + 2 * oh - 1:2, kw:kw + 2 * ow - 1:2] for kh in range(3) for kw in range(3)])
  if not first:
    win = win.flip(0)
  arg = torch.argmax(win, dim=0)                # documented to return the first maximal index
  if not first:
    arg = 8 - arg
  return win.amax(0), arg.permute(0, 2, 3, 1).to(torch.uint8)


def maxpool_backward_reference(arg, dy, h, w, skip_slot=None):
  """dx of TF 'SAME' 3x3/2 pooling from the window-relative argmax [N,OH,OW,C] and dy [N,C,OH,OW] (float): each
  pixel adds the <= 4 contributions of the windows that chose it in fp32, windows in (oh, ow) ascending order, and
  rounds once to bf16.  skip_slot drops one of those four window positions (a sensitivity control)."""
  n, c, oh, ow = dy.shape
  _, _, pt, pl, _, _ = _pool_geom(h, w)
  hp, wp = 2 * oh + 1, 2 * ow + 1
  arg = arg.permute(0, 3, 1, 2)
  # slot (jh, jw): jh = 0 for the window above (kh = 2, the smaller oh), 1 for the window below or the only one
  slots = torch.zeros((2, 2, n, c, hp, wp), dtype=torch.float32, device=dy.device)
  for kh in range(3):
    for kw in range(3):
      jh, jw = (0 if kh == 2 else 1), (0 if kw == 2 else 1)
      if (jh, jw) == skip_slot:
        continue
      slots[jh, jw, :, :, kh:kh + 2 * oh - 1:2, kw:kw + 2 * ow - 1:2] = torch.where(arg == kh * 3 + kw, dy, 0.0)
  acc = torch.zeros((n, c, hp, wp), dtype=torch.float32, device=dy.device)
  for jh, jw in ((0, 0), (0, 1), (1, 0), (1, 1)):
    acc = acc + slots[jh, jw]
  return acc[:, :, pt:pt + h, pl:pl + w].to(torch.bfloat16)


@pytest.mark.parametrize('shape', [(256, 112, 112, 64), (32, 113, 111, 64)], ids=['256x112x112x64', '32x113x111x64'])
@pytest.mark.parametrize('sign', ['mixed', 'negative'])
def test_maxpool_b256_exact(shape, sign):
  """Forward bit-exact against F.max_pool2d on a -inf-padded input, the stored argmax = the first maximum in
  (kh, kw) order on inputs quantised to a few values (ties everywhere), and the backward bit-exact against the
  fp32 gather in the kernel's order.  The even extent takes the 2x2-quad backward kernel, the odd one (pad 1) the
  generic kernel (pool.cu: the quad kernel needs a 3x3/2 window, no leading pad and even extents)."""
  cabi = _lib()
  lib = cabi.lib()
  n, h, w, c = shape
  oh, ow = (h + 1) // 2, (w + 1) // 2
  gen = torch.Generator(device=DEV)
  gen.manual_seed(h * w)
  q = torch.randint(0, 4, (n, c, h, w), generator=gen, device=DEV, dtype=torch.int16).to(torch.bfloat16) * 0.5
  x = (q - 1.0 if sign == 'mixed' else -q - 0.25).contiguous(memory_format=torch.channels_last)   # exact in bf16
  del q
  y = torch.empty((n, c, oh, ow), dtype=torch.bfloat16, device=DEV, memory_format=torch.channels_last)
  arg = torch.empty((n, oh, ow, c), dtype=torch.uint8, device=DEV)
  cabi.check(lib.rigl_maxpool_same_forward(x.data_ptr(), n, h, w, c, 3, 2, y.data_ptr(), arg.data_ptr(),
                                           cabi.stream_ptr()), 'rigl_maxpool_same_forward')
  dy = torch.randn((n, c, oh, ow), generator=gen, device=DEV).to(torch.bfloat16)
  dy = dy.contiguous(memory_format=torch.channels_last)
  dx = torch.empty_like(x)
  cabi.check(lib.rigl_maxpool_same_backward(dy.data_ptr(), arg.data_ptr(), n, h, w, c, 3, 2, dx.data_ptr(),
                                            cabi.stream_ptr()), 'rigl_maxpool_same_backward')
  step = 32
  for a in range(0, n, step):
    b = min(a + step, n)
    xs = x[a:b].float()
    want, want_arg = maxpool_reference(xs)
    assert torch.equal(y[a:b].float(), want), 'forward'
    assert torch.equal(y[a:b].float(), F.max_pool2d(F.pad(xs, _pool_pads(h, w), value=float('-inf')), 3, 2))
    assert torch.equal(arg[a:b], want_arg), 'argmax'
    assert not torch.equal(arg[a:b], maxpool_reference(xs, first=False)[1]), 'control: ties to the last maximum'
    want_dx = maxpool_backward_reference(arg[a:b], dy[a:b].float(), h, w)
    assert torch.equal(dx[a:b], want_dx), 'backward'
    assert not torch.equal(dx[a:b], maxpool_backward_reference(arg[a:b], dy[a:b].float(), h, w, skip_slot=(0, 0))), \
        'control: one window contribution dropped'


def _pool_pads(h, w):
  _, _, pt, pl, pb, pr = _pool_geom(h, w)
  return (pl, pr, pt, pb)


# ---------------------------------------------------------------------------------------------------------------
# CUDA graph with the dense wgrad on a side stream, at batch 256 / 224^2
# ---------------------------------------------------------------------------------------------------------------

def test_cuda_graph_wgrad_side_stream_b256_matches_serial_backward():
  """At batch 256 the BN-backward chain's grid-barrier kernels run next to the wgrad kernels of the side stream.
  Every kernel is deterministic, so the replayed graph must reproduce the serial eager backward bit for bit: dense
  weight gradients, BN gradients and the running statistics one forward leaves behind."""
  from rigl_b200 import workloads
  torch.manual_seed(3)
  model = workloads.ResNet50(num_classes=1000, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=3)
  h = workloads.TrainHarness(model, lr=0.1)
  x = torch.randn(_B, 3, 224, 224, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  y = torch.randint(0, 1000, (_B,), device=DEV)
  bns = [m for m in model.modules() if m.__class__.__name__ == 'FusedBatchNormReLU']
  stats0 = [(b.running_mean.clone(), b.running_var.clone()) for b in bns]
  h._forward_backward(x, y, set_to_none=False)            # serial reference (no fork: _overlap is unset)
  torch.cuda.synchronize()
  layers_ = model.registry.layers()
  ref_dense = [l.masked_weights.dense_grad.clone() for l in layers_]
  ref_bn = [(b.weight.grad.clone(), b.bias.grad.clone(), b.running_mean.clone(), b.running_var.clone()) for b in bns]
  assert h.enable_cuda_graph(x, y, overlap_wgrad=True) and h._overlap
  try:
    for _ in range(2):
      for b, (m0, v0) in zip(bns, stats0):
        b.running_mean.copy_(m0)
        b.running_var.copy_(v0)
      h._g_fb.replay()
      torch.cuda.synchronize()
      for l, d in zip(layers_, ref_dense):
        assert torch.equal(l.masked_weights.dense_grad, d), l.scope
      for i, (b, ref) in enumerate(zip(bns, ref_bn)):
        for got, want, what in zip((b.weight.grad, b.bias.grad, b.running_mean, b.running_var), ref,
                                   ('dgamma', 'dbeta', 'running mean', 'running variance')):
          assert torch.equal(got, want), 'BN %d %s' % (i, what)
  finally:                    # the graph pool and the model hold ~12 GB: give them back
    h.release_cuda_graph()
    del h, model
    torch.cuda.empty_cache()
