"""VGG-16's training path against float64 at the size tools/bench_vgg.py runs it: batch 256, 224 x 224, ERK 0.8.

Covered: every distinct masked layer of VGG-16 with the flags the model gives it (the ReLU fprop epilogue, the dgrad
gated by the layer's forward input, the 3-channel first conv on the patch matrix, the halo ReLU fprop of conv2_1, and
the fp32 logits of fc8), the 2x2 ReLU pool and the standalone gate on the pooled shapes, and the whole step (fused
route against the standalone-gate route, CUDA-graph replay with the wgrad on a side stream against the serial eager
backward).  The (shape, gate) cases of VGG-A and VGG-19 are a subset of VGG-16's, so this covers all three models.
At this size the launchers take decisions nothing smaller reaches: the two 224^2 layers are the largest activations
of the project (822 M elements), conv1_2's dense wgrad adds 428 k pixels per split, and the patch matrix of conv1_1
has 12.8 M rows.

The float64 references run on the device per tap over chunks of whole images (test_bench_c4_c5_gpu._float64_layer);
no fp32 or float64 copy of a whole activation is made.  Bounds (u = 2^-24; |terms| = the same float64 computation on
|x|, |w * m| and |dy|), as in test_bench_c4_c5_gpu:
- ReLU fprop: |y - relu(y_ref)| <= the bf16 bound of the unrectified reference (_bf16_tol with |terms|).  ReLU is
  1-Lipschitz and the bf16 rounding keeps the sign, so relu of a value within the bound is within it too.  No output
  is negative (+-0 compare equal).
- Gated dgrad: where x > 0 is false (x = +0, -0 or negative) dx is exactly +-0; elsewhere the bf16 bound.  x > 0 is
  TF's `features > 0`, which passes subnormals: at least one subnormal x must let its gradient through.
- Ungated dgrad (a layer after a pool) and fc8's input gradient: the bf16 bound.
- fc8's fp32 logits: (K + 1) u |terms| with K = 512.
- Dense wgrad: (pps + splits) u |terms| (_wgrad_plan).  Each case also prints the plain max |err| / |terms|.
Every bound has a control that must fail by at least 1.2x: the centre tap (fc8: one input channel for the logits,
one output channel for dgrad) dropped from the fprop / dgrad reference, and the first wgrad split left out.  A split
is 1/splits of the sum; at conv1_2 (30 splits of 428 k pixels) the bound is 2.55 % of |terms|, so x >= 0 and dy with
a mean four times its spread make every term positive and |dw| ~ |terms|: the one-split control then fails by 1.24x
(conv1_1, 264 splits: 1.26x; measured on an H100 SXM at 700 W; the inputs are seeded, so the figure is fixed).
The gate has two controls: the ungated reference fails the exact-zero check, and the reference gated by x shifted
one pixel along W fails the bf16 bound.

Inputs: x = relu(N(0.5, 1)) in bf16 (~31 % exact zeros) with -0.0 and the smallest positive bf16 subnormal (bits
0x0001) sprinkled in; dy = N(1, 0.25) in bf16.
"""
import pytest
import torch

import vgg_oracle as vo
from isolated import assert_not_ran, assert_ran, run_isolated
from test_bench_c4_c5_gpu import (U, _activation, _bf16_ratio, _first_split, _float64_layer, _geom, _halo_eligible,
                                  _nhwc, _ratio, _report, _shape_id, _wgrad_plan)
from test_streaming_b256_gpu import DEV, _bf16_tol, _chunks, _fill

gpu = pytest.mark.gpu
BATCH, HW, SPARSITY = 256, 224, 0.8
X_MEAN, X_SD, DY_MEAN, DY_SD = 0.5, 1.0, 1.0, 0.25
CONTROL = 1.2                 # every control fails its bound by at least this factor
_TABLE = []


def _oracle_cases(vgg_type):
  """[(first scope, key)] of the distinct masked layers of `vgg_type` at 224^2, from the reference's layer table:
  key = (kind, cin, cout, k, h, w, relu_out, gate_dgrad, patch_mode).  Every 3x3 conv is followed by a ReLU; its
  input comes from a ReLU conv (gated dgrad) unless it is the first conv of a stage (the image or a pool)."""
  out, seen = [], set()
  for scope, (k, _, cin, cout), hw in vo.masked_layers(vgg_type):
    fc8 = scope.endswith('/fc8')
    key = ('conv', cin, cout, k, hw, hw, not fc8, not fc8 and not scope.endswith('_1'), cin % 8 != 0 and k > 1)
    if key not in seen:
      seen.add(key)
      out.append((scope.split('/')[-1], key))
  return out


_CASES = _oracle_cases('vgg_16')


def _table():
  """[entry] of VGG-16's distinct masked layers in first-use order, from the model itself: a batch-1 forward records
  each layer's input extent.  Entries are dicts with the module, its input extent and its key (_oracle_cases).  The
  model is built and masked once per process."""
  if _TABLE:
    return _TABLE
  from rigl_b200 import workloads
  from rigl_b200.layers import SparseConv2d
  torch.manual_seed(0)
  model = workloads.VGG('vgg_16', num_classes=1000, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', SPARSITY, seed=0)
  seen = set()

  def hook(mod, args):
    h, w = int(args[0].shape[2]), int(args[0].shape[3])
    key = ('conv', mod.in_channels, mod.out_channels, mod.ksize, h, w, mod.relu_out, mod.gate_dgrad, mod.patch_mode)
    if key not in seen:
      seen.add(key)
      _TABLE.append(dict(layer=mod, kind='conv', h=h, w=w, key=key))

  handles = [m.register_forward_pre_hook(hook) for m in model.modules() if isinstance(m, SparseConv2d)]
  model.eval()
  try:
    with torch.no_grad():
      model(torch.zeros((1, 3, HW, HW), device=DEV))
  finally:
    for h in handles:
      h.remove()
    model.train()
  torch.cuda.synchronize()
  return _TABLE


def _relu_input(n, h, w, c, gen):
  """bf16 [n, c, h, w] channels_last: relu(N(X_MEAN, X_SD)) with -0.0 at every 97th element and the smallest positive
  subnormal (bits 0x0001) at every 89th from the 13th, generated in chunks."""
  t = _fill(n * h * w, c, X_MEAN, X_SD, gen)
  for a, b in _chunks(n * h * w, c):
    t[a:b].clamp_(min=0)
  bits = t.view(torch.int16).view(-1)
  bits[::97] = -0x8000
  bits[13::89] = 1
  return t.view(n, h, w, c).permute(0, 3, 1, 2)


def _positive(t):
  """t > 0 of a bf16 tensor without NaNs, from its bits: sign clear and not +0 (subnormals included)."""
  return t.view(torch.int16) > 0


def _run_case(i):
  """Case i of _table at batch 256: fprop, then dgrad (not for the first conv: the training step never asks for the
  image gradient) and dense wgrad (beta = 0) through the layer's autograd function.  Returns (entry, x, dy, y, dx or
  None, dense wgrad, weight.grad)."""
  entry = _table()[i]
  layer = entry['layer']
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  gen = torch.Generator(device=DEV)
  gen.manual_seed(1000 * i + cin + cout)
  x = _relu_input(n, h, w, cin, gen)
  dy = _activation(n, oh, ow, cout, DY_MEAN, DY_SD, gen).to(layer.out_dtype)     # (bf16 values: exact in fp32)
  x = x.detach().requires_grad_(not layer.patch_mode)
  layer.masked_weights.fresh = False
  layer.weight.grad = None
  y = layer(x)
  assert tuple(y.shape) == tuple(dy.shape), (tuple(y.shape), tuple(dy.shape))
  y.backward(dy)
  torch.cuda.synchronize()
  return entry, x.detach(), dy, y.detach(), x.grad, layer.masked_weights.dense_grad, layer.weight.grad


def _control(cls, shape, ratio):
  print('control  %-34s %-52s %.4f' % (cls, shape, ratio))
  assert ratio >= CONTROL, '%s %s: control fails its bound by only %.3gx' % (shape, cls, ratio)


def _case(i):
  torch.cuda.reset_peak_memory_stats()
  entry, x, dy, y, dx, dense, masked = _run_case(i)
  layer = entry['layer']
  geom = n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  taps = k * k
  shape = _shape_id(entry, BATCH)
  f32_out = y.dtype == torch.float32
  gate = layer.gate_dgrad
  if layer.patch_mode:      # wgrad over the [n * oh * ow, kpitch] patch matrix: splits are ranges of its rows
    plan = _wgrad_plan(n * oh * ow, 1, 1, 1, taps * cin, cout, pitch=layer._kpitch)
    first = lambda a, b: _first_split(plan, a * oh * ow, b * oh * ow, 1, 1).view(b - a, oh, ow)
    fkern = 'patch relu fprop (bf16)'
  else:
    plan = _wgrad_plan(n, oh, ow, taps, cin, cout)
    first = lambda a, b: _first_split(plan, a, b, oh, ow)
    fkern = 'igemm fprop (fp32)' if f32_out else \
        '%s relu fprop (bf16)' % ('halo' if _halo_eligible(k, s, pad, h, w, oh, ow, cin) else 'igemm')
  dkern = 'igemm %sdgrad (bf16)' % ('gated ' if gate else '')
  xs, dys, ys = _nhwc(x), _nhwc(dy), _nhwc(y)
  dxs = None if dx is None else _nhwc(dx)
  r = dict(y=0.0, ctl_y=0.0, dx=0.0, ctl_dx=0.0, shift=0.0, ungated=False, subnormal=0, through=0)

  def check(a, b, yr, ya, ydrop, dxr, dxa, dxdrop):
    yc = ys[a:b]
    if f32_out:
      tol = (taps * cin + 1) * U * ya + 1e-300
      r['y'] = max(r['y'], _ratio(yc, yr, tol))
      r['ctl_y'] = max(r['ctl_y'], _ratio(yc, yr - ydrop, tol))
    else:
      assert not bool((yc < 0).any()), '%s: negative ReLU output in images %d:%d' % (shape, a, b)
      r['y'] = max(r['y'], _ratio(yc, yr.clamp_min(0), _bf16_tol(yr, ya)))
      r['ctl_y'] = max(r['ctl_y'], _ratio(yc, (yr - ydrop).clamp_min(0), _bf16_tol(yr - ydrop, ya)))
    if dxr is None:
      return
    dc = dxs[a:b]
    if not gate:
      r['dx'] = max(r['dx'], _bf16_ratio(dc, dxr, dxa))
      r['ctl_dx'] = max(r['ctl_dx'], _bf16_ratio(dc, dxr - dxdrop, dxa))
      return
    pos = _positive(xs[a:b])
    assert not bool(((dc != 0) & ~pos).any()), '%s: dx is not +-0 where x > 0 is false (images %d:%d)' % (shape, a, b)
    r['dx'] = max(r['dx'], _bf16_ratio(dc, dxr * pos, dxa))
    r['ctl_dx'] = max(r['ctl_dx'], _bf16_ratio(dc, (dxr - dxdrop) * pos, dxa))
    r['shift'] = max(r['shift'], _bf16_ratio(dc, dxr * torch.roll(pos, 1, dims=2), dxa))
    r['ungated'] = r['ungated'] or bool(((dxr != 0) & ~pos).any())
    sub = xs[a:b].view(torch.int16) == 1
    r['subnormal'] += int(sub.sum())
    r['through'] += int((sub & (dc != 0)).sum())

  dw, dw_abs, dw_first = _float64_layer(layer, geom, first, xs, dys, check, dgrad=dx is not None)
  _report(fkern, shape, r['y'])
  assert r['y'] <= 1, '%s: fprop off by %.3g bounds' % (shape, r['y'])
  _control(fkern + (' -channel' if k == 1 else ' -centre'), shape, r['ctl_y'])
  if dx is None:
    assert layer.patch_mode
  else:
    _report(dkern, shape, r['dx'])
    assert r['dx'] <= 1, '%s: dgrad off by %.3g bounds' % (shape, r['dx'])
    _control(dkern + (' -channel' if k == 1 else ' -centre'), shape, r['ctl_dx'])
  if gate:
    _control('gate by x shifted along W', shape, r['shift'])
    assert r['ungated'], '%s: the ungated reference passes the exact-zero check' % shape
    assert r['subnormal'] > 0 and r['through'] > 0, '%s: no subnormal x let its gradient through (%d of %d)' % (
        shape, r['through'], r['subnormal'])

  # dense wgrad: every position, masked-out ones included (RigL's grow scores)
  got = dense.view(taps, cin, cout)
  wtol = (plan['pps'] + plan['splits']) * U * dw_abs + 1e-300
  wkern = '%s wgrad (pps %d, %d splits)' % (plan['kernel'], plan['pps'], plan['splits'])
  r_w = _ratio(got, dw, wtol)
  _report(wkern, shape, r_w)
  print('wgrad    %-34s %-52s max |err| / |terms| %.3e (bound %.3e)' % (
      wkern, shape, float(((got.double() - dw).abs() / (dw_abs + 1e-300)).max()),
      (plan['pps'] + plan['splits']) * U))
  assert r_w <= 1, '%s: dense wgrad off by %.3g bounds' % (shape, r_w)
  _control(wkern + ' -first split', shape, _ratio(got, dw - dw_first, wtol))
  mask = layer.mask.to_dense().reshape(-1)
  assert torch.equal(masked.reshape(-1), dense * mask), '%s: mask * wgrad' % shape
  print('peak %s %.0f MB' % (shape, torch.cuda.max_memory_allocated() / 2 ** 20))
  del entry, x, dy, y, dx, dw, dw_abs, dw_first
  layer.weight.grad = None
  torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# Tables and launches
# ---------------------------------------------------------------------------------------------------------------

def test_vgg16_cases_cover_all_three_models():
  """The distinct cases, from the reference's table (no GPU): 10 convs and fc8; VGG-A's and VGG-19's cases are
  among them; the product's gate rule (workloads.VGG: gate_dgrad unless the input is the image or a pool) gives the
  same gates; and the launch rules send conv1_1 alone to the patch matrix and conv2_1's fprop alone to the halo
  kernels, and no gated dgrad to the halo kernels (which have no gate: that would be plain dgrad + k_relu_gate)."""
  from rigl_b200 import workloads
  keys = [key for _, key in _CASES]
  assert len(keys) == 11 and sum(key[3] == 3 for key in keys) == 10
  assert keys[-1] == ('conv', 512, 1000, 1, 1, 1, False, False, False)
  for other in ('vgg_a', 'vgg_19'):
    assert {key for _, key in _oracle_cases(other)} <= set(keys), other
  for vgg_type in sorted(vo.CFG):
    prev_pool = True
    for scope, cin, cout, pool in workloads.vgg_plan(vgg_type):
      assert (not prev_pool) == (not scope.endswith('_1')), scope
      prev_pool = pool
  assert [name for name, key in _CASES if key[8]] == ['conv1_1']
  halo = [name for name, (_, cin, cout, k, h, w, relu, g, p) in _CASES
          if k == 3 and _halo_eligible(k, 1, 1, h, w, h, w, cin)]
  assert halo == ['conv2_1']
  assert not [name for name, (_, cin, cout, k, h, w, relu, g, p) in _CASES
              if g and _halo_eligible(k, 1, 1, h, w, h, w, cout)]


@gpu
def test_model_table_matches_the_oracle():
  table = _table()
  assert [e['key'] for e in table] == [key for _, key in _CASES]
  assert [e['layer'].scope.split('/')[-1] for e in table] == [name for name, _ in _CASES]
  for e in table:
    n, h, w, cin, cout, k, s, pad, oh, ow = _geom(e, BATCH)
    if e['layer'].patch_mode:
      plan = _wgrad_plan(n * oh * ow, 1, 1, 1, k * k * cin, cout, pitch=e['layer']._kpitch)
    else:
      plan = _wgrad_plan(n, oh, ow, k * k, cin, cout)
    print('plan %-52s %s wgrad: %d splits x %d pixels' % (_shape_id(e, BATCH), plan['kernel'], plan['splits'],
                                                         plan['pps']))
    assert plan['kernel'] == 'tc' and plan['splits'] > 1


@gpu
def test_vgg16_layers_run_their_kernels():
  """Which kernels each case launches at full size, in a fresh process (the first call builds the table: its batch-1
  forward is not witnessed).  No case runs the standalone gate or a CUDA-core kernel."""
  table = _table()
  calls = [('_table', ())] + [('_run_case', (i,)) for i in range(len(table))]
  torch.cuda.empty_cache()
  ran = run_isolated('test_vgg_b256_gpu', calls, timeout=900)[1:]
  for entry, names in zip(table, ran):
    layer = entry['layer']
    what = _shape_id(entry, BATCH)
    n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
    assert_not_ran(names, r'k_relu_gate', what)
    assert_not_ran(names, r'k_simt_', what)
    assert_ran(names, r'k_igemm_wgrad<', what)
    assert_ran(names, r'k_splitk_reduce', what)
    if layer.patch_mode:
      assert_ran(names, r'k_im2col', what)
      assert_ran(names, r'k_igemm_kmajor_relu<.*false>', what)
      assert_not_ran(names, r'k_igemm_kmajor(_relu)?<.*true>|k_igemm_kmajor<', what)     # no dgrad
      continue
    assert_not_ran(names, r'k_im2col', what)
    if not layer.relu_out:                                     # fc8
      assert_ran(names, r'k_igemm_kmajor<', what)
      assert_not_ran(names, r'relu|k_halo3x3', what)
      continue
    if _halo_eligible(k, s, pad, h, w, oh, ow, cin):
      assert_ran(names, r'k_halo3x3_kmajor_relu', what)
      assert_not_ran(names, r'k_igemm_kmajor_relu<.*false>', what)
    else:
      assert_ran(names, r'k_igemm_kmajor_relu<.*false>', what)
      assert_not_ran(names, r'k_halo3x3', what)
    if layer.gate_dgrad:
      assert_ran(names, r'k_igemm_kmajor_relu<.*true>', what)
      assert_not_ran(names, r'k_igemm_kmajor<', what)          # the one dgrad is the gated one
    else:
      assert_ran(names, r'k_igemm_kmajor<', what)
      assert_not_ran(names, r'k_igemm_kmajor_relu<.*true>', what)


# ---------------------------------------------------------------------------------------------------------------
# Every masked layer against float64
# ---------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('i', range(len(_CASES)), ids=[name for name, _ in _CASES])
def test_vgg16_layer_b256_against_float64(i):
  _case(i)


# ---------------------------------------------------------------------------------------------------------------
# Pool and gate at batch 256, exact
# ---------------------------------------------------------------------------------------------------------------

def _key(bits):
  """An int32 that orders bf16 values (NaN-free) as floats do, from their int16 bits: +-0 both map to 0."""
  b = bits.int()
  return torch.where(b >= 0, b, -(b & 0x7FFF))


def _pool_input(n, h, w, c, gen):
  """bf16 [n, h, w, c]: values in {0, 0.5, 1, 1.5} (ties everywhere), the first c / 4 channels all zero (windows
  whose maximum is 0), -0.0 at every 97th element and the smallest positive subnormal at every 89th from the 13th."""
  t = torch.empty((n * h * w, c), dtype=torch.bfloat16, device=DEV)
  for a, b in _chunks(n * h * w, c):
    t[a:b] = torch.randint(0, 4, (b - a, c), generator=gen, device=DEV, dtype=torch.int16).to(torch.bfloat16) * 0.5
  t[:, :c // 4] = 0.0
  bits = t.view(torch.int16).view(-1)
  bits[::97] = -0x8000
  bits[13::89] = 1
  return t.view(n, h, w, c)


_POOL_SHAPES = [(224, 64), (112, 128), (56, 256), (28, 512)]


@gpu
@pytest.mark.parametrize('hw,c', _POOL_SHAPES, ids=['256x%dx%dx%d' % (hw, hw, c) for hw, c in _POOL_SHAPES])
def test_pool2x2_relu_b256_exact(hw, c):
  """max_pool2x2_relu forward (the first maximum's bits), route bytes (the window index of the first maximum if it
  is > 0, else 0xFF) and backward (dy's bits at the routed pixel, +0 elsewhere), bit for bit against a reference
  computed on the device in chunks of images.  Control: the route of the last maximum differs (ties)."""
  from rigl_b200.norm import max_pool2x2_relu
  torch.cuda.reset_peak_memory_stats()
  gen = torch.Generator(device=DEV)
  gen.manual_seed(hw * c)
  n, oh = BATCH, hw // 2
  xn = _pool_input(n, hw, hw, c, gen)
  x = xn.permute(0, 3, 1, 2).requires_grad_(True)
  y = max_pool2x2_relu(x)
  arg = y.grad_fn.saved_tensors[0]                    # route bytes [n, oh, ow, c] (freed by the backward)
  dy = _activation(n, oh, oh, c, 0.0, 1.0, gen)
  y.backward(dy)
  torch.cuda.synchronize()
  yn, dyn, dxn = _nhwc(y.detach()), _nhwc(dy), _nhwc(x.grad)
  differs = False
  step = max(1, (1 << 24) // (hw * hw * c))
  for a in range(0, n, step):
    b = min(a + step, n)
    win = torch.stack([xn[a:b, i:2 * oh:2, j:2 * oh:2] for i in (0, 1) for j in (0, 1)]).view(torch.int16)
    keys = _key(win)
    first = torch.argmax(keys, dim=0)                 # documented: the first maximal index
    top = keys.amax(0)
    want_y = torch.gather(win, 0, first[None])[0]
    assert torch.equal(yn[a:b].view(torch.int16), want_y), 'forward, images %d:%d' % (a, b)
    route = torch.where(top > 0, first, 255).to(torch.uint8)
    assert torch.equal(arg[a:b], route), 'route bytes, images %d:%d' % (a, b)
    last = 3 - torch.argmax(keys.flip(0), dim=0)
    differs = differs or not torch.equal(arg[a:b], torch.where(top > 0, last, 255).to(torch.uint8))
    d = dyn[a:b].view(torch.int16)
    for j in range(4):
      want = torch.where(route == j, d, torch.zeros_like(d))
      got = dxn[a:b, j >> 1:2 * oh:2, j & 1:2 * oh:2].view(torch.int16)
      assert torch.equal(got, want), 'backward window position %d, images %d:%d' % (j, a, b)
    del win, keys, first, top, want_y, route, last
  assert differs, 'control: routing ties to the last maximum passes'
  print('peak pool 256x%dx%dx%d %.0f MB' % (hw, hw, c, torch.cuda.max_memory_allocated() / 2 ** 20))
  del x, y, dy, xn, arg
  torch.cuda.empty_cache()


@gpu
def test_relu_grad_gate_b256_exact():
  """relu_grad_gate's backward on VGG-16's last conv output (256 x 512 x 14 x 14): dy's bits where x > 0 (subnormals
  included), +0 elsewhere (-0.0 included)."""
  from rigl_b200.norm import relu_grad_gate
  gen = torch.Generator(device=DEV)
  gen.manual_seed(14)
  x = _relu_input(BATCH, 14, 14, 512, gen).requires_grad_(True)
  dy = _activation(BATCH, 14, 14, 512, 0.0, 1.0, gen)
  relu_grad_gate(x).backward(dy)
  torch.cuda.synchronize()
  xs = _nhwc(x.detach())
  d = _nhwc(dy).view(torch.int16)
  got = _nhwc(x.grad).view(torch.int16)
  pos = _positive(xs)
  assert torch.equal(got, torch.where(pos, d, torch.zeros_like(d)))
  sub = xs.view(torch.int16) == 1
  assert bool(sub.any()) and bool(((got != 0) & sub).any()), 'no subnormal x let its gradient through'
  assert bool((~pos & (d != 0)).any()), 'control: the ungated gradient would pass'


# ---------------------------------------------------------------------------------------------------------------
# The whole step at batch 256
# ---------------------------------------------------------------------------------------------------------------

def _step_setup(seed):
  from rigl_b200 import workloads
  torch.manual_seed(seed)
  model = workloads.VGG('vgg_16', num_classes=1000, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', SPARSITY, seed=seed)
  h = workloads.TrainHarness(model, lr=0.01)
  g = torch.Generator(device=DEV).manual_seed(seed)
  x = torch.randn(BATCH, 3, HW, HW, device=DEV, generator=g).to(torch.bfloat16) \
      .contiguous(memory_format=torch.channels_last)
  labels = torch.randint(0, 1000, (BATCH,), device=DEV, generator=g)
  return model, h, x, labels


@gpu
def test_fused_route_equals_standalone_gate_route_b256(monkeypatch):
  """One VGG-16 step with the ReLU in the conv epilogues against the same step with layers.FUSE_RELU = False (plain
  conv + k_relu_gate): gating only selects values, so the loss and every dense gradient are bit-identical (+-0
  compare equal).  rigl_relu_gate calls are counted, each one checked to be one launch: the fused route makes exactly
  one (the last conv's relu_grad_gate), the standalone route one per ReLU conv, one per gated edge, and that one."""
  from rigl_b200 import _cabi, layers, norm
  torch.cuda.reset_peak_memory_stats()
  model, h, x, labels = _step_setup(31)
  gates = []
  real = layers.relu_gate

  def counted(a, g, out):
    before = _cabi.launch_count()
    res = real(a, g, out)
    assert _cabi.launch_count() - before == 1
    gates.append(1)
    return res

  monkeypatch.setattr(layers, 'relu_gate', counted)
  monkeypatch.setattr(norm, 'relu_gate', counted)
  out = {}
  try:
    for fuse in (True, False):
      monkeypatch.setattr(layers, 'FUSE_RELU', fuse)
      del gates[:]
      loss = h._forward_backward(x, labels, set_to_none=False)
      torch.cuda.synchronize()
      out[fuse] = (len(gates), loss.detach().clone(),
                   [l.masked_weights.dense_grad.clone() for l in model.registry.layers()])
    convs = list(model.convs)
    want = sum(c.relu_out for c in convs) + sum(c.gate_dgrad for c in convs) + 1
    assert (out[True][0], out[False][0]) == (1, want) and want == 13 + 8 + 1, (out[True][0], out[False][0], want)
    assert torch.equal(out[True][1], out[False][1]), (float(out[True][1]), float(out[False][1]))
    for l, p, q in zip(model.registry.layers(), out[True][2], out[False][2]):
      assert torch.equal(p, q), l.scope
    print('peak whole step, two routes %.0f MB' % (torch.cuda.max_memory_allocated() / 2 ** 20))
  finally:
    del h, model, out
    torch.cuda.empty_cache()


@gpu
def test_cuda_graph_wgrad_side_stream_b256_matches_serial_backward():
  """VGG-16's step captured with the dense wgrad on a forked stream, replayed twice, against the serial eager
  backward: every kernel is deterministic, so the loss and every dense gradient match bit for bit.  The eager loss
  is kept detached only: a live autograd graph of the eager step would keep the weights' gradient accumulators, and
  the stream they were created on, into the capture, whose backward would then wait on uncaptured work."""
  torch.cuda.reset_peak_memory_stats()
  model, h, x, labels = _step_setup(41)
  want_loss = h._forward_backward(x, labels, set_to_none=False).detach().clone()     # serial (_overlap is unset)
  torch.cuda.synchronize()
  layers_ = model.registry.layers()
  ref = [l.masked_weights.dense_grad.clone() for l in layers_]
  try:
    assert h.enable_cuda_graph(x, labels, overlap_wgrad=True) and h._overlap
    for _ in range(2):
      for l in layers_:
        l.masked_weights.dense_grad.fill_(float('nan'))
      h._g_fb.replay()
      torch.cuda.synchronize()
      assert torch.equal(h._sloss, want_loss), (float(h._sloss), float(want_loss))
      for l, d in zip(layers_, ref):
        assert torch.equal(l.masked_weights.dense_grad, d), l.scope
    print('peak whole step, CUDA graph %.0f MB' % (torch.cuda.max_memory_allocated() / 2 ** 20))
  finally:                    # the graph pool and the model hold the step's activations: give them back
    h.release_cuda_graph()
    del h, model
    torch.cuda.empty_cache()
