"""ResNet-50's training path against float64 at the size the benchmark's headline configuration runs it: batch 256,
224 x 224, ERK 0.8 (bench.py c2).

Covered: every distinct masked layer of workloads.ResNet50 -- the space-to-depth stem (csrc/stem_s2d.cuh), the 22
distinct conv shapes and final_dense -- run as the model trains them: train mode, bf16 channels_last input, fprop
with the batch-norm statistics epilogue where the model asks for it and the policy of conv_route grants it, then
dgrad (not for the stem: the image needs no gradient) and the dense wgrad through the layer's autograd function.
At this size the launchers take decisions nothing smaller reaches: the stem's wgrad runs 7168 strips over one CTA
per SM (~55 strips, 24 k positions accumulated in fp32 per CTA) and adds the 132 partials in k_stem_s2d_reduce;
group 1's 3x3 (56^2, 64 -> 64) runs fprop, dgrad and wgrad on the halo kernels, whose wgrad adds 55 strips per CTA
and then 132 partials in k_splitk_reduce; 16 of the 22 conv shapes take the K-major fprop with the statistics
epilogue.

The float64 references run on the device per tap over chunks of whole images (test_bench_c4_c5_gpu._float64_layer).
Bounds (u = 2^-24; |terms| = the same float64 computation on |x|, |w * m| and |dy|), as in test_bench_c4_c5_gpu:
- bf16 fprop / dgrad: _bf16_tol with |terms|.
- The 1x1 stride-2 projections: input pixels no tap reaches (odd h or w) get dx exactly +-0 (tc_dgrad clears them).
- Statistics-epilogue layers: the same layer with collect_bn_stats = False gives a bit-identical output (both run
  the same K loop per output element; the epilogue only adds column sums of the staged tile).
- Dense wgrad (k_igemm_wgrad): (pps + splits) u |terms| (_wgrad_plan).
- Strip wgrads (stem, halo layer): one CTA per SM adds strips b, b + grid, ... in fp32, then the grid partials
  are added in CTA order: (valid positions per CTA + grid) u |terms| (_strip_plan restates s2d_geom / halo_geom).
- final_dense's fp32 logits with a nonzero bias: (K + 1) u (|terms| + |bias|), K = 2048; bias.grad against the
  float64 column sum of dy, n u sum |dy|.
- mask * wgrad equals dense * mask exactly.
Every bound has a control that must fail by at least CONTROL: the centre tap (1x1 and final_dense: the input channel
with the most surviving weights for fprop, that output channel for dgrad) dropped from the fprop / dgrad reference,
the first wgrad split -- for the strip wgrads the strips of CTA 0 -- left out, the bias left out of the logits and
the first row of dy left out of its column sum.  x >= 0 and dy with a mean four times its spread make every wgrad
term positive, so |dw| ~ |terms| and the one-split control is not vacuous.  Measured on an H100 SXM (80 GB HBM3)
at 700 W, the largest err / bound is 0.39 on the bf16 outputs, 0.0022 on the logits, 0.055 on the stem's wgrad,
0.038 on the halo wgrad and 0.042 on the split-K wgrads; the weakest control (the stem's wgrad without CTA 0's
strips) fails by 5.3x, every other by more than 20x.  The inputs are seeded, so the figures are fixed.

Inputs: x = relu(N(0.5, 1)) in bf16 (the stem's image too); dy = N(1, 0.25) in bf16.
"""
import pytest
import torch

from isolated import assert_not_ran, assert_ran, run_isolated
from oracle import rigl_oracle as orc
from test_bench_c4_c5_gpu import (U, _activation, _bf16_ratio, _first_split, _float64_layer, _geom, _halo_eligible,
                                  _nhwc, _ratio, _report, _shape_id, _wgrad_plan)
from test_streaming_b256_gpu import DEV, _chunks, _fill

gpu = pytest.mark.gpu
BATCH, HW, SPARSITY = 256, 224, 0.8
X_MEAN, X_SD, DY_MEAN, DY_SD = 0.5, 1.0, 1.0, 0.25
CONTROL = 1.2                 # every control fails its bound by at least this factor
_TABLE = []


def _oracle_cases():
  """[(first scope, key)] of ResNet-50's distinct masked layers at 224^2, from the reference's layer table:
  key = (kind, cin, cout, k, stride, input extent)."""
  out, seen = [], set()
  for scope, shape, stride, out_hw in orc.resnet50_masked_layers():
    if len(shape) == 2:
      key = ('linear', shape[0], shape[1], 1, 1, 1)
    else:
      key = ('conv', shape[2], shape[3], shape[0], stride, out_hw * stride)
    if key not in seen:
      seen.add(key)
      out.append((scope.split('/')[-1], key))
  return out


_CASES = _oracle_cases()


def _table():
  """[entry] of ResNet-50's distinct masked layers in first-use order, from the model itself: a batch-1 forward
  records each layer's input extent.  Entries are dicts with the module, its kind, input extent and key
  (_oracle_cases).  The model is built and masked once per process, as bench.py builds c2."""
  if _TABLE:
    return _TABLE
  from rigl_b200 import workloads
  from rigl_b200.layers import SparseConv2d, SparseLinear
  torch.manual_seed(0)
  model = workloads.ResNet50(1000, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', SPARSITY, seed=0)
  seen = set()

  def hook(mod, args):
    if isinstance(mod, SparseLinear):
      key, h, w, kind = ('linear', mod.in_channels, mod.out_channels, 1, 1, 1), 1, 1, 'linear'
    else:
      h, w, kind = int(args[0].shape[2]), int(args[0].shape[3]), 'conv'
      key = ('conv', mod.in_channels, mod.out_channels, mod.ksize, mod.stride, h)
    if key not in seen:
      seen.add(key)
      _TABLE.append(dict(layer=mod, kind=kind, h=h, w=w, key=key, model=model))

  handles = [m.register_forward_pre_hook(hook) for m in model.modules() if isinstance(m, (SparseConv2d, SparseLinear))]
  model.eval()
  try:
    with torch.no_grad():
      model(torch.zeros((1, 3, HW, HW), device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
  finally:
    for h in handles:
      h.remove()
    model.train()
  torch.cuda.synchronize()
  return _TABLE


# ---------------------------------------------------------------------------------------------------------------
# Launch rules, restated from the launchers
# ---------------------------------------------------------------------------------------------------------------

def _is_stem(entry):
  return entry['kind'] == 'conv' and entry['layer'].patch_mode


def _is_halo(entry):
  """csrc/igemm_tc.cu: fprop, dgrad and wgrad all on the halo kernels (halo_fprop_ok, halo_dgrad_ok and
  halo_wgrad_ok's cout <= 64)."""
  if entry['kind'] != 'conv':
    return False
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  return _halo_eligible(k, s, pad, h, w, oh, ow, cin) and _halo_eligible(k, s, pad, h, w, oh, ow, cout) and cout <= 64


def _stats_epilogue(entry):
  """conv_route's policy for the batch-norm statistics epilogue: the layer asks for it (collect_bn_stats), is not on
  the halo kernels or the stem's path, and K = taps * cin >= 512, or K >= 256 with cout <= 128."""
  l = entry['layer']
  if entry['kind'] != 'conv' or _is_stem(entry) or _is_halo(entry) or not l.collect_bn_stats:
    return False
  kk = l.ksize * l.ksize * l.in_channels
  return kk >= 512 or (kk >= 256 and l.out_channels <= 128)


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _strip_plan(kernel, n, oh, ow, r):
  """The summation structure of a strip wgrad (k_stem_s2d_wgrad, k_halo3x3_wgrad): strips of r output rows,
  ceil(oh / r) per image; grid = min(strips, SMs) CTAs, CTA b adding strips b, b + grid, ... in fp32; then the grid
  partials are added in CTA order.  pps = the most valid output positions one CTA adds."""
  spi = -(-oh // r)
  total = spi * n
  grid = min(total, _sms())
  per_cta = [0] * grid
  for strip in range(total):
    h0 = (strip % spi) * r
    per_cta[strip % grid] += min(r, oh - h0) * ow
  return dict(kernel=kernel, r=r, spi=spi, grid=grid, pps=max(per_cta), splits=grid)


def _stem_plan(n, oh, ow):
  """stem_s2d.cuh s2d_geom(wgrad = true): R = 4 output rows per strip."""
  return _strip_plan('s2d', n, oh, ow, min(4, oh))


def _halo_plan(n, h, w):
  """halo3x3.cuh halo_geom for the wgrad (smem_fixed = 0, dy_tile = 1): the strip height R = (128 / Wp) * t and
  buffer count of least cost that fit in 227 KB of shared memory."""
  wp = 8
  while wp < w + 2:
    wp *= 2
  rt = 128 // wp
  best = None
  for nbuf in (2, 3, 4):
    for t in range(1, 9):
      r = rt * t
      a_buf = -(-((r + 2) * wp + 8) * 128 // 1024) * 1024
      if nbuf * (a_buf + r * wp * 128) + 2048 > 227 * 1024:
        break
      strips = -(-h // r)
      cost = (strips * (r + 2) + strips * r) * 16 + strips * 8
      if nbuf == 2:
        cost = cost * 3 // 2
      if best is None or cost < best[0]:
        best = (cost, r)
      if r >= h:
        break
  return _strip_plan('halo', n, h, w, best[1])


def _first_cta(plan, a, b, oh, ow):
  """bool [b - a, oh, ow]: the output pixels of images [a, b) whose strips CTA 0 adds."""
  n = torch.arange(a, b, device=DEV)[:, None, None]
  h = torch.arange(oh, device=DEV)[None, :, None]
  strip = n * plan['spi'] + h // plan['r']
  return (strip % plan['grid'] == 0).expand(b - a, oh, ow)


def _plan(entry):
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  if _is_stem(entry):
    return _stem_plan(n, oh, ow)
  if _is_halo(entry):
    return _halo_plan(n, h, w)
  return _wgrad_plan(n, oh, ow, k * k, cin, cout)


def _first(plan, oh, ow):
  if plan['kernel'] in ('s2d', 'halo'):
    return lambda a, b: _first_cta(plan, a, b, oh, ow)
  return lambda a, b: _first_split(plan, a, b, oh, ow)


# ---------------------------------------------------------------------------------------------------------------
# One layer at batch 256
# ---------------------------------------------------------------------------------------------------------------

def _relu_input(rows, c, gen):
  """bf16 [rows, c]: relu(N(X_MEAN, X_SD)), generated in chunks."""
  t = _fill(rows, c, X_MEAN, X_SD, gen)
  for a, b in _chunks(rows, c):
    t[a:b].clamp_(min=0)
  return t


def _bias(cout):
  """A nonzero classifier bias in +-[0.25, 2], in a fixed shuffled order."""
  g = torch.Generator(device=DEV)
  g.manual_seed(cout)
  mag = torch.linspace(0.25, 2.0, cout, device=DEV)
  sign = torch.where(torch.arange(cout, device=DEV) % 2 == 0, 1.0, -1.0)
  return (mag * sign)[torch.randperm(cout, generator=g, device=DEV)]


def _run_case(i):
  """Case i of _table at batch 256 in train mode: fprop, then dgrad (not for the stem) and dense wgrad (beta = 0)
  through the layer's autograd function.  Returns (entry, x, dy, y, dx or None, dense wgrad, weight.grad, bias.grad
  or None)."""
  entry = _table()[i]
  layer = entry['layer']
  assert layer.training
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  gen = torch.Generator(device=DEV)
  gen.manual_seed(1000 * i + cin + cout)
  if entry['kind'] == 'linear':
    x = _relu_input(n, cin, gen)
    dy = _fill(n, cout, DY_MEAN, DY_SD, gen).to(layer.out_dtype)        # (bf16 values: exact in fp32)
    with torch.no_grad():
      layer.bias.copy_(_bias(cout))
    layer.bias.grad = None
  else:
    x = _relu_input(n * h * w, cin, gen).view(n, h, w, cin).permute(0, 3, 1, 2)
    dy = _activation(n, oh, ow, cout, DY_MEAN, DY_SD, gen).to(layer.out_dtype)
  x = x.detach().requires_grad_(not _is_stem(entry))        # the image needs no gradient, as in training
  layer.masked_weights.fresh = False
  layer.weight.grad = None
  y = layer(x)
  assert tuple(y.shape) == tuple(dy.shape), (tuple(y.shape), tuple(dy.shape))
  y.backward(dy)
  torch.cuda.synchronize()
  bias_grad = layer.bias.grad if entry['kind'] == 'linear' else None
  return entry, x.detach(), dy, y.detach(), x.grad, layer.masked_weights.dense_grad, layer.weight.grad, bias_grad


def _control(cls, shape, ratio):
  print('control  %-34s %-52s %.4f' % (cls, shape, ratio))
  assert ratio >= CONTROL, '%s %s: control fails its bound by only %.3gx' % (shape, cls, ratio)


def _case(i):
  torch.cuda.reset_peak_memory_stats()
  entry, x, dy, y, dx, dense, masked, bias_grad = _run_case(i)
  layer = entry['layer']
  geom = n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, BATCH)
  taps = k * k
  shape = _shape_id(entry, BATCH)
  linear = entry['kind'] == 'linear'
  stem, halo, stats = _is_stem(entry), _is_halo(entry), _stats_epilogue(entry)
  proj_s2 = k == 1 and s == 2

  # where the launch rules sent it (deterministic witnesses; test_resnet50_layers_run_their_kernels names them)
  if stem:
    assert layer._use_s2d, '%s: the stem did not take the space-to-depth path' % shape
  if not linear and not stem:
    assert (layer.bn_partial is not None) == stats, '%s: statistics epilogue %s, policy says %s' % (
        shape, layer.bn_partial is not None, stats)

  if linear:
    fkern = 'igemm fprop (fp32 + bias)'
  elif stem:
    fkern = 's2d stem fprop (bf16)'
  elif halo:
    fkern = 'halo fprop (bf16)'
  else:
    fkern = 'igemm fprop%s (bf16)' % (' + bn stats' if stats else '')
  dkern = '%s dgrad (bf16)' % ('halo' if halo else 'igemm')
  plan = _plan(entry)
  xs, dys, ys = _nhwc(x), _nhwc(dy), _nhwc(y)
  dxs = None if dx is None else _nhwc(dx)
  bias = layer.bias.detach().double() if linear else None
  r = dict(y=0.0, ctl_y=0.0, ctl_bias=0.0, dx=0.0, ctl_dx=0.0, holes=0, filled=0)

  def check(a, b, yr, ya, ydrop, dxr, dxa, dxdrop):
    yc = ys[a:b]
    if linear:
      tol = (taps * cin + 1) * U * (ya + bias.abs()) + 1e-300
      r['y'] = max(r['y'], _ratio(yc, yr + bias, tol))
      r['ctl_y'] = max(r['ctl_y'], _ratio(yc, yr + bias - ydrop, tol))
      r['ctl_bias'] = max(r['ctl_bias'], _ratio(yc, yr, tol))
    else:
      r['y'] = max(r['y'], _bf16_ratio(yc, yr, ya))
      r['ctl_y'] = max(r['ctl_y'], _bf16_ratio(yc, yr - ydrop, ya))
    if dxr is None:
      return
    dc = dxs[a:b]
    r['dx'] = max(r['dx'], _bf16_ratio(dc, dxr, dxa))
    r['ctl_dx'] = max(r['ctl_dx'], _bf16_ratio(dc, dxr - dxdrop, dxa))
    if proj_s2:
      # no tap reaches an odd input row or column: exactly +-0 there (the bf16 bound would pass small values)
      for hole in (dc[:, 1::2], dc[:, 0::2, 1::2]):
        assert not bool((hole != 0).any()), '%s: dx is not +-0 where no tap reaches (images %d:%d)' % (shape, a, b)
        r['holes'] += hole.numel()
      r['filled'] += int((dc[:, 0::2, 0::2] != 0).sum())

  dw, dw_abs, dw_first = _float64_layer(layer, geom, _first(plan, oh, ow), xs, dys, check, dgrad=dx is not None)
  _report(fkern, shape, r['y'])
  assert r['y'] <= 1, '%s: fprop off by %.3g bounds' % (shape, r['y'])
  _control(fkern + (' -channel' if k == 1 else ' -centre'), shape, r['ctl_y'])
  if linear:
    _control(fkern + ' -bias', shape, r['ctl_bias'])
  if stem:
    assert dx is None
  else:
    _report(dkern, shape, r['dx'])
    assert r['dx'] <= 1, '%s: dgrad off by %.3g bounds' % (shape, r['dx'])
    _control(dkern + (' -channel' if k == 1 else ' -centre'), shape, r['ctl_dx'])
  if proj_s2:
    assert r['holes'] == n * h * w * cin * 3 // 4 and r['filled'] > 0, (r['holes'], r['filled'])

  # dense wgrad: every position, masked-out ones included (RigL's grow scores)
  got = dense.view(taps, cin, cout)
  wtol = (plan['pps'] + plan['splits']) * U * dw_abs + 1e-300
  what = 'CTA' if plan['kernel'] in ('s2d', 'halo') else 'split'
  wkern = '%s wgrad (pps %d, %d %ss)' % (plan['kernel'], plan['pps'], plan['splits'], what)
  r_w = _ratio(got, dw, wtol)
  _report(wkern, shape, r_w)
  print('wgrad    %-34s %-52s max |err| / |terms| %.3e (bound %.3e)' % (
      wkern, shape, float(((got.double() - dw).abs() / (dw_abs + 1e-300)).max()),
      (plan['pps'] + plan['splits']) * U))
  assert r_w <= 1, '%s: dense wgrad off by %.3g bounds' % (shape, r_w)
  _control(wkern + ' -first ' + what, shape, _ratio(got, dw - dw_first, wtol))
  mask = layer.mask.to_dense().reshape(-1)
  assert torch.equal(masked.reshape(-1), dense * mask), '%s: mask * wgrad' % shape

  if linear:                  # bias.grad: the fp32 column sum of dy
    d = dy.double()
    want, mag = d.sum(0), d.abs().sum(0)
    btol = n * U * mag + 1e-300
    r_b = _ratio(bias_grad, want, btol)
    _report('bias grad (fp32 column sum)', shape, r_b)
    assert r_b <= 1, '%s: bias.grad off by %.3g bounds' % (shape, r_b)
    _control('bias grad -first row', shape, _ratio(bias_grad, want - d[0], btol))

  if stats:                   # the plain fprop gives the statistics variant's output bit for bit
    layer.collect_bn_stats = False
    try:
      with torch.no_grad():
        y_plain = layer(x)
    finally:
      layer.collect_bn_stats = True
    assert layer.bn_partial is None
    assert torch.equal(_nhwc(y_plain).view(torch.int16), ys.view(torch.int16)), \
        '%s: plain fprop differs from the statistics-epilogue fprop' % shape
    del y_plain
  print('peak %s %.0f MB' % (shape, torch.cuda.max_memory_allocated() / 2 ** 20))
  del entry, x, dy, y, dx, dw, dw_abs, dw_first
  layer.weight.grad = None
  torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# Tables and launches
# ---------------------------------------------------------------------------------------------------------------

def test_oracle_cases_and_launch_rules():
  """The distinct cases, from the reference's table (no GPU): the stem, 22 conv shapes and final_dense; and where
  the launch rules send them -- one layer (group 1's 3x3) on the halo kernels, the statistics epilogue on 16."""
  keys = [key for _, key in _CASES]
  assert len(keys) == 24 and keys[0] == ('conv', 3, 64, 7, 2, 224) and keys[-1] == ('linear', 2048, 1000, 1, 1, 1)
  assert sum(key[0] == 'conv' for key in keys) == 23
  halo = [key for key in keys if key[0] == 'conv' and key[3] == 3 and key[4] == 1 and key[2] <= 64 and
          _halo_eligible(3, 1, 1, key[5], key[5], key[5], key[5], key[1])]
  assert halo == [('conv', 64, 64, 3, 1, 56)]
  kk = lambda key: key[3] * key[3] * key[1]
  stats = [key for key in keys[1:-1] if key not in halo and (kk(key) >= 512 or (kk(key) >= 256 and key[2] <= 128))]
  assert len(stats) == 16


@gpu
def test_model_table_matches_the_oracle():
  """The model's own table: 24 entries equal to the oracle's; the stem is supported by the space-to-depth kernels,
  exactly one layer runs on the halo kernels, and the statistics epilogue is predicted on 16 layers."""
  from rigl_b200 import _cabi
  table = _table()
  assert len(table) == 24
  assert [e['key'] for e in table] == [key for _, key in _CASES]
  assert [e['layer'].scope.split('/')[-1] for e in table] == [name for name, _ in _CASES]
  stem = table[0]['layer']
  assert stem.patch_mode and stem.s2d_mode and stem.collect_bn_stats
  assert _cabi.lib().rigl_stem_s2d_supported(stem._desc(BATCH, HW, HW))
  assert [e['key'] for e in table if _is_halo(e)] == [('conv', 64, 64, 3, 1, 56)]
  assert sum(_stats_epilogue(e) for e in table) == 16
  assert all(e['layer'].collect_bn_stats for e in table if e['kind'] == 'conv')
  for e in table:
    p = _plan(e)
    print('plan %-52s %s wgrad: %d %s x %d positions' % (_shape_id(e, BATCH), p['kernel'], p['splits'],
                                                        'CTAs' if p['kernel'] in ('s2d', 'halo') else 'splits',
                                                        p['pps']))
    assert p['kernel'] in ('tc', 's2d', 'halo')


@gpu
def test_resnet50_layers_run_their_kernels():
  """Which kernels each case launches at full size, in a fresh process (the first call builds the table: its
  batch-1 forward is not witnessed)."""
  table = _table()
  calls = [('_table', ())] + [('_run_case', (i,)) for i in range(len(table))]
  torch.cuda.empty_cache()
  ran = run_isolated('test_resnet50_b256_gpu', calls, timeout=900)[1:]
  for entry, names in zip(table, ran):
    what = _shape_id(entry, BATCH)
    assert_not_ran(names, r'k_simt_', what)
    if _is_stem(entry):
      for kern in ('k_stem_s2d_fold', 'k_stem_s2d_fprop', 'k_stem_s2d_wgrad', 'k_stem_s2d_reduce'):
        assert_ran(names, kern, what)
      assert_not_ran(names, r'k_im2col', what)
      continue
    if _is_halo(entry):
      assert_ran(names, r'k_halo3x3_kmajor(?!_relu)', what)
      assert_ran(names, r'k_halo3x3_wgrad', what)
      continue
    assert_ran(names, r'k_igemm_kmajor<', what)
    assert_ran(names, r'k_igemm_wgrad<', what)
    if _plan(entry)['splits'] > 1:
      assert_ran(names, r'k_splitk_reduce', what)
    assert_not_ran(names, r'k_halo3x3', what)


# ---------------------------------------------------------------------------------------------------------------
# Every masked layer against float64
# ---------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize('i', range(len(_CASES)), ids=['%d-%s' % (i, name) for i, (name, _) in enumerate(_CASES)])
def test_resnet50_layer_b256_against_float64(i):
  _case(i)
