"""The kernels of the two smaller benchmark configurations against float64, at the size the benchmark runs them:
MobileNet-v1 (batch 256, 224 x 224, 90 % uniform) and WideResNet-22-2 (batch 128, 32 x 32, 95 % ERK).

Covered: every distinct masked conv and linear layer of the two models (fprop, dgrad, dense wgrad and mask * wgrad),
the native depthwise 3x3 kernels (csrc/depthwise.cu) on MobileNet-v1's nine depthwise shapes, and batch norm at
WRN's four shapes.  At this size the launchers take decisions small problems never reach: wgrad split-K with a
few hundred splits, K-major tiles with a partial 64-channel K block (cin = 16, 32) over millions of pixels, WRN's
3x3 layers on the generic per-tap kernels (too narrow for the halo kernels), TF 'SAME' stride-2 padding, and
depthwise weight gradients that add a hundred terms per thread.

The layer tables come from workloads.MobileNetV1 / workloads.WideResNet(22, 2) themselves (a batch-1 forward
records every layer's input shape), masked by init_masks with the benchmark's method and sparsity.  The float64
references run on the device, per tap as DGEMMs over chunks of whole images, so no float64 copy of a whole
activation is ever made.

Bounds (u = 2^-24, the fp32 unit roundoff; |terms| = the same float64 computation on |x|, |w * m| and |dy|):
- bf16 outputs (fprop, dgrad, depthwise fprop / dgrad): test_streaming_b256_gpu._close_bf16 with `cancelled` =
  |terms|: one bf16 ulp, 2^-9 of the chunk's largest magnitude, and 2^-22 of |terms|.
- fp32 outputs (the classifiers' fprop): a sum of K = taps * cin products, (K + 1) u |terms|.
- Dense wgrad.  k_igemm_wgrad splits the output pixels into `splits` ranges of `pps` pixels (64-pixel boxes,
  _wgrad_plan restates wgrad_ws_elems and choose_box of csrc/igemm_tc.cu).  Within a range one CTA accumulates every
  weight in fp32, in pixel order: at most pps roundings of a partial sum no larger than |terms|.  k_splitk_reduce
  then adds the `splits` fp32 partials in split order: splits more roundings.  In all,
  |err| <= (pps + splits) u |terms|.  The CUDA-core wgrad (k_simt_wgrad, the 10-unit WRN classifier) has the same
  form, with 2048-pixel chunks combined by fp32 atomics.  Whether wgmma rounds its fp32 accumulator to nearest or
  toward zero is not documented; either way each addition errs by at most one fp32 ulp of the partial sum, which
  would double the worst case.  The measured error stays within the nearest-rounding bound used here, with a wide
  margin (at most 5 % of it on an H100 SXM at 700 W), because the worst case needs every rounding to err in the
  same direction by its full amount.
- Depthwise wgrad (k_depthwise3x3_wgrad): each thread adds `terms` = rows per CTA * columns per lane products in
  fp32, the column lanes are added in fp32, the CTA partials in fp64, and the result is rounded to fp32 once (and
  added to the old value when beta = 1): (terms + lanes + 2) u |terms| (_dw_wgrad_plan restates dw_wgrad_blocks).
x and dy have a nonzero mean (0.75 +- 0.5 and 0.5 +- 0.5), so |terms| of a wgrad is within a small factor of
|result| and the wgrad bounds are not vacuous.

Every bound has a control that must fail: the same check against a reference that drops one tap (3x3) or one input
channel (1x1 and linear) for fprop / dgrad, one split's pixel range for the dense wgrad, and one CTA's output rows
for the depthwise wgrad.  Each case prints its max(err / bound) per kernel class (`headroom` lines, pytest -s).
"""
import pytest
import torch

from isolated import assert_not_ran, assert_ran, run_isolated
from test_streaming_b256_gpu import DEV, _bf16_tol, _bn_case, _fill

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
REF_ELEMS = 1 << 23          # elements per float64 temporary of the references (64 MB)
CONFIGS = {'mbv1': ('random', 0.9, 256, 224), 'wrn': ('erdos_renyi_kernel', 0.95, 128, 32)}
X_MEAN, X_SD, DY_MEAN, DY_SD = 0.75, 0.5, 0.5, 0.5
_TABLES = {}


def _lib():
  from rigl_b200 import _cabi
  return _cabi


# ---------------------------------------------------------------------------------------------------------------
# Layer tables
# ---------------------------------------------------------------------------------------------------------------

def _layer_table(name):
  """{'layers': distinct masked conv / linear layers, 'depthwise': distinct depthwise layers, 'bn': distinct
  (rows, channels) of the BNs} of the benchmark model `name`, at its batch size.  Layer entries are dicts with the
  module and its input extent; the model is built and masked once per process."""
  if name in _TABLES:
    return _TABLES[name]
  from rigl_b200 import workloads
  from rigl_b200.layers import SparseConv2d, SparseLinear
  from rigl_b200.norm import FusedBatchNormReLU
  method, sparsity, batch, hw = CONFIGS[name]
  torch.manual_seed(0)
  model = workloads.MobileNetV1(num_classes=1000, device=DEV) if name == 'mbv1' else \
      workloads.WideResNet(depth=22, width=2, num_classes=10, device=DEV)
  workloads.init_masks(model, method, sparsity, seed=0)
  table = {'model': model, 'batch': batch, 'layers': [], 'depthwise': [], 'bn': []}
  seen = set()

  def hook(mod, args):
    x = args[0]
    if isinstance(mod, SparseConv2d):
      key = ('conv', mod.in_channels, mod.out_channels, mod.ksize, mod.stride, mod.padding) + tuple(x.shape[2:])
      entry = dict(layer=mod, kind='conv', h=int(x.shape[2]), w=int(x.shape[3]))
    elif isinstance(mod, SparseLinear):
      key = ('linear', mod.in_channels, mod.out_channels)
      entry = dict(layer=mod, kind='linear', h=1, w=1)
    elif isinstance(mod, workloads.DepthwiseConv2d):
      key = ('depthwise', mod.channels, mod.stride) + tuple(x.shape[2:])
      entry = dict(layer=mod, kind='depthwise', h=int(x.shape[2]), w=int(x.shape[3]))
    else:
      assert mod.relu, 'WRN batch norms are BN + ReLU'
      key = ('bn', batch * x.shape[2] * x.shape[3], mod.channels)
      entry = key[1:]
    if key not in seen:
      seen.add(key)
      table['bn' if key[0] == 'bn' else 'depthwise' if key[0] == 'depthwise' else 'layers'].append(entry)

  kinds = (SparseConv2d, SparseLinear, workloads.DepthwiseConv2d) + ((FusedBatchNormReLU,) if name == 'wrn' else ())
  handles = [m.register_forward_pre_hook(hook) for m in model.modules() if isinstance(m, kinds)]
  model.eval()
  try:
    with torch.no_grad():
      model(torch.zeros((1, 3, hw, hw), device=DEV))
  finally:
    for h in handles:
      h.remove()
    model.train()
  torch.cuda.synchronize()
  _TABLES[name] = table
  return table


def _geom(entry, batch):
  """(n, h, w, cin, cout, k, stride, pad_before, oh, ow) of a masked layer at the benchmark batch."""
  l = entry['layer']
  if entry['kind'] == 'linear':
    return batch, 1, 1, l.in_channels, l.out_channels, 1, 1, 0, 1, 1
  oh, pad = l.out_size(entry['h'])
  ow, _ = l.out_size(entry['w'])
  return batch, entry['h'], entry['w'], l.in_channels, l.out_channels, l.ksize, l.stride, pad, oh, ow


def _shape_id(entry, batch):
  n, h, w, cin, cout, k, s, _, _, _ = _geom(entry, batch)
  if entry['kind'] == 'linear':
    return '%s %dx%d->%d' % (entry['layer'].scope, n, cin, cout)
  return '%s %dx%dx%dx%d k%ds%d %s ->%d' % (entry['layer'].scope, n, h, w, cin, k, s, entry['layer'].padding, cout)


# ---------------------------------------------------------------------------------------------------------------
# Launch rules, restated from the launchers
# ---------------------------------------------------------------------------------------------------------------

def _choose_box(gw, gh, nb, total):
  """csrc/igemm_tc.cu choose_box: the power-of-two box bw * bh * bn == total with the least padding of the
  gw x gh x nb pixel grid, then the longest contiguous runs."""
  best = None
  w = 1
  while w <= total:
    h = 1
    while w * h <= total:
      n = total // (w * h)
      padded = (-(-gw // w) * w) * (-(-gh // h) * h) * (-(-nb // n) * n)
      score = padded * 1024 - w * 16 - h
      if best is None or score < best[0]:
        best = (score, w, h, n)
      h *= 2
    w *= 2
  return best[1:]


def _tc_supported(cin, cout):
  """csrc/igemm_tc.cu tc_supported for the layers here (stride 1 / 2, <= 9 taps): 16-byte row pitches."""
  return cin % 8 == 0 and cout % 8 == 0


def _wgrad_plan(n, oh, ow, taps, cin, cout, pitch=None):
  """The summation structure of the dense wgrad: pixels per split (`pps`), the number of splits, and the pixel
  box order that maps pixel blocks to splits.  Tensor cores: wgrad_ws_elems -- splits = ceil(2 SMs / output
  tiles), at most one per 64-pixel block, then evened out.  CUDA cores (simt_wgrad): 2048-pixel chunks in
  flattened (n, oh, ow) order, one fp32 atomic add each.  The wgrad's tensor-core test reads the row pitch of x,
  not cin: `pitch` is that of a padded operand (a patch matrix's [rows, kpitch]), None for x's own cin."""
  if not _tc_supported(cin if pitch is None else pitch, cout):
    chunk = 2048
    while -(-n * oh * ow // chunk) > 65535:
      chunk *= 2
    return dict(kernel='simt', bw=1, bh=1, bn=1, tiles_w=ow, tiles_h=oh, bps=chunk,
                pps=min(chunk, n * oh * ow), splits=-(-n * oh * ow // chunk))
  bw, bh, bn = _choose_box(ow, oh, n, 64)
  tiles_w, tiles_h, tiles_n = -(-ow // bw), -(-oh // bh), -(-n // bn)
  pblocks = tiles_w * tiles_h * tiles_n
  bn_tile = 128 if cout >= 128 else 64
  out_tiles = taps * -(-cin // 128) * -(-cout // bn_tile)
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  splits = max(1, min(-(-2 * sms // out_tiles), pblocks))
  bps = -(-pblocks // splits)
  splits = -(-pblocks // bps)
  return dict(kernel='tc', bw=bw, bh=bh, bn=bn, tiles_w=tiles_w, tiles_h=tiles_h, bps=bps, pps=bps * 64,
              splits=splits)


def _first_split(plan, a, b, oh, ow):
  """bool [b - a, oh, ow]: the output pixels of images [a, b) that the first split (pixel blocks [0, bps)) adds."""
  n = torch.arange(a, b, device=DEV)[:, None, None]
  h = torch.arange(oh, device=DEV)[None, :, None]
  w = torch.arange(ow, device=DEV)[None, None, :]
  pb = w // plan['bw'] + plan['tiles_w'] * (h // plan['bh'] + plan['tiles_h'] * (n // plan['bn']))
  return pb < plan['bps']


def _halo_eligible(k, s, pad, h, w, oh, ow, kred):
  """csrc/halo3x3.cuh halo_geom, without its shared-memory fit: 3x3 / stride 1 / pad 1, <= 64 reduction channels,
  and a row pitch (W + 2 rounded up to a power of two >= 8) of at most 128 of which >= 75 % is useful (W * 4 >= Wp
  * 3)."""
  if k != 3 or s != 1 or pad != 1 or (h, w) != (oh, ow) or kred > 64 or kred % 8:
    return False
  wp = 8
  while wp < w + 2:
    wp *= 2
  return wp <= 128 and w * 4 >= wp * 3


def _dw_wgrad_plan(n, oh, ow, c):
  """csrc/depthwise.cu dw_wgrad_blocks and the k_depthwise3x3_wgrad block shape: output rows (n, oh) per CTA,
  CTAs, column lanes, and the products one thread adds per weight."""
  rows = n * oh
  v = c // 8
  bx = min(v, 32)
  groups = -(-v // bx)
  target = max(1, min(-(-132 * 4 // groups), rows))     # kNumSmsHint = 132: ~4 CTAs per SM
  rpb = -(-rows // target)
  lanes = 256 // bx
  return dict(rpb=rpb, ctas=-(-rows // rpb), lanes=lanes, terms=rpb * -(-ow // lanes))


# ---------------------------------------------------------------------------------------------------------------
# Checks
# ---------------------------------------------------------------------------------------------------------------

def _ratio(got, want, tol):
  return float(((got.double() - want).abs() / tol).max())


def _bf16_ratio(got, want, cancelled):
  """max(err / bound) of a bf16 output chunk under test_streaming_b256_gpu._close_bf16's bound."""
  return _ratio(got, want, _bf16_tol(want, cancelled))


def _report(cls, shape, ratio):
  print('headroom %-34s %-52s %.4f' % (cls, shape, ratio))


def _nhwc(t):
  return t.permute(0, 2, 3, 1) if t.dim() == 4 else t[:, None, None, :]


def _taps(xp, k, s, oh, ow):
  """(tap, x at the tap's offset for every output pixel) of a padded NHWC chunk."""
  for kh in range(k):
    for kw in range(k):
      yield kh * k + kw, kh, kw, xp[:, kh:kh + s * (oh - 1) + 1:s, kw:kw + s * (ow - 1) + 1:s, :]


def _activation(n, h, w, c, mean, sd, gen):
  """bf16 [n, c, h, w] in channels_last memory (a view of NHWC storage)."""
  return _fill(n * h * w, c, mean, sd, gen).view(n, h, w, c).permute(0, 3, 1, 2)


def _run_layer(name, i):
  """The masked layer i of model `name` at the benchmark batch: fprop, then dgrad and dense wgrad (beta = 0) through
  the layer's autograd function.  Returns (entry, x, dy, y, dx, dense wgrad, weight.grad)."""
  table = _layer_table(name)
  entry, batch = table['layers'][i], table['batch']
  layer = entry['layer']
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, batch)
  gen = torch.Generator(device=DEV)
  gen.manual_seed(1000 * i + cin + cout)
  if entry['kind'] == 'linear':
    x = _fill(n, cin, X_MEAN, X_SD, gen)
    dy = _fill(n, cout, DY_MEAN, DY_SD, gen).to(layer.out_dtype)      # (bf16 values: exact in either type)
  else:
    x = _activation(n, h, w, cin, X_MEAN, X_SD, gen)
    dy = _activation(n, oh, ow, cout, DY_MEAN, DY_SD, gen)
  x = x.detach().requires_grad_(True)
  layer.masked_weights.fresh = False
  layer.weight.grad = None
  y = layer(x)
  assert tuple(y.shape) == tuple(dy.shape), (tuple(y.shape), tuple(dy.shape))
  y.backward(dy)
  torch.cuda.synchronize()
  return entry, x.detach(), dy, y.detach(), x.grad, layer.masked_weights.dense_grad, layer.weight.grad


def _float64_layer(layer, geom, first, xs, dys, epilogue, dgrad=True):
  """The float64 references of a masked layer with geometry `geom` (_geom), per tap as DGEMMs over chunks of whole
  images, on the bf16-rounded masked weights (the packed operand).  xs, dys: the NHWC input and output gradient.

  For every chunk of images [a, b) it calls epilogue(a, b, yr, ya, ydrop, dxr, dxa, dxdrop): the NHWC fprop
  reference, its |terms| and its control part, then the same three for dgrad (None with dgrad=False).  The control
  part is the centre tap of a 3x3, else the input channel with the most surviving weights (fprop: an x channel;
  dgrad: a dy channel).  first(a, b): bool [b - a, oh, ow], the output pixels of those images that the wgrad's
  first split adds (_first_split).  Returns (dw, |terms| of dw, the first split's share of dw), each
  [taps, cin, cout]."""
  n, h, w, cin, cout, k, s, pad, oh, ow = geom
  taps = k * k
  mask = layer.mask.to_dense().view(taps, cin, cout).double()
  wm = (layer.weight.detach().view(taps, cin, cout) * mask).to(torch.bfloat16).double()     # the packed operand
  wa = wm.abs()
  ph = max(0, (oh - 1) * s + k - h - pad)
  pw = max(0, (ow - 1) * s + k - w - pad)
  ctap = taps // 2
  ci = int(mask.sum((0, 2)).argmax())
  co = int(mask.sum((0, 1)).argmax())
  dw = torch.zeros((taps, cin, cout), dtype=torch.float64, device=DEV)
  dw_abs, dw_first = torch.zeros_like(dw), torch.zeros_like(dw)
  step = max(1, REF_ELEMS // max(h * w * cin, oh * ow * cout))
  for a in range(0, n, step):
    b = min(a + step, n)
    xp = torch.nn.functional.pad(xs[a:b].double(), (0, 0, pad, pw, pad, ph))
    g = dys[a:b].double()
    ga = g.abs()
    f = first(a, b)
    g_first = g * f[..., None] if bool(f.any()) else None
    yr = torch.zeros((b - a, oh, ow, cout), dtype=torch.float64, device=DEV)
    ya, ydrop = torch.zeros_like(yr), torch.zeros_like(yr)
    dxp = dxa = dxdrop = None
    if dgrad:
      dxp = torch.zeros_like(xp)
      dxa, dxdrop = torch.zeros_like(xp), torch.zeros_like(xp)
    for t, kh, kw, xt in _taps(xp, k, s, oh, ow):
      xt = xt.reshape(-1, cin)
      gt = g.reshape(-1, cout)
      yt = (xt @ wm[t]).view_as(yr)
      yr += yt
      ya += (xt.abs() @ wa[t]).view_as(yr)
      if k == 1:
        ydrop += (xt[:, ci:ci + 1] @ wm[t, ci:ci + 1]).view_as(yr)
      elif t == ctap:
        ydrop += yt
      del yt
      if dgrad:
        sl = (slice(None), slice(kh, kh + s * (oh - 1) + 1, s), slice(kw, kw + s * (ow - 1) + 1, s))
        dxt = (gt @ wm[t].T).view(b - a, oh, ow, cin)
        dxp[sl] += dxt
        dxa[sl] += (ga.reshape(-1, cout) @ wa[t].T).view(b - a, oh, ow, cin)
        if k == 1:
          dxdrop[sl] += (gt[:, co:co + 1] @ wm[t][:, co:co + 1].T).view(b - a, oh, ow, cin)
        elif t == ctap:
          dxdrop[sl] += dxt
        del dxt
      dw[t] += xt.T @ gt
      dw_abs[t] += xt.abs().T @ ga.reshape(-1, cout)
      if g_first is not None:
        dw_first[t] += xt.T @ g_first.reshape(-1, cout)
    del xp, g, ga, g_first
    if dgrad:
      crop = (slice(None), slice(pad, pad + h), slice(pad, pad + w))
      dxp, dxa, dxdrop = dxp[crop], dxa[crop], dxdrop[crop]
    epilogue(a, b, yr, ya, ydrop, dxp, dxa, dxdrop)
    del yr, ya, ydrop, dxp, dxa, dxdrop
  return dw, dw_abs, dw_first


def _layer_case(name, i):
  torch.cuda.reset_peak_memory_stats()
  table = _layer_table(name)
  entry, x, dy, y, dx, dense, masked = _run_layer(name, i)
  batch = table['batch']
  layer = entry['layer']
  geom = n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, batch)
  taps = k * k
  shape = _shape_id(entry, batch)
  mask = layer.mask.to_dense().view(taps, cin, cout).double()
  plan = _wgrad_plan(n, oh, ow, taps, cin, cout)
  xs, dys, ys, dxs = _nhwc(x), _nhwc(dy), _nhwc(y), _nhwc(dx)
  f32_out = y.dtype == torch.float32
  r = dict(y=0.0, dx=0.0, ctl_y=False, ctl_dx=False)

  def check(a, b, yr, ya, ydrop, dxr, dxa, dxdrop):
    if f32_out:            # the classifiers: fp32 output, a sum of taps * cin products
      tol = (taps * cin + 1) * U * ya + 1e-300
      r['y'] = max(r['y'], _ratio(ys[a:b], yr, tol))
      r['ctl_y'] = r['ctl_y'] or _ratio(ys[a:b], yr - ydrop, tol) > 1
    else:
      r['y'] = max(r['y'], _bf16_ratio(ys[a:b], yr, ya))
      r['ctl_y'] = r['ctl_y'] or _bf16_ratio(ys[a:b], yr - ydrop, ya) > 1
    r['dx'] = max(r['dx'], _bf16_ratio(dxs[a:b], dxr, dxa))
    r['ctl_dx'] = r['ctl_dx'] or _bf16_ratio(dxs[a:b], dxr - dxdrop, dxa) > 1

  dw, dw_abs, dw_first = _float64_layer(layer, geom, lambda a, b: _first_split(plan, a, b, oh, ow), xs, dys, check)
  r_y, r_dx, ctl_y, ctl_dx = r['y'], r['dx'], r['ctl_y'], r['ctl_dx']
  kern = 'simt' if not _tc_supported(cin, cout) else 'igemm'
  _report('%s fprop (%s)' % (kern, 'fp32' if f32_out else 'bf16'), shape, r_y)
  _report('%s dgrad (bf16)' % kern, shape, r_dx)
  assert r_y <= 1, '%s: fprop off by %.3g bounds' % (shape, r_y)
  assert r_dx <= 1, '%s: dgrad off by %.3g bounds' % (shape, r_dx)
  assert ctl_y, '%s: fprop control (%s dropped) passes the bound' % (shape, 'centre tap' if k > 1 else 'channel')
  assert ctl_dx, '%s: dgrad control (%s dropped) passes the bound' % (shape, 'centre tap' if k > 1 else 'channel')

  # dense wgrad: every position, masked-out ones included (RigL's grow scores)
  got = dense.view(taps, cin, cout)
  wtol = (plan['pps'] + plan['splits']) * U * dw_abs + 1e-300
  r_w = _ratio(got, dw, wtol)
  _report('%s wgrad (pps %d, %d splits)' % (plan['kernel'], plan['pps'], plan['splits']), shape, r_w)
  assert r_w <= 1, '%s: dense wgrad off by %.3g bounds (pps %d, splits %d)' % (shape, r_w, plan['pps'],
                                                                               plan['splits'])
  assert _ratio(got, dw - dw_first, wtol) > 1, '%s: wgrad control (first split left out) passes' % shape
  # mask * wgrad: the masked gradient is the dense one where the mask is set, exactly, and zero elsewhere
  assert torch.equal(masked.reshape(-1), (dense * mask.reshape(-1).float())), '%s: mask * wgrad' % shape
  print('peak %s %.0f MB' % (shape, torch.cuda.max_memory_allocated() / 2 ** 20))
  del entry, x, dy, y, dx, dw, dw_abs, dw_first
  layer.weight.grad = None
  torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# Native depthwise 3x3
# ---------------------------------------------------------------------------------------------------------------

def _run_depthwise(i):
  """Depthwise layer i of MobileNet-v1 at batch 256 through the C entry points: fprop, dgrad, the weight gradient
  with beta = 0 and with beta = 1 onto `old`.  Returns (entry, x, dy, weight, y, dx, dw, old, dw_beta1) (NHWC)."""
  cabi = _lib()
  lib = cabi.lib()
  table = _layer_table('mbv1')
  entry, n = table['depthwise'][i], table['batch']
  mod = entry['layer']
  h, w, c, s = entry['h'], entry['w'], mod.channels, mod.stride
  oh, ow = (h - 1) // s + 1, (w - 1) // s + 1
  gen = torch.Generator(device=DEV)
  gen.manual_seed(77 + i)
  x = _fill(n * h * w, c, X_MEAN, X_SD, gen).view(n, h, w, c)
  dy = _fill(n * oh * ow, c, DY_MEAN, DY_SD, gen).view(n, oh, ow, c)
  wt = mod.weight.detach().contiguous()
  y = torch.empty((n, oh, ow, c), dtype=torch.bfloat16, device=DEV)
  dx = torch.empty_like(x)
  dw = torch.empty((c, 9), dtype=torch.float32, device=DEV)
  old = torch.randn((c, 9), generator=gen, device=DEV)
  dw1 = old.clone()
  ws = torch.empty(lib.rigl_depthwise3x3_workspace_bytes(n, h, w, c, s), dtype=torch.uint8, device=DEV)
  st = cabi.stream_ptr()
  cabi.check(lib.rigl_depthwise3x3_fprop(x.data_ptr(), wt.data_ptr(), n, h, w, c, s, y.data_ptr(), st), 'fprop')
  cabi.check(lib.rigl_depthwise3x3_dgrad(dy.data_ptr(), wt.data_ptr(), n, h, w, c, s, dx.data_ptr(), st), 'dgrad')
  for out, beta in ((dw, 0.0), (dw1, 1.0)):
    cabi.check(lib.rigl_depthwise3x3_wgrad(x.data_ptr(), dy.data_ptr(), n, h, w, c, s, out.data_ptr(), beta,
                                           ws.data_ptr(), ws.numel(), st), 'wgrad')
  torch.cuda.synchronize()
  return entry, x, dy, wt, y, dx, dw, old, dw1


def _depthwise_case(i):
  torch.cuda.reset_peak_memory_stats()
  entry, x, dy, wt, y, dx, dw, old, dw1 = _run_depthwise(i)
  n, h, w, c = x.shape
  _, oh, ow, _ = dy.shape
  s = entry['layer'].stride
  shape = 'depthwise %dx%dx%dx%d s%d' % (n, h, w, c, s)
  # beta = 1 adds the new sum to the old value in fp32, which is what the finalize computes: bit for bit
  assert torch.equal(dw1, old + dw), '%s: beta = 1 is not old + result(beta = 0)' % shape
  plan = _dw_wgrad_plan(n, oh, ow, c)
  w64 = wt.view(c, 9).to(torch.bfloat16).double()     # the kernels round the fp32 weights to bf16 on load
  wa = w64.abs()
  ref = torch.zeros((9, c), dtype=torch.float64, device=DEV)
  ref_abs, ref_cta = torch.zeros_like(ref), torch.zeros_like(ref)
  r_y = r_dx = 0.0
  ctl_y = ctl_dx = False
  step = max(1, REF_ELEMS // (h * w * c))
  for a in range(0, n, step):
    b = min(a + step, n)
    xp = torch.nn.functional.pad(x[a:b].double(), (0, 0, 1, 1, 1, 1))
    g = dy[a:b].double()
    rows = torch.arange(a, b, device=DEV)[:, None] * oh + torch.arange(oh, device=DEV)[None, :]
    cta0 = (rows < plan['rpb'])[:, :, None, None]                    # output rows of the first CTA
    yr = torch.zeros_like(g)
    ya, ydrop = torch.zeros_like(g), torch.zeros_like(g)
    dxp = torch.zeros_like(xp)
    dxa, dxdrop = torch.zeros_like(xp), torch.zeros_like(xp)
    for t, kh, kw, xt in _taps(xp, 3, s, oh, ow):
      yr += xt * w64[:, t]
      ya += xt.abs() * wa[:, t]
      sl = (slice(None), slice(kh, kh + s * (oh - 1) + 1, s), slice(kw, kw + s * (ow - 1) + 1, s))
      dxp[sl] += g * w64[:, t]
      dxa[sl] += g.abs() * wa[:, t]
      if t == 4:
        ydrop += xt * w64[:, t]
        dxdrop[sl] += g * w64[:, t]
      ref[t] += (xt * g).sum((0, 1, 2))
      ref_abs[t] += (xt * g).abs().sum((0, 1, 2))
      if a * oh < plan['rpb']:
        ref_cta[t] += (xt * g * cta0).sum((0, 1, 2))
    del xp, g
    crop = (slice(None), slice(1, 1 + h), slice(1, 1 + w))
    dxr, dxa, dxdrop = dxp[crop], dxa[crop], dxdrop[crop]
    r_y = max(r_y, _bf16_ratio(y[a:b], yr, ya))
    ctl_y = ctl_y or _bf16_ratio(y[a:b], yr - ydrop, ya) > 1
    r_dx = max(r_dx, _bf16_ratio(dx[a:b], dxr, dxa))
    ctl_dx = ctl_dx or _bf16_ratio(dx[a:b], dxr - dxdrop, dxa) > 1
    del yr, ya, ydrop, dxp, dxr, dxa, dxdrop
  _report('depthwise fprop (bf16)', shape, r_y)
  _report('depthwise dgrad (bf16)', shape, r_dx)
  assert r_y <= 1 and r_dx <= 1, '%s: fprop / dgrad off by %.3g / %.3g bounds' % (shape, r_y, r_dx)
  assert ctl_y and ctl_dx, '%s: fprop / dgrad control (centre tap dropped) passes the bound' % shape
  got = dw.T                                          # [c][9] -> [tap][c]
  tol = (plan['terms'] + plan['lanes'] + 2) * U * ref_abs + 1e-300
  r_w = _ratio(got, ref, tol)
  _report('depthwise wgrad (%d terms, %d lanes)' % (plan['terms'], plan['lanes']), shape, r_w)
  assert r_w <= 1, '%s: wgrad off by %.3g bounds' % (shape, r_w)
  assert _ratio(got, ref - ref_cta, tol) > 1, '%s: wgrad control (first CTA left out) passes' % shape
  print('peak %s %.0f MB' % (shape, torch.cuda.max_memory_allocated() / 2 ** 20))
  del entry, x, dy, y, dx
  torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------------
# Tests
# ---------------------------------------------------------------------------------------------------------------

# (model, index into its table of distinct masked layers): MobileNet-v1's 9 pointwise shapes and final_dense, WRN's
# 9 conv shapes and logits
_LAYER_CASES = [('mbv1', i) for i in range(10)] + [('wrn', i) for i in range(10)]


def test_layer_tables_match_the_models():
  """The distinct shapes the benchmark runs, counted, so a model change cannot silently shrink the coverage; and
  where the launch rules send them."""
  mb, wrn = _layer_table('mbv1'), _layer_table('wrn')
  conv = lambda t: [e for e in t['layers'] if e['kind'] == 'conv']
  lin = lambda t: [(e['layer'].in_channels, e['layer'].out_channels) for e in t['layers'] if e['kind'] == 'linear']
  assert len(conv(mb)) == 9 and all(e['layer'].ksize == 1 for e in conv(mb))
  assert lin(mb) == [(1024, 1000)] and mb['layers'][-1]['kind'] == 'linear'
  assert len(mb['depthwise']) == 9
  assert len(conv(wrn)) == 9
  assert sorted(e['layer'].ksize for e in conv(wrn)) == [1] * 3 + [3] * 6
  assert lin(wrn) == [(128, 10)] and wrn['layers'][-1]['kind'] == 'linear'
  assert sorted(wrn['bn']) == [(8192, 128), (32768, 64), (131072, 16), (131072, 32)]
  assert len(mb['layers']) + len(wrn['layers']) == len(_LAYER_CASES)
  for e in conv(wrn):
    n, h, w, cin, cout, k, s, pad, oh, ow = _geom(e, wrn['batch'])
    # WRN's 3x3 layers are at most 64 channels wide but 32 / 16 / 8 pixels: never the halo kernels
    assert not _halo_eligible(k, s, pad, h, w, oh, ow, cin) and not _halo_eligible(k, s, pad, h, w, oh, ow, cout)
  # the first pointwise conv of MobileNet-v1 (112^2, 32 -> 64) is one output tile: a few hundred wgrad splits
  n, h, w, cin, cout, k, s, pad, oh, ow = _geom(conv(mb)[0], mb['batch'])
  assert (h, cin, cout) == (112, 32, 64) and _wgrad_plan(n, oh, ow, 1, cin, cout)['splits'] > 200


@pytest.mark.parametrize('name,i', _LAYER_CASES, ids=['%s-layer%d' % c for c in _LAYER_CASES])
def test_masked_layer_at_bench_size_against_float64(name, i):
  _layer_case(name, i)


@pytest.mark.parametrize('i', range(9), ids=['mbv1-depthwise%d' % i for i in range(9)])
def test_native_depthwise_b256_against_float64(i):
  _depthwise_case(i)


@pytest.mark.parametrize('i', range(4), ids=['wrn-bn%d' % i for i in range(4)])
def test_wrn_bn_against_float64(i):
  rows, c = sorted(_layer_table('wrn')['bn'])[i]
  _bn_case(rows, c, 'relu')


def test_wrn_bn_on_the_three_kernel_path():
  calls = [('_bn_case', (rows, c, 'relu')) for rows, c in sorted(_layer_table('wrn')['bn'])]
  torch.cuda.empty_cache()
  for (fn, args), ran in zip(calls, run_isolated('test_streaming_b256_gpu', calls, {'RIGL_BN_FUSED': '0'})):
    assert_not_ran(ran, r'k_bn_(fwd|bwd)_fused', args)      # (each call asserts its path by launch count)


@pytest.mark.parametrize('name', ['mbv1', 'wrn'])
def test_bench_layers_run_their_kernels(name):
  """Which kernels the benchmark's layers launch at full size, in a fresh process (the first call builds the table:
  its batch-1 forward is not witnessed).  fprop and dgrad both launch k_igemm_kmajor; with no CUDA-core or halo
  kernel in the list, neither took another path."""
  table = _layer_table(name)
  calls = [('_layer_table', (name,))] + [('_run_layer', (name, i)) for i in range(len(table['layers']))]
  if name == 'mbv1':
    calls += [('_run_depthwise', (i,)) for i in range(len(table['depthwise']))]
  torch.cuda.empty_cache()
  ran = run_isolated('test_bench_c4_c5_gpu', calls, timeout=600)[1:]
  for i, names in enumerate(ran[:len(table['layers'])]):
    entry = table['layers'][i]
    n, h, w, cin, cout, k, s, pad, oh, ow = _geom(entry, table['batch'])
    what = _shape_id(entry, table['batch'])
    if not _tc_supported(cin, cout):
      # WRN's 10-unit classifier: cout % 8 != 0 has no 16-byte row pitch for TMA, so all three run on CUDA cores
      assert (name, cout) == ('wrn', 10), what
      for kern in ('k_simt_fprop', 'k_simt_dgrad', 'k_simt_wgrad'):
        assert_ran(names, kern, what)
      assert_not_ran(names, r'k_igemm', what)
      continue
    assert_ran(names, r'k_igemm_kmajor<', what)
    assert_ran(names, r'k_igemm_wgrad<', what)
    if _wgrad_plan(n, oh, ow, k * k, cin, cout)['splits'] > 1:
      assert_ran(names, r'k_splitk_reduce', what)
    assert_not_ran(names, r'k_simt_', what)
    assert_not_ran(names, r'k_halo3x3', what)
  for i, names in enumerate(ran[len(table['layers']):]):
    what = 'depthwise %d' % i
    assert_ran(names, r'k_depthwise3x3<false>', what)
    assert_ran(names, r'k_depthwise3x3<true>', what)
    assert_ran(names, r'k_depthwise3x3_wgrad\b', what)
    assert_ran(names, r'k_depthwise3x3_wgrad_finalize', what)
