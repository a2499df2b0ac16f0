"""Evaluation on the H100: the conv epilogue's inference batch norm (rigl_masked_conv2d_fprop_bnapply) against
rigl_masked_conv2d_fprop + rigl_bn_apply bit for bit, eval logits with and without the fusion, the metrics against a
numpy restatement, and an evaluation leaving the training state untouched."""
import tempfile

import numpy as np
import pytest
import torch

from rigl_b200 import _cabi, checkpoint, layers, pruning, workloads
from rigl_b200.evaluate import Evaluator
from rigl_b200.layers import SparseConv2d, _workspace
from rigl_b200.norm import FusedBatchNormReLU

from isolated import assert_not_ran, assert_ran
from tile_masks import tile_mask

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
_BN_KERNEL = r'k_igemm_kmajor_bn<'


def _act(n, c, h, w, gen):
  return torch.randn(n, c, h, w, device=DEV, generator=gen).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)


def _coef(c, gen):
  scale = torch.rand(c, device=DEV, generator=gen) * 1.5 + 0.25
  scale[::5] *= -1
  shift = torch.randn(c, device=DEV, generator=gen)
  return scale, shift


def _compare(cin, cout, k, stride, h, batch=2, residual=False, relu=True, pattern=None, seed=0):
  """(rc of the fused call, fused output, conv + rigl_bn_apply output) of one layer."""
  gen = torch.Generator(device=DEV).manual_seed(seed)
  layer = SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', device=DEV, registry=pruning.MaskedLayerRegistry())
  if pattern is not None:
    layer.mask.assign(tile_mask(pattern, tuple(layer.weight.shape), np.random.RandomState(seed)))
  layer.pack()
  x = _act(batch, cin, h, h, gen)
  d = layer._desc(batch, h, h)
  scale, shift = _coef(cout, gen)
  res = _act(batch, cout, d.out_h, d.out_w, gen) if residual else None
  shape = (batch, cout, d.out_h, d.out_w)
  y = torch.empty(shape, dtype=torch.bfloat16, device=DEV, memory_format=torch.channels_last)
  ref = torch.empty_like(y)
  out = torch.full_like(y, float('nan'))
  ws = _workspace(x.device, _cabi.lib().rigl_conv_workspace_bytes(d))
  lib, st = _cabi.lib(), _cabi.stream_ptr()
  _cabi.check(lib.rigl_masked_conv2d_fprop(d, x.data_ptr(), layer.packed.data_ptr(), y.data_ptr(), None, None,
                                           ws.data_ptr(), ws.numel(), st), 'fprop')
  _cabi.check(lib.rigl_bn_apply(y.data_ptr(), None if res is None else res.data_ptr(), scale.data_ptr(),
                                shift.data_ptr(), batch * d.out_h * d.out_w, cout, int(relu), ref.data_ptr(), st),
              'bn_apply')
  rc = lib.rigl_masked_conv2d_fprop_bnapply(d, x.data_ptr(), layer.packed.data_ptr(),
                                            None if res is None else res.data_ptr(), scale.data_ptr(),
                                            shift.data_ptr(), int(relu), out.data_ptr(), ws.data_ptr(), ws.numel(), st)
  torch.cuda.synchronize()
  return rc, out, ref


def _model_conv_shapes(model, size, batch=1):
  """(cin, cout, k, stride, input extent) of every distinct SparseConv2d of `model` in an eval forward."""
  shapes = set()
  hooks = [m.register_forward_hook(lambda m, i, o: shapes.add((m.in_channels, m.out_channels, m.ksize, m.stride,
                                                               i[0].shape[-1])))
           for m in model.modules() if isinstance(m, SparseConv2d)]
  model.eval()
  with torch.no_grad():
    model(torch.randn(batch, 3, size, size, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
  for hk in hooks:
    hk.remove()
  return sorted(shapes)


_SHAPES = {}


def _shapes():
  if not _SHAPES:
    torch.manual_seed(0)
    for name, mk in (('resnet50', workloads.ResNet50), ('mobilenet_v1', workloads.MobileNetV1),
                     ('mobilenet_v2', workloads.MobileNetV2)):
      _SHAPES[name] = _model_conv_shapes(mk(device=DEV), 96)
  return _SHAPES


@pytest.mark.parametrize('model', ['resnet50', 'mobilenet_v1', 'mobilenet_v2'])
def test_bnapply_matches_conv_then_bn_apply_on_every_model_shape(model):
  n_fused = 0
  for i, (cin, cout, k, s, h) in enumerate(_shapes()[model]):
    for residual, relu in ((False, True), (True, True), (True, False), (False, False)):
      rc, out, ref = _compare(cin, cout, k, s, h, residual=residual, relu=relu, seed=i)
      case = (cin, cout, k, s, h, residual, relu)
      if rc == -4:          # the stem (CUDA-core / patch-matrix path) and the 3x3 layers of the halo kernels
        assert cin % 8 or (k == 3 and s == 1 and b'halo' in _cabi.lib().rigl_last_error()), case
        continue
      assert rc == 0, (case, _cabi.lib().rigl_last_error())
      assert torch.equal(out, ref), case
      n_fused += 1
  assert n_fused >= 8


@pytest.mark.parametrize('cin,cout,k,stride,h,batch', [
    (64, 24, 1, 1, 9, 3),        # ragged: one slab of 24 channels, partial pixel boxes
    (96, 144, 1, 1, 7, 2),       # ragged second slab of a 128-wide tile
    (160, 320, 1, 1, 5, 1),
    (128, 200, 3, 2, 11, 2),     # 3x3/2 through the parity maps, ragged last N tile
    (256, 72, 3, 1, 6, 1),
])
def test_bnapply_ragged_channels_and_partial_boxes(cin, cout, k, stride, h, batch):
  for residual in (False, True):
    rc, out, ref = _compare(cin, cout, k, stride, h, batch=batch, residual=residual)
    assert rc == 0, _cabi.lib().rigl_last_error()
    assert torch.equal(out, ref)


@pytest.mark.parametrize('pattern', ['staircase', 'block0', 'half', 'dead_taps', 'corner', 'dead'])
def test_bnapply_dead_weight_tiles(pattern):
  rc, out, ref = _compare(192, 256, 3, 1, 8, residual=True, pattern=pattern)
  assert rc == 0
  assert torch.equal(out, ref)


def test_bnapply_unsupported_shapes_launch_nothing():
  lib = _cabi.lib()
  rc, _, _ = _compare(64, 64, 3, 1, 56, batch=1)        # halo kernels (ResNet-50 block group 1)
  assert rc == -4 and b'halo' in lib.rigl_last_error()
  rc, _, _ = _compare(3, 64, 7, 2, 32)                  # 3-channel stem
  assert rc == -4
  lib.rigl_set_force_simt(1)
  try:
    rc, _, _ = _compare(64, 128, 1, 1, 8)
  finally:
    lib.rigl_set_force_simt(0)
  assert rc == -4


def _random_bn_state(model, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  with torch.no_grad():
    for m in model.modules():
      if isinstance(m, FusedBatchNormReLU):
        c = m.channels
        m.weight.copy_(torch.rand(c, device=DEV, generator=g) + 0.5)
        m.bias.copy_(torch.randn(c, device=DEV, generator=g) * 0.2)
        m.running_mean.copy_(torch.randn(c, device=DEV, generator=g) * 0.2)
        m.running_var.copy_(torch.rand(c, device=DEV, generator=g) + 0.5)


def _build(name, seed=0):
  torch.manual_seed(seed)
  model = {'resnet50': workloads.ResNet50, 'mobilenet_v1': workloads.MobileNetV1,
           'mobilenet_v2': workloads.MobileNetV2}[name](device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=seed)
  _random_bn_state(model, seed + 1)
  return model


def _images(n, size, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randn(n, 3, size, size, device=DEV, generator=g).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)


def _eval_logits(model, x, fused):
  old = layers.FUSE_BN_INFER
  layers.FUSE_BN_INFER = fused
  try:
    model.eval()
    with torch.no_grad():
      return model(x).clone()
  finally:
    layers.FUSE_BN_INFER = old


@pytest.mark.parametrize('name', ['resnet50', 'mobilenet_v1', 'mobilenet_v2'])
def test_eval_logits_fused_equal_unfused_eager_and_graph(name):
  model = _build(name)
  x = _images(4, 96, 1)
  plain = _eval_logits(model, x, False)
  fused = _eval_logits(model, x, True)
  assert torch.isfinite(plain).all()
  assert torch.equal(fused, plain)
  ev = Evaluator(model)
  ev.reset()
  labels = torch.zeros(4, dtype=torch.long, device=DEV)
  assert ev.enable_cuda_graph(x, labels)
  got = ev.update(x, labels).clone()
  assert torch.equal(got, plain)
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    ev.update(x, labels)
    torch.cuda.synchronize()
  names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
  assert_ran(names, _BN_KERNEL, 'graph replay of %s' % name)


def _np_metrics(logits, labels, ls):
  z = logits.astype(np.float64)
  top1 = (np.argmax(logits, 1) == labels).sum()
  tgt = logits[np.arange(len(labels)), labels]
  top5 = (((logits > tgt[:, None]).sum(1) < 5) & np.isfinite(logits).all(1)).sum()
  logp = z - z.max(1, keepdims=True)
  logp = logp - np.log(np.exp(logp).sum(1, keepdims=True))
  soft = np.eye(z.shape[1])[labels] * (1 - ls) + ls / z.shape[1]
  return top1, top5, -(soft * logp).sum(1).mean()


@pytest.mark.parametrize('graph', [False, True])
def test_metrics_equal_a_numpy_restatement(graph):
  model = _build('resnet50', seed=3)
  batches = [(_images(6, 64, 10 + i), torch.randint(0, 1000, (6,), device=DEV)) for i in range(3)]
  ev = Evaluator(model, weight_decay=1e-4)
  ev.reset()
  if graph:
    assert ev.enable_cuda_graph(batches[0][0], batches[0][1])
  for x, y in batches:
    ev.update(x, y)
  got = ev.result()
  # the same logits from the plain forward, which packs every layer per call
  top1 = top5 = cross = 0.0
  for x, y in batches:
    z = _eval_logits(model, x, False).cpu().numpy()
    t1, t5, c = _np_metrics(z, y.cpu().numpy(), 0.1)
    top1, top5, cross = top1 + t1, top5 + t5, cross + 6 * c
  assert got['eval_accuracy'] == top1 / 18.0
  assert got['top_5_eval_accuracy'] == top5 / 18.0
  assert got['cross_loss'] == pytest.approx(cross / 18.0, rel=1e-5)
  ws = [m.weight.detach().double() for m in model.modules()
        if isinstance(m, (layers._MaskedLayer, workloads.DenseConv2d, torch.nn.Linear))]
  assert got['reg_loss'] == pytest.approx(1e-4 * 0.5 * float(sum(w.pow(2).sum() for w in ws)), rel=1e-4)


def _fingerprint(model, harness):
  parts = {}
  for n, p in list(model.named_parameters()) + list(model.named_buffers()):
    parts['p/' + n] = p.detach().clone()
  for l in model.registry.layers():
    parts['mask/' + l.scope] = l.mask.bits.clone()
    parts['grad/' + l.scope] = l.masked_weights.dense_grad.clone()
    parts['fresh/' + l.scope] = l.masked_weights.fresh
  for i, st in enumerate(harness.inner.state.values()):
    for k, v in (st.items() if isinstance(st, dict) else ()):
      if torch.is_tensor(v):
        parts['slot/%d/%s' % (i, k)] = v.clone()
  parts['step'] = harness.global_step.value
  parts['ahead'] = frozenset(layers._PACKED_AHEAD)
  parts['training'] = model.training
  return parts


def _same(a, b):
  assert a.keys() == b.keys()
  for k in a:
    if torch.is_tensor(a[k]):
      assert torch.equal(a[k], b[k]), k
    else:
      assert a[k] == b[k], k


def _harness(model):
  return workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)


def test_evaluation_leaves_the_training_state_untouched():
  x = _images(8, 64, 20)
  y = torch.randint(0, 1000, (8,), device=DEV)
  a, b = _build('resnet50', seed=5), _build('resnet50', seed=5)
  ha, hb = _harness(a), _harness(b)
  a.train(); b.train()
  ha.step(x, y); hb.step(x, y)
  before = _fingerprint(a, ha)
  for stats in (False, True):
    ev = Evaluator(a, use_batch_statistics=stats, mask_summaries=True)
    ev.reset()
    ev.update(_images(4, 64, 21), torch.randint(0, 1000, (4,), device=DEV))
    r = ev.result()
    assert np.isfinite(r['cross_loss'])
  _same(before, _fingerprint(a, ha))
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    la = ha.step(x, y)
    torch.cuda.synchronize()
  names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
  assert_not_ran(names, _BN_KERNEL, 'training step')
  lb = hb.step(x, y)
  assert torch.equal(la, lb)
  for pa, pb in zip(a.parameters(), b.parameters()):
    assert torch.equal(pa, pb)


def test_batch_statistics_differ_from_moving_averages():
  model = _build('mobilenet_v2', seed=6)
  x, y = _images(8, 64, 30), torch.randint(0, 1000, (8,), device=DEV)
  res = {}
  for stats in (False, True):
    ev = Evaluator(model, use_batch_statistics=stats)
    ev.reset()
    ev.update(x, y)
    res[stats] = ev.result()['cross_loss']
  assert np.isfinite(res[True]) and res[True] != res[False]


def test_eval_once_after_restore_matches_the_original():
  x, y = _images(8, 64, 40), torch.randint(0, 1000, (8,), device=DEV)
  model = _build('resnet50', seed=7)
  h = _harness(model)
  model.train()
  for _ in range(3):
    h.step(x, y)
  data = [(_images(4, 64, 41 + i), torch.randint(0, 1000, (4,), device=DEV)) for i in range(2)]

  def evaluate(m):
    ev = Evaluator(m, mask_summaries=True)
    ev.reset()
    for a, b in data:
      ev.update(a, b)
    return ev.result()
  want = evaluate(model)
  with tempfile.TemporaryDirectory() as d:
    checkpoint.save(d, checkpoint.variables_of(model), h.global_step.value)
    fresh = workloads.ResNet50(device=DEV)
    checkpoint.restore(checkpoint.latest_checkpoint(d), checkpoint.variables_of(fresh))
  got = evaluate(fresh)
  assert got == want
  assert len([k for k in got if k.startswith('pruning/')]) == 54
  l = model.registry.layers()[5]
  assert got['pruning/%s/mask/sparsity' % l.scope] == pytest.approx(l.mask.sparsity())

