"""VGG on the H100: the ReLU conv epilogues against the plain kernels followed by a ReLU / gate, the 2x2 ReLU pool
and the standalone gate against float64, the whole network against a float64 restatement of the reference graph
(teacher-forced per layer, and free-running), and training / evaluation on it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_eval_gpu as teg
import test_whole_step_parity_gpu as wsp
import vgg_oracle as vo
from isolated import assert_ran
from oracle import rigl_oracle as orc
from rigl_b200 import _cabi, layers, pruning, workloads
from rigl_b200.evaluate import Evaluator, regularized_kernels
from rigl_b200.layers import SparseConv2d, _workspace
from rigl_b200.norm import max_pool2x2_relu
from tile_masks import tile_mask

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _act(n, c, h, w, gen, relu=False):
  t = torch.randn(n, c, h, w, device=DEV, generator=gen)
  return (torch.relu(t) if relu else t).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _layer(cin, cout, sparsity=0.8, pattern=None, seed=0):
  layer = SparseConv2d(cin, cout, 3, strides=1, padding='SAME', device=DEV, registry=pruning.MaskedLayerRegistry())
  rng = np.random.RandomState(seed)
  m = tile_mask(pattern, (3, 3, cin, cout), rng) if pattern else \
      orc.get_mask_random_numpy((3, 3, cin, cout), sparsity, rng).astype(np.float32)
  layer.mask.assign(m)
  layer.pack()
  return layer


def relu_conv_case(cin, cout, h, batch=2, pattern=None, seed=0, expect_fused=True):
  """Fused ReLU fprop == plain fprop + ReLU, gated dgrad == plain dgrad + where(x > 0, dx, 0), bit for bit (+-0
  compare equal).  expect_fused: the fused entry points returned RIGL_OK (else RIGL_ERR_UNSUPPORTED is fine)."""
  gen = torch.Generator(device=DEV).manual_seed(seed)
  layer = _layer(cin, cout, pattern=pattern, seed=seed)
  x = _act(batch, cin, h, h, gen, relu=True)
  lib, st = _cabi.lib(), _cabi.stream_ptr()
  layer.relu_out, layer.gate_dgrad = False, False
  y0 = layer._fprop(x, None, False)
  layer.relu_out = True
  y1 = layer._fprop(x, None, False)
  assert torch.equal(y1, torch.relu(y0)), (cin, cout, h)
  assert bool((y1 >= 0).all())
  if layer.patch_mode:
    return
  d = layer._desc(batch, h, h)
  ws = _workspace(x.device, lib.rigl_conv_workspace_bytes(d))
  out = torch.empty_like(y0)
  rc = lib.rigl_masked_conv2d_fprop_relu(d, x.data_ptr(), layer.packed.data_ptr(), out.data_ptr(), ws.data_ptr(),
                                         ws.numel(), st)
  assert rc == (0 if expect_fused else rc), lib.rigl_last_error()
  dy = _act(batch, cout, h, h, gen)
  dx0 = layer._dgrad(dy, x)
  layer.gate_dgrad = True
  dx1 = layer._dgrad(dy, x)
  assert torch.equal(dx1, torch.where(x > 0, dx0, torch.zeros_like(dx0))), (cin, cout, h)
  dx2 = torch.empty_like(x)
  rc = lib.rigl_masked_conv2d_dgrad_relu(d, dy.data_ptr(), layer.packed.data_ptr(), x.data_ptr(), dx2.data_ptr(),
                                         ws.data_ptr(), ws.numel(), st)
  torch.cuda.synchronize()
  if expect_fused:
    assert rc == 0, lib.rigl_last_error()
  if rc == 0:
    assert torch.equal(dx2, dx1)


# every distinct VGG-16 conv shape (input extent, cin, cout) at 224x224
_VGG16 = sorted({(hw, sh[2], sh[3]) for _, sh, hw in vo.masked_layers('vgg_16', prune_last_layer=False)}, reverse=True)


@pytest.mark.parametrize('hw,cin,cout', _VGG16, ids=lambda v: str(v))
def test_relu_epilogues_on_every_vgg16_conv_shape(hw, cin, cout):
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    relu_conv_case(cin, cout, hw, batch=2, seed=cin + cout)
    torch.cuda.synchronize()
  names = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
  # conv2_1 (64 -> 128 at 112) is on the halo kernel; the 3-channel first conv on the patch matrix (K-major)
  assert_ran(names, r'k_halo3x3_kmajor_relu' if (hw, cin) == (112, 64) else r'k_igemm_kmajor_relu<.*false>', str(hw))
  if cin != 3:
    assert_ran(names, r'k_igemm_kmajor_relu<.*true>', 'gated dgrad %d' % hw)


@pytest.mark.parametrize('cin,cout,h,batch', [(64, 72, 9, 3), (96, 200, 7, 2), (40, 24, 11, 1), (256, 136, 6, 2)])
def test_relu_epilogues_ragged_channels_and_partial_boxes(cin, cout, h, batch):
  relu_conv_case(cin, cout, h, batch=batch, seed=h, expect_fused=cin % 8 == 0 and cout % 8 == 0)


@pytest.mark.parametrize('pattern', ['staircase', 'block0', 'half', 'dead_taps', 'corner', 'dead'])
def test_relu_epilogues_dead_weight_tiles(pattern):
  relu_conv_case(192, 256, 8, pattern=pattern, seed=3)


def test_gated_dgrad_unsupported_shapes_launch_nothing():
  lib = _cabi.lib()
  gen = torch.Generator(device=DEV).manual_seed(0)

  def call(cin, cout, h, stride):
    layer = SparseConv2d(cin, cout, 3, strides=stride, padding='SAME', device=DEV,
                         registry=pruning.MaskedLayerRegistry())
    layer.pack()
    x = _act(2, cin, h, h, gen, relu=True)
    d = layer._desc(2, h, h)
    dy = _act(2, cout, d.out_h, d.out_w, gen)
    dx = torch.empty_like(x)
    ws = _workspace(x.device, lib.rigl_conv_workspace_bytes(d))
    torch.cuda.synchronize()
    before = _cabi.launch_count()
    rc = lib.rigl_masked_conv2d_dgrad_relu(d, dy.data_ptr(), layer.packed.data_ptr(), x.data_ptr(), dx.data_ptr(),
                                           ws.data_ptr(), ws.numel(), _cabi.stream_ptr())
    return rc, _cabi.launch_count() - before
  assert call(64, 64, 30, 1) == (-4, 0) and b'halo' in lib.rigl_last_error()      # halo dgrad (reduced size)
  assert call(64, 128, 16, 2) == (-4, 0)                                           # stride-2 parity launches
  lib.rigl_set_force_simt(1)
  try:
    assert call(64, 128, 16, 1) == (-4, 0)
  finally:
    lib.rigl_set_force_simt(0)


# ---- pool and gate against float64 ----
def _pool_ref(x):
  """(y, route bytes) of the 2x2/2 VALID pool over x [N,C,H,W] in float64 / numpy."""
  a = x.permute(0, 2, 3, 1).double().cpu().numpy()
  n, h, w, c = a.shape
  oh, ow = h // 2, w // 2
  win = np.stack([a[:, 0:2 * oh:2, 0:2 * ow:2], a[:, 0:2 * oh:2, 1:2 * ow:2], a[:, 1:2 * oh:2, 0:2 * ow:2],
                  a[:, 1:2 * oh:2, 1:2 * ow:2]])
  y = win.max(0)
  arg = np.argmax(win, 0)                     # first maximum in scan order
  route = np.where(y > 0, arg, 255).astype(np.uint8)
  return y, route


@pytest.mark.parametrize('shape', [(2, 7, 9, 16), (3, 8, 8, 64), (1, 15, 13, 24), (2, 224, 224, 64)],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_pool2x2_relu_vs_fp64(shape):
  n, h, w, c = shape
  gen = torch.Generator(device=DEV).manual_seed(h * w)
  # values in {0, 0.5, 1, 1.5}: many ties and all-zero windows, as after a ReLU
  x = (torch.randint(0, 4, (n, h, w, c), device=DEV, generator=gen).float() * 0.5)
  x[:, :, :, :c // 4] = 0.0                    # whole channels of zeros: windows whose maximum is 0
  x = x.to(torch.bfloat16).permute(0, 3, 1, 2).requires_grad_(True)
  y = max_pool2x2_relu(x)
  want_y, route = _pool_ref(x.detach())
  assert np.array_equal(y.detach().permute(0, 2, 3, 1).double().cpu().numpy(), want_y)
  g = _act(n, c, h // 2, w // 2, gen)
  y.backward(g)
  gd = g.permute(0, 2, 3, 1).double().cpu().numpy()
  want_dx = np.zeros((n, h, w, c))
  for j in range(4):
    sel = np.where(route == j, gd, 0.0)
    want_dx[:, (j >> 1):2 * (h // 2):2, (j & 1):2 * (w // 2):2] = sel
  assert np.array_equal(x.grad.permute(0, 2, 3, 1).double().cpu().numpy(), want_dx)


def test_relu_gate_vs_fp64_and_in_place():
  gen = torch.Generator(device=DEV).manual_seed(1)
  x = torch.randn(4096 + 8, device=DEV, generator=gen).to(torch.bfloat16)
  x[::7] = 0.0
  g = torch.randn(x.shape, device=DEV, generator=gen).to(torch.bfloat16)
  out = layers.relu_gate(x, g, torch.empty_like(g))
  assert torch.equal(out, torch.where(x > 0, g, torch.zeros_like(g)))
  gi = g.clone()
  layers.relu_gate(x, gi, gi)
  assert torch.equal(gi, out)
  xi = x.clone()
  layers.relu_gate(xi, xi, xi)
  assert torch.equal(xi, torch.relu(x))


# ---- the model ----
def _model(vgg_type, seed, width=0.125, num_classes=16, prune_last_layer=True, sparsity=0.8):
  torch.manual_seed(seed)
  model = workloads.VGG(vgg_type, num_classes=num_classes, width=width, prune_last_layer=prune_last_layer, device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', sparsity, seed=seed)
  return model


def _images(n, size, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randn(n, 3, size, size, device=DEV, generator=g).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)


def test_registry_scopes_init_and_regularized_kernels():
  for prune_last in (True, False):
    model = _model('vgg_16', 0, width=1.0, num_classes=1000, prune_last_layer=prune_last)
    want = [(n + '/mask:0', list(sh)) for n, sh, _ in vo.masked_layers('vgg_16', 1000, prune_last)]
    assert [(m.name, list(m.shape)) for m in model.registry.get_masks()] == want
    assert [l.weight.name for l in model.registry.layers()][0] == 'vgg_16/conv1/conv1_1/weights:0'
    conv = model.registry.layers()[3]                     # variance_scaling(2.0), truncated at 2 sigma
    w = conv.weight.detach().double()
    std = np.sqrt(2.0 / (9 * conv.in_channels)) / .87962566103423978
    assert float(w.abs().max()) <= 2 * std and abs(float(w.std()) / np.sqrt(2.0 / (9 * conv.in_channels)) - 1) < 0.02
    ks = regularized_kernels(model)
    assert [id(k) for k in ks] == [id(l.weight) for l in model.registry.layers()]
    if not prune_last:
      assert float(model.fc8.bias.detach().abs().max()) == 0.0 and model.fc8.weight.shape == (1000, 512)
    del model
    torch.cuda.empty_cache()


def _ref_step(model, x, labels, prune_last):
  """float64 restatement on the model's bf16-rounded masked weights: logits, loss, dense gradients and the input /
  pre-activation gradient of every masked conv (for the teacher-forced replay)."""
  convs = list(model.convs)
  ws = [(c.weight.detach() * c.mask.to_dense()).to(torch.bfloat16).double().requires_grad_(True) for c in convs]
  if prune_last:
    f8 = model.fc8
    w8 = (f8.weight.detach() * f8.mask.to_dense()).to(torch.bfloat16).double().requires_grad_(True)
    bias = None
  else:
    w8 = model.fc8.weight.detach().double().requires_grad_(True)
    bias = model.fc8.bias.detach().double()
  record = {}
  h = x.detach().double()
  i = 0
  for s, reps in enumerate(vo.CFG[model.vgg_type], 1):
    for _ in range(reps):
      inp = h
      z = F.conv2d(inp, ws[i].permute(3, 2, 0, 1), padding=1)
      z.retain_grad()
      record[convs[i].scope] = (inp, z)
      h = torch.relu(z)
      i += 1
    if s < 5:
      h = F.max_pool2d(h, 2, 2)
  feat = h.mean(dim=(2, 3))
  logits = feat @ w8.reshape(-1, w8.shape[-1]) if bias is None else feat @ w8.t() + bias
  loss = F.cross_entropy(logits, labels.cpu().to(logits.device), label_smoothing=0.1)
  loss.backward()
  dense = [w.grad for w in ws] + [w8.grad]
  return logits.detach(), float(loss.detach()), dense, record


def _nhwc(t):
  return t.detach().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _rel(got, want):
  got, want = got.double(), want.double()
  return float((got - want).norm() / (want.norm() + 1e-30))


@pytest.mark.parametrize('vgg_type', sorted(vo.CFG))
def test_whole_network_vs_fp64_reference_graph(vgg_type):
  """Teacher-forced: every masked conv replayed alone on the restatement's bf16-rounded input and pre-activation
  gradient: fprop (ReLU epilogue), dgrad (gated where the layer has gate_dgrad) <= 1e-3 and dense wgrad <= 2e-5
  relative L2 (DESIGN.md 5).  A missing gate on an edge leaves the gradient of inactive units in dx (an O(1) error),
  and so does a gate by the wrong tensor.  Free-running: loss and dense gradients of the whole step (see the bounds
  below)."""
  prune_last = vgg_type != 'vgg_a'            # the dense fc8 on one variant
  model = _model(vgg_type, 11, prune_last_layer=prune_last)
  x = _images(2, 32, 12)
  labels = torch.randint(0, 16, (2,), device=DEV)
  want_logits, want_loss, want_dense, record = _ref_step(model, x.to(DEV), labels, prune_last)
  forced = {}
  for conv in model.convs:
    inp, z = record[conv.scope]
    xb = _nhwc(inp)
    gb = _nhwc(z.grad)
    conv.pack()
    y = conv._fprop(xb, None, False)
    w = (conv.weight.detach() * conv.mask.to_dense()).to(torch.bfloat16).double().permute(3, 2, 0, 1)
    want_y = torch.relu(F.conv2d(xb.double(), w, padding=1))
    e_y = _rel(y, want_y.to(torch.bfloat16))               # (both sides store bf16)
    e_dx = 0.0
    if conv.gate_dgrad:
      dx = conv._dgrad(gb, xb)
      # conv^T of the stored incoming gradient, times the derivative of the ReLU that produced the input
      want_dx = torch.nn.grad.conv2d_input(xb.shape, w, gb.double(), padding=1) * (xb > 0).double()
      e_dx = _rel(dx, want_dx.to(torch.bfloat16))
    dense = torch.zeros_like(conv.masked_weights.dense_grad)
    conv._wgrad(xb, gb, dense, accumulate=False)
    want_w = torch.nn.grad.conv2d_weight(xb.double(), (conv.out_channels, conv.in_channels, 3, 3), gb.double(),
                                         padding=1)
    e_w = _rel(dense.view(conv.weight.shape), want_w.permute(2, 3, 1, 0))
    forced[conv.scope] = (e_y, e_dx, e_w)
    assert e_y <= 1e-3 and e_dx <= 1e-3 and e_w <= 2e-5, (conv.scope, forced[conv.scope])
  # free-running
  h = workloads.TrainHarness(model, lr=0.05, frequency=1000, end_step=2000)
  got_loss = float(h._forward_backward(x, labels, set_to_none=False).detach())
  torch.cuda.synchronize()
  rel = {}
  for i, l in enumerate(model.registry.layers()):
    rel[l.scope] = _rel(l.masked_weights.dense_grad.view(l.weight.shape), want_dense[i])
  wsp._record('vgg_%s' % vgg_type, dict(loss_cuda=got_loss, loss_ref=want_loss, rel_l2=rel,
                                         teacher_forced={k: list(v) for k, v in forced.items()}))
  # The step stores every activation and gradient in bf16, the restatement none: rounding flips (a ReLU or pool
  # decision on the other side of a rounded value) grow from the classifier down, as in the plain BN stacks of
  # test_whole_step_parity_gpu.  Measured on an H100 (width 1/8, 32x32, batch 2): loss within 2e-6 relative; dense-
  # gradient relative L2 0.004-0.006 at fc8, 0.03-0.06 on the stage-5 convs, rising to 0.17 / 0.23 / 0.44 at
  # conv1_1 of vgg_a / vgg_16 / vgg_19.  Bounded: the loss at 5e-3, fc8 and stage 5 at 0.2 (~3x); earlier layers are
  # recorded, and their kernels bounded by the teacher-forced pass above.
  assert abs(got_loss - want_loss) <= 5e-3 * abs(want_loss), (got_loss, want_loss)
  tail = {k: v for k, v in rel.items() if '/conv5/' in k or k.endswith('/fc8')}
  assert len(tail) == vo.CFG[vgg_type][4] + int(prune_last) and max(tail.values()) <= 0.2, rel


def _fallback_outputs(vgg_type, fuse):
  old = layers.FUSE_RELU
  layers.FUSE_RELU = fuse
  try:
    model = _model(vgg_type, 21, width=0.25)
    x = _images(2, 56, 22)
    labels = torch.randint(0, 16, (2,), device=DEV)
    h = workloads.TrainHarness(model, lr=0.05, frequency=1000, end_step=2000)
    logits = model(x).detach().clone()
    h._forward_backward(x, labels, set_to_none=False)
    torch.cuda.synchronize()
    return [logits] + [l.masked_weights.dense_grad.clone() for l in model.registry.layers()]
  finally:
    layers.FUSE_RELU = old


def test_standalone_gate_route_equals_fused_route():
  """RIGL_FUSE_RELU=0 (the switch is read into layers.FUSE_RELU): plain conv + rigl_relu_gate everywhere.  Gating only
  selects values, so the logits and every dense gradient are bit-identical (+-0 compare equal).  The fused route mixes
  both forms: at width 0.25 and 56x56 the gated dgrads that reduce over <= 64 channels run on the halo kernel, which
  has no gate, and fall back to the plain call + rigl_relu_gate; the 128-channel ones gate in the K-major epilogue.
  (At 64x64 no layer would take the halo kernel: every stage width is a power of two, which it refuses.)"""
  for vgg_type in ('vgg_a', 'vgg_16'):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
      a = _fallback_outputs(vgg_type, True)
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert_ran(names, r'k_igemm_kmajor_relu<.*true>', vgg_type)
    # (one k_relu_gate is the last conv's relu_grad_gate; the others are the halo dgrads' fallbacks)
    n_gate = sum('k_relu_gate' in n for n in names)
    assert n_gate > 1, (vgg_type, n_gate)
    b = _fallback_outputs(vgg_type, False)
    for i, (p, q) in enumerate(zip(a, b)):
      assert torch.equal(p, q), (vgg_type, i)


def _train(graph, inner, steps=5):
  model = _model('vgg_16', 5, width=0.25, sparsity=0.8)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100, inner_optimizer=inner)
  x = _images(8, 64, 6)
  y = torch.randint(0, 16, (8,), device=DEV)
  if graph:
    assert h.enable_cuda_graph(x, y)
  losses, masks = [], []
  for _ in range(steps):
    losses.append(h.step(x, y).detach().clone())
    masks.append([m.numpy().copy() for m in model.registry.get_masks()])
  torch.cuda.synchronize()
  return torch.stack(losses), masks, [l.weight.detach().clone() for l in model.registry.layers()], h.global_step.value


@pytest.mark.parametrize('inner', ['momentum', 'adam'])
def test_cuda_graph_replay_bit_identical_to_eager(inner):
  le, me, we, ge = _train(False, inner)
  lg, mg, wg, gg = _train(True, inner)
  assert ge == gg == 3
  assert torch.isfinite(le).all()
  assert torch.equal(le, lg), (le.tolist(), lg.tolist())
  for a, b in zip(me, mg):
    assert all(np.array_equal(p, q) for p, q in zip(a, b))
  for a, b in zip(we, wg):
    assert torch.equal(a, b)


def test_mask_updates_match_the_oracle_drop_grow():
  model = _model('vgg_a', 7, width=0.25)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  images = torch.randn(4, 3, 64, 64).to(torch.bfloat16)
  labels = torch.randint(0, 16, (4,))
  wsp._check_update_steps(model, h, images, labels, 4, [0, 2])


def test_evaluator_matches_numpy_metrics_and_leaves_training_state():
  model = _model('vgg_16', 9, width=0.25)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  x, y = _images(4, 64, 30), torch.randint(0, 16, (4,), device=DEV)
  h.step(x, y)
  before = teg._fingerprint(model, h)
  batches = [(_images(3, 64, 31 + i), torch.randint(0, 16, (3,), device=DEV)) for i in range(2)]
  ev = Evaluator(model, weight_decay=1e-4)
  ev.reset()
  for a, b in batches:
    ev.update(a, b)
  got = ev.result()
  teg._same(before, teg._fingerprint(model, h))
  model.eval()
  top1 = top5 = cross = 0.0
  with torch.no_grad():
    for a, b in batches:
      t1, t5, c = teg._np_metrics(model(a).float().cpu().numpy(), b.cpu().numpy(), 0.1)
      top1, top5, cross = top1 + t1, top5 + t5, cross + 3 * c
  model.train()
  assert got['eval_accuracy'] == top1 / 6.0
  assert got['top_5_eval_accuracy'] == top5 / 6.0
  assert got['cross_loss'] == pytest.approx(cross / 6.0, rel=1e-5)
