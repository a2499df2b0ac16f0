"""ResNet-18 ... 200 on the H100: the space-to-depth stem's 64-channel groups against one launch per group,
ResNet(50) against ResNet50, the whole network against a float64 restatement of the reference graph
(tests/resnet_oracle.py; teacher-forced per layer, and free-running), and training / evaluation on it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnet_oracle as ro
import test_whole_step_parity_gpu as wsp
from oracle import rigl_oracle as orc
from rigl_b200 import checkpoint, layers, pruning, workloads
from rigl_b200.evaluate import Evaluator, regularized_kernels
from rigl_b200.layers import SparseConv2d
from rigl_b200.norm import FusedBatchNormReLU

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _images(n, size, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randn(n, 3, size, size, device=DEV, generator=g).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)


# ---- the stem's 64-channel groups ----
def _stem(weight, mask):
  layer = SparseConv2d(3, weight.shape[-1], 7, strides=2, padding='FIXED', device=DEV,
                       registry=pruning.MaskedLayerRegistry())
  with torch.no_grad():
    layer.weight.copy_(weight)
  layer.mask.assign(mask)
  return layer


def _stem_step(layer, x, dy):
  """fprop and the dense wgrad of one training step of the stem, through its autograd function."""
  layer.masked_weights.fresh = False
  layer.weight.grad = None
  y = layer(x)
  assert layer._use_s2d
  y.backward(dy)
  torch.cuda.synchronize()
  return y.detach(), layer.masked_weights.dense_grad.detach().clone().view(layer.weight.shape)


@pytest.mark.parametrize('cout', [72, 96, 128, 256])
def test_stem_groups_equal_one_launch_per_group(cout):
  """At batch 256, 224^2: the grouped stem's output and dense wgrad, channels 64j .. 64j+63, are bit-identical to a
  separate launch on that weight slice (64 channels, or the ragged remainder): every group runs a 64-channel launch's
  grid and strip-to-CTA assignment, and the reduce adds the partials in the same CTA order."""
  rng = np.random.RandomState(cout)
  mask = orc.get_mask_random_numpy((7, 7, 3, cout), 0.5, rng).astype(np.float32)
  gen = torch.Generator(device=DEV).manual_seed(cout)
  weight = torch.randn(7, 7, 3, cout, device=DEV, generator=gen) * 0.1
  x = torch.relu(torch.randn(256, 3, 224, 224, device=DEV, generator=gen) + 0.5).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)
  dy = (torch.randn(256, cout, 112, 112, device=DEV, generator=gen) * 0.25 + 1).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)
  big = _stem(weight, mask)
  y, dw = _stem_step(big, x, dy)
  assert torch.isfinite(y.float()).all() and float(y.float().abs().max()) > 0
  del big
  for a in range(0, cout, 64):
    b = min(a + 64, cout)
    part = _stem(weight[..., a:b].contiguous(), np.ascontiguousarray(mask[..., a:b]))
    yp, dwp = _stem_step(part, x, dy[:, a:b].contiguous(memory_format=torch.channels_last))
    assert torch.equal(y[:, a:b].view(torch.int16), yp.view(torch.int16)), (cout, a)
    assert torch.equal(dw[..., a:b], dwp), (cout, a)
    del part, yp, dwp
  torch.cuda.empty_cache()


# ---- ResNet(50) is ResNet50 ----
def test_resnet_50_builds_and_trains_as_resnet50():
  """Same seed: the same scopes, shapes, modules and initial weights; one train step gives bit-identical logits,
  loss and gradients (dense wgrads, BN parameters)."""
  models = []
  for build in (lambda: workloads.ResNet50(device=DEV), lambda: workloads.ResNet(50, device=DEV)):
    torch.manual_seed(3)
    m = build()
    workloads.init_masks(m, 'erdos_renyi_kernel', 0.8, seed=3)
    models.append(m)
  a, b = models
  assert [(m.name, m.shape) for m in a.registry.get_masks()] == [(m.name, m.shape) for m in b.registry.get_masks()]
  pa, pb = list(a.named_parameters()), list(b.named_parameters())
  assert [(n, p.shape) for n, p in pa] == [(n, p.shape) for n, p in pb]
  assert all(torch.equal(p, q) for (_, p), (_, q) in zip(pa, pb))
  assert all(np.array_equal(p.numpy(), q.numpy()) for p, q in zip(a.registry.get_masks(), b.registry.get_masks()))
  x, labels = _images(4, 64, 5), torch.randint(0, 1000, (4,), device=DEV)
  outs = []
  for m in models:
    h = workloads.TrainHarness(m, lr=0.05, frequency=1000, end_step=2000)
    logits = m(x).detach().clone()
    loss = h._forward_backward(x, labels, set_to_none=False).detach().clone()
    torch.cuda.synchronize()
    grads = [l.masked_weights.dense_grad.clone() for l in m.registry.layers()]
    grads += [p.grad.clone() for p in m.parameters() if p.grad is not None]
    outs.append((logits, loss, grads))
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
  assert len(outs[0][2]) == len(outs[1][2]) > 54
  for p, q in zip(outs[0][2], outs[1][2]):
    assert torch.equal(p, q)


# ---- the whole network against float64 ----
def _model(depth, seed, width=0.25, num_classes=16, sparsity=0.8, **kw):
  torch.manual_seed(seed)
  model = workloads.ResNet(depth, num_classes=num_classes, width=width, device=DEV, **kw)
  workloads.init_masks(model, 'erdos_renyi_kernel', sparsity, seed=seed)
  return model


def _conv_bn_pairs(model):
  """[(conv, the batch norm after it)] of the model."""
  pairs = [(model.initial_conv, model.initial_bn)]
  for blk in model.blocks:
    for c, n in (('proj', 'proj_bn'), ('conv1', 'bn1'), ('conv2', 'bn2'), ('conv3', 'bn3')):
      if getattr(blk, c, None) is not None:
        pairs.append((getattr(blk, c), getattr(blk, n)))
  return pairs


def _bn_state(model, seed, last_gain=0.1):
  """gamma ~ U[0.5, 1.5], beta ~ 0.1 N(0, 1); the zero-init last BN of a block at `last_gain` times that (near the
  reference's zero, with the residual branches' gradients alive), as test_whole_step_parity_gpu does."""
  g = torch.Generator(device=DEV).manual_seed(seed)
  with torch.no_grad():
    for m in model.modules():
      if isinstance(m, FusedBatchNormReLU):
        gain = last_gain if float(m.weight.abs().max()) == 0 else 1.0
        m.weight.copy_((torch.rand(m.channels, device=DEV, generator=g) + 0.5) * gain)
        m.bias.copy_(torch.randn(m.channels, device=DEV, generator=g) * 0.1)


def _ref_step(model, x, labels):
  """float64 restatement on the model's bf16-rounded masked weights: loss, dense gradients (registry order) and the
  input / output of every masked conv with their gradients (for the teacher-forced replay)."""
  ws = {}
  for l in model.registry.layers():
    ws[l.scope] = (l.weight.detach() * l.mask.to_dense()).to(torch.bfloat16).double().requires_grad_(True)
  bn = {c.scope: (n.weight.detach(), n.bias.detach()) for c, n in _conv_bn_pairs(model)}
  record = {}
  logits = ro.forward(x, ws, bn, model.depth, model.width, fc_bias=model.final_dense.bias.detach(), record=record)
  loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
  loss.backward()
  return float(loss.detach()), [ws[l.scope].grad for l in model.registry.layers()], record


def _nhwc(t):
  return t.detach().to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _rel(got, want):
  got, want = got.double(), want.double()
  return float((got - want).norm() / (want.norm() + 1e-30))


# Free-running bounds, about 3x the figures measured on an H100 80GB HBM3 (700 W) at width 1/4, 64 x 64 (the inputs
# are seeded, so the figures are fixed).  ResNet-18, batch 4: loss within 6.4e-5 relative; dense-gradient relative
# L2 0.008 at final_dense, 0.13-0.27 on the last block, 0.12-0.42 elsewhere (the 2 x 2 last stage normalises over 16
# values per channel).  ResNet-101, batch 2: loss within 3.3e-4; 0.019 at final_dense, 0.18-0.25 on the last block,
# median 0.38 and at most 0.54 over all 105 layers.  The teacher-forced pass stays below 1.1e-4 on every layer.
_FREE = {18: dict(loss=2e-4, tail=0.8), 101: dict(loss=1e-3, tail=0.75)}


@pytest.mark.parametrize('depth,batch', [(18, 4), (101, 2)])
def test_whole_network_vs_fp64_reference_graph(depth, batch):
  """Teacher-forced: every masked conv replayed alone on the restatement's bf16-rounded input and output gradient:
  fprop and dgrad <= 1e-3, dense wgrad <= 2e-5 relative L2 (DESIGN.md 5).  Free-running: the loss, and the dense
  gradients of the last block and final_dense, within about 3x of the figures measured on the H100; the earlier
  layers' figures are recorded (a BN stack amplifies rounding flips from the classifier down) and their kernels are
  bounded by the teacher-forced pass."""
  model = _model(depth, 11)
  _bn_state(model, 12)
  x = _images(batch, 64, 13)
  labels = torch.randint(0, 16, (batch,), device=DEV)
  want_loss, want_dense, record = _ref_step(model, x, labels)
  forced = {}
  for conv, _ in _conv_bn_pairs(model):
    inp, z = record[conv.scope]
    xb, gb = _nhwc(inp), _nhwc(z.grad)
    k, s, p = conv.ksize, conv.stride, (conv.ksize - 1) // 2
    w = (conv.weight.detach() * conv.mask.to_dense()).to(torch.bfloat16).double().permute(3, 2, 0, 1)
    conv.pack()
    y = conv._fprop(xb, None, False)
    e_y = _rel(y, F.conv2d(xb.double(), w, stride=s, padding=p).to(torch.bfloat16))
    e_dx = 0.0
    if inp.requires_grad:
      dx = conv._dgrad(gb, xb)
      want_dx = torch.nn.grad.conv2d_input(xb.shape, w, gb.double(), stride=s, padding=p)
      e_dx = _rel(dx, want_dx.to(torch.bfloat16))
    dense = torch.zeros_like(conv.masked_weights.dense_grad)
    conv._wgrad(xb, gb, dense, accumulate=False)
    want_w = torch.nn.grad.conv2d_weight(xb.double(), tuple(w.shape), gb.double(), stride=s, padding=p)
    e_w = _rel(dense.view(conv.weight.shape), want_w.permute(2, 3, 1, 0))
    forced[conv.scope] = (e_y, e_dx, e_w)
    assert e_y <= 1e-3 and e_dx <= 1e-3 and e_w <= 2e-5, (conv.scope, forced[conv.scope])
  assert record['resnet_model/initial_conv'][0].requires_grad is False and model.initial_conv._use_s2d
  # free-running
  h = workloads.TrainHarness(model, lr=0.05, frequency=1000, end_step=2000)
  got_loss = float(h._forward_backward(x, labels, set_to_none=False).detach())
  torch.cuda.synchronize()
  rel = {}
  for i, l in enumerate(model.registry.layers()):
    rel[l.scope] = _rel(l.masked_weights.dense_grad.view(l.weight.shape), want_dense[i])
  wsp._record('resnet%d' % depth, dict(loss_cuda=got_loss, loss_ref=want_loss, rel_l2=rel,
                                       teacher_forced={k: list(v) for k, v in forced.items()}))
  last = model.blocks[-1]
  tail = {l.scope: rel[l.scope] for l in model.registry.layers()
          if l is model.final_dense or any(l is m for m in last.modules())}
  print('resnet%d loss %.6g vs %.6g; tail %s; max rel %.4f' % (depth, got_loss, want_loss, tail, max(rel.values())))
  assert abs(got_loss - want_loss) <= _FREE[depth]['loss'] * abs(want_loss), (got_loss, want_loss)
  assert len(tail) == (3 if depth < 50 else 4) and max(tail.values()) <= _FREE[depth]['tail'], tail


# ---- training and evaluation ----
def _train(graph, steps=5):
  model = _model(18, 5)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
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


def test_cuda_graph_replay_bit_identical_to_eager():
  le, me, we, ge = _train(False)
  lg, mg, wg, gg = _train(True)
  assert ge == gg == 3
  assert torch.isfinite(le).all()
  assert torch.equal(le, lg), (le.tolist(), lg.tolist())
  for a, b in zip(me, mg):
    assert all(np.array_equal(p, q) for p, q in zip(a, b))
  for a, b in zip(we, wg):
    assert torch.equal(a, b)


@pytest.mark.parametrize('depth', [18, 101])
def test_mask_updates_match_the_oracle_drop_grow(depth):
  model = _model(depth, 7)
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  images = torch.randn(4, 3, 64, 64).to(torch.bfloat16)
  labels = torch.randint(0, 16, (4,))
  wsp._check_update_steps(model, h, images, labels, 4, [0, 2])


@pytest.mark.parametrize('first,last', [(False, True), (True, False), (False, False)])
def test_dense_first_and_last_layers(first, last):
  """prune_first_layer / prune_last_layer off: those layers are outside the registry, keep the l2 regularizer, are
  initialised as the reference initialises them, and train."""
  model = _model(18, 8, prune_first_layer=first, prune_last_layer=last)
  want = [(n + '/mask:0', list(sh)) for n, sh in ro.masked_layers(18, 0.25, 16, first, last)]
  assert [(m.name, list(m.shape)) for m in model.registry.get_masks()] == want
  masked = [id(l.weight) for l in model.registry.layers()]
  ks = [id(k) for k in regularized_kernels(model)]
  dense = ([] if first else [model.initial_conv.weight]) + ([] if last else [model.final_dense.weight])
  assert all(id(w) in ks and id(w) not in masked for w in dense)
  assert sorted(ks) == sorted(masked + [id(w) for w in dense])
  if not first:
    assert isinstance(model.initial_conv, workloads.DenseConv2d) and model.initial_conv.weight.shape == (16, 3, 7, 7)
    assert abs(float(model.initial_conv.weight.detach().std()) / np.sqrt(2.0 / 147) - 1) < 0.1
  if not last:
    assert isinstance(model.final_dense, torch.nn.Linear) and float(model.final_dense.bias.detach().abs().max()) == 0
    assert abs(float(model.final_dense.weight.detach().std()) / 0.01 - 1) < 0.1
  names = checkpoint.variables_of(model)
  assert ('initial_conv/weight' in names) != first and ('final_dense/weight' in names) != last
  assert ('resnet_model/initial_conv/mask' in names) == first and ('resnet_model/final_dense/mask' in names) == last
  before = [w.detach().clone() for w in dense]
  h = workloads.TrainHarness(model, lr=0.05, frequency=1000, end_step=2000)
  x, y = _images(4, 64, 9), torch.randint(0, 16, (4,), device=DEV)
  for _ in range(2):
    loss = h.step(x, y)
  torch.cuda.synchronize()
  assert torch.isfinite(loss).all()
  assert all(not torch.equal(a, w.detach()) for a, w in zip(before, dense))


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


@pytest.mark.parametrize('depth', [18, 101])
def test_evaluator_same_metrics_with_and_without_fused_inference_bn(depth):
  model = _model(depth, 9)
  _random_bn_state(model, 10)
  batches = [(_images(3, 64, 31 + i), torch.randint(0, 16, (3,), device=DEV)) for i in range(2)]
  results, logits = [], []
  old = layers.FUSE_BN_INFER
  try:
    for fused in (True, False):
      layers.FUSE_BN_INFER = fused
      ev = Evaluator(model, weight_decay=1e-4)
      ev.reset()
      logits.append([ev.update(a, b).clone() for a, b in batches])
      results.append(ev.result())
  finally:
    layers.FUSE_BN_INFER = old
  assert all(torch.isfinite(t).all() for t in logits[0])
  for p, q in zip(*logits):
    assert torch.equal(p, q)
  assert results[0] == results[1], results
