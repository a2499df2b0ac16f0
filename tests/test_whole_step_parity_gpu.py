"""Whole-train-step parity: ONE CUDA sparse train step against the CPU restatement of the reference's step
(oracle/cpu_train_step.py), for the three model families of BASELINE.json (ResNet-50 C2/C3, WRN-22-2 C5,
MobileNet-v1 C4), plus bit-identical masks / re-initialised weights / momentum slots after the mask updates.

What is compared and how tight it can be (DESIGN.md 5, "whole-step bound"):
  * The CUDA path stores every activation and activation gradient in bf16 (fp32 accumulation inside each conv /
    BN reduction), as BASELINE C2 prescribes.  The oracle therefore runs in its `bf16_act` mode: the reference's
    fp32 step with every STORED tensor (conv outputs, BN / ReLU / residual outputs, pooled features) and its
    gradient rounded to bf16 at the same points, fp32 arithmetic inside each op.  Against the plain fp32 oracle
    a whole-network comparison is meaningless at initialisation: a batch-normalised ReLU network amplifies any
    perturbation ~1.2x per layer, so bf16 storage alone moves the dense gradients of ResNet-50 by a relative L2
    of ~1.3 -- measured on the CPU with no kernel involved (tools/noise_growth.py), and the CUDA step shows the
    same figures.
  * With matching rounding points what remains is fp32 summation order plus the rare bf16 rounding flips it
    causes (~1e-4 of a tensor per rounding point), amplified the same way.  Two checks follow from that:
    (1) TEACHER-FORCED: every masked layer replayed alone on the oracle's tensors of this very step -- no
        amplification, tight bounds (dense wgrad <= 2e-5, fprop / dgrad <= 1e-3 relative L2);
    (2) FREE-RUNNING: the whole CUDA step against the oracle's, bounded by ~3x the MEASURED figures (ResNet-50
        with the last BN of each block near the reference's zero init: median 0.15 / max 0.18; WRN-22-2: 0.08 /
        0.09; MobileNet-v1, a plain 27-BN stack with nothing to damp the growth: 0.09 at the classifier rising to
        0.7 at the first layer -- only its last two layers are bounded).  A wrong tap, stride, padding, transposed
        operand, BN statistic or residual wiring gives errors of order 1 in every layer downstream of it and
        fails (1) outright.  Measurements are recorded into gpurun_out/whole_step_parity_<model>.json.
  * Mask updates are integer work: given the dense gradients the CUDA step produced, the oracle's drop/grow
    (base.py:276-343 restated) must give BIT-IDENTICAL masks, weights and momentum slots; the optimizer step is
    checked against the oracle's Nesterov-momentum arithmetic on the same gradients.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import cpu_train_step as cpu
from oracle import rigl_oracle as orc
from rigl_b200 import workloads
from rigl_b200.norm import FusedBatchNormReLU

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _bn_init(seed, last_bn_gain=1.0):
  """gamma ~ U[0.5, 1.5], beta ~ 0.1 N(0,1); `last_bn_gain` scales the gamma of the LAST BN of a ResNet bottleneck
  (the reference initialises that one to ZERO, resnet_model.py:41-80 `init_zero`; a small non-zero value keeps the
  residual branches' gradients alive while staying near that regime)."""
  def init(key, c):
    r = np.random.RandomState((__import__('zlib').crc32(key.encode()) ^ seed) & 0x7fffffff)
    g = (0.5 + r.rand(c)).astype(np.float32)
    if key.endswith('3'):
      g = (g * np.float32(last_bn_gain)).astype(np.float32)
    return g, (0.1 * r.standard_normal(c)).astype(np.float32)
  return init


def _load(model, net):
  """Copies the oracle net's masked weights / masks / BN parameters into the CUDA model (BNs in execution order,
  which is the registration order in both)."""
  with torch.no_grad():
    for l in model.registry.layers():
      l.weight.copy_(net.w[l.scope].to(DEV))
      l.mask.assign(net.m[l.scope].numpy())
    bns = [m for m in model.modules() if isinstance(m, FusedBatchNormReLU)]
    assert len(bns) == len(net.bn_order)
    for mod, key in zip(bns, net.bn_order):
      g, b = net.bn[key]
      mod.weight.copy_(g.detach().to(DEV))
      mod.bias.copy_(b.detach().to(DEV))


def _rel_l2(got, want):
  return float(np.linalg.norm(got.astype(np.float64) - want.astype(np.float64)) /
               (np.linalg.norm(want.astype(np.float64)) + 1e-30))


def _record(tag, payload):
  if os.path.isdir('gpurun_out'):
    with open(os.path.join('gpurun_out', 'whole_step_parity_%s.json' % tag), 'w') as f:
      json.dump(payload, f, indent=1)


def _nhwc_dev(t):
  """oracle NCHW float32 (bf16-valued) -> device bf16 channels_last (logical NCHW)."""
  return t.detach().to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _teacher_forced_layers(model, net, tol_act=1e-3, tol_dense=2e-5):
  """Every masked layer of the model, replayed ALONE through the CUDA kernels on the tensors of the oracle's real
  train step: its stored (bf16) input activation x and the stored (bf16) gradient dy of its output.  Independent
  of how the network amplifies perturbations, so the bounds are tight:
    fprop / dgrad (bf16 outputs): relative L2 <= 1e-3 -- the two sides round fp32 accumulators that differ in
      summation order, so a small fraction of elements lands on the neighbouring bf16 value;
    DENSE wgrad (fp32 accumulators, identical bf16 operands): relative L2 <= 2e-5, the north-star's 1e-5-class
      bound."""
  out = {}
  for l in model.registry.layers():
    x, y, stride, padding = net.record[l.scope]
    dy = y.grad.to(torch.bfloat16).float()                  # the storage rounding of that gradient
    w = net.last_masked[l.scope].detach()
    want_dense = net.last_masked[l.scope].grad               # the oracle's dense gradient of this step
    if padding == 'LINEAR':
      xd = x.detach().to(DEV).to(torch.bfloat16).requires_grad_(True)
      l.masked_weights.fresh = False
      yd = l(xd)
      yd.backward(dy.to(DEV).to(yd.dtype))
      got_y, got_dx = yd.detach().float().cpu(), xd.grad.float().cpu()
      want_y = y.detach()                                      # (fp32 logits, bias included on both sides)
      want_dx = dy @ w.t()
    else:
      xd = _nhwc_dev(x).requires_grad_(x.requires_grad)
      l.masked_weights.fresh = False
      yd = l(xd)
      yd.backward(_nhwc_dev(dy))
      got_y = yd.detach().float().cpu()
      got_dx = xd.grad.float().cpu() if xd.grad is not None else None
      want_y = y.detach()
      xl = x.detach().clone().requires_grad_(True)
      want_dx, = torch.autograd.grad(cpu._conv_tf(xl, w, stride, padding), xl, dy)
    got_dense = l.masked_weights.dense_grad.view(l.weight.shape).cpu()
    e_y = _rel_l2(got_y.numpy(), want_y.numpy())
    e_dw = _rel_l2(got_dense.numpy(), want_dense.numpy())
    e_dx = _rel_l2(got_dx.numpy(), want_dx.to(torch.bfloat16).float().numpy()) if got_dx is not None else 0.0
    out[l.scope] = (e_y, e_dx, e_dw)
    assert e_y <= tol_act, 'fprop of %s on the step tensors: rel L2 %.2e' % (l.scope, e_y)
    assert e_dx <= tol_act, 'dgrad of %s on the step tensors: rel L2 %.2e' % (l.scope, e_dx)
    assert e_dw <= tol_dense, 'dense wgrad of %s on the step tensors: rel L2 %.2e' % (l.scope, e_dw)
  return out


def _compare_step(tag, model, net, images, labels, harness, loss_tol, grad_tol, label_smoothing, last_layers=None):
  """last_layers: bound the free-running dense gradients of only the last N masked layers (a plain feed-forward
  BN stack such as MobileNet-v1 amplifies rounding flips ~1.2x per layer with nothing to damp them: the early
  layers' free-running figures are recorded, not bounded; their kernels are bounded by the teacher-forced pass)."""
  x32 = images.float()
  net.record = {}
  want_loss, want_dense = net.forward_backward(x32, labels) if label_smoothing is None else \
      net.forward_backward(x32, labels, label_smoothing=label_smoothing)
  _load(model, net)
  # (1) every masked layer alone, on the tensors of this step: tight bounds
  forced = _teacher_forced_layers(model, net)
  for l in model.registry.layers():
    l.weight.grad = None                  # (the replay left masked gradients behind; the step below owns them)
  # (2) the free-running step: bounded by how the network amplifies rounding flips (see the module docstring)
  xd = images.to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  yd = labels.to(DEV)
  got_loss = float(harness._forward_backward(xd, yd, set_to_none=False).detach())
  torch.cuda.synchronize()
  rel = {}
  for l in model.registry.layers():
    got = l.masked_weights.dense_grad.view(l.weight.shape).cpu().numpy()
    want = want_dense[l.scope].numpy()
    rel[l.scope] = _rel_l2(got, want)
    # masked gradient = mask * dense, exactly (with the fused inner optimizer it is formed inside the step kernel
    # and never materialised: see the optimizer-step check in _check_update_steps)
    if l.weight.grad is not None:
      m = net.m[l.scope].numpy()
      assert np.array_equal(l.weight.grad.cpu().numpy(), got * m), l.scope
  bounded = dict(list(rel.items())[-last_layers:]) if last_layers else rel
  worst = max(bounded, key=bounded.get)
  _record(tag, dict(loss_cuda=got_loss, loss_oracle=want_loss, rel_l2=rel, worst=worst,
                    teacher_forced={k: list(v) for k, v in forced.items()}))
  assert abs(got_loss - want_loss) <= loss_tol * abs(want_loss), (got_loss, want_loss)
  assert bounded[worst] <= grad_tol, 'dense grad of %s: rel L2 %.4f (median %.4f)' % (
      worst, bounded[worst], float(np.median(list(rel.values()))))
  return rel


def _check_update_steps(model, harness, images, labels, n_steps, expect_updates):
  """Runs `n_steps` public train steps; at every mask-update step the oracle's drop/grow on the SAME dense
  gradients / noise must reproduce masks, weights and momentum slots bit for bit."""
  xd = images.to(DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  yd = labels.to(DEV)
  layers = model.registry.layers()
  updates = []
  for step in range(n_steps):
    before = []
    for l in layers:
      st = harness.inner.state.get(l.weight, {})
      mom = st.get('momentum_buffer')
      before.append((l.mask.numpy().copy(), l.weight.detach().cpu().numpy().copy(),
                     None if mom is None else mom.detach().cpu().numpy().copy()))
    gs = harness.global_step.value
    harness.step(xd, yd)
    torch.cuda.synchronize()
    if not harness.opt.last_update_was_mask_update:
      assert harness.global_step.value == gs + 1
      # the optimizer step on THESE gradients: Nesterov momentum on mask * dense + wd * w (SURVEY Appendix C)
      group = harness.inner.param_groups[0]
      for l, (m0, w0, mom0) in zip(layers, before):
        dense = l.masked_weights.dense_grad.view(l.weight.shape).cpu().numpy()
        g = (m0 * dense + np.float32(group['weight_decay']) * w0).astype(np.float32)
        w_want, mom_want = orc.momentum_step(w0, np.zeros_like(w0) if mom0 is None else mom0, g, group['lr'],
                                             group['momentum'], True)
        w_got = l.weight.detach().cpu().numpy()
        mom_got = harness.inner.state[l.weight]['momentum_buffer'].cpu().numpy()
        assert np.allclose(mom_got, mom_want, rtol=1e-5, atol=1e-7 * float(np.abs(mom_want).max() + 1e-30)), l.scope
        assert np.allclose(w_got, w_want, rtol=1e-5, atol=1e-6 * float(np.abs(w_want).max())), l.scope
      continue
    assert harness.global_step.value == gs            # RigL: no optimizer step on update iterations
    updates.append(gs)
    frac = np.float32(harness.opt.drop_fraction)
    for l, (m0, w0, mom0) in zip(layers, before):
      dense = l.masked_weights.dense_grad.view(l.weight.shape).cpu().numpy()
      noise = harness.opt.last_update_noise(l.weight).view(l.weight.shape).cpu().numpy()   # what the kernels drew
      want = orc.rigl_mask_update(m0, w0, dense, frac, noise=noise, slots=[] if mom0 is None else [mom0])
      assert np.array_equal(l.mask.numpy(), want['mask']), (gs, l.scope)
      assert l.weight.detach().cpu().numpy().tobytes() == want['weights'].tobytes(), (gs, l.scope)
      if mom0 is not None:
        got_mom = harness.inner.state[l.weight]['momentum_buffer'].cpu().numpy()
        assert got_mom.tobytes() == want['slots'][0].tobytes(), (gs, l.scope)
  assert updates == expect_updates, updates


def test_resnet50_step_vs_cpu_oracle():
  torch.manual_seed(0)
  net = cpu.CpuResNet50(sparsity=0.8, seed=11, bf16_weights=True)
  net.bn_init, net.bf16_act = _bn_init(11, last_bn_gain=0.1), True
  model = workloads.ResNet50(device=DEV)
  images = torch.randn(8, 3, 64, 64).to(torch.bfloat16)
  labels = torch.randint(0, 1000, (8,))
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  _compare_step('resnet50', model, net, images, labels, h, loss_tol=2e-2, grad_tol=0.5, label_smoothing=None)
  _check_update_steps(model, h, images, labels, 4, [0, 2])


def test_wrn22_2_step_vs_cpu_oracle():
  torch.manual_seed(1)
  net = cpu.CpuWideResNet(depth=22, width=2, sparsity=0.95, seed=12, bf16_weights=True)
  net.bn_init, net.bf16_act = _bn_init(12), True
  model = workloads.WideResNet(depth=22, width=2, droprate=0.0, device=DEV)
  with torch.no_grad():
    model.conv_1.weight.copy_(net.p['conv_1'].detach().permute(3, 2, 0, 1).to(DEV))
  images = torch.randn(16, 3, 32, 32).to(torch.bfloat16)
  labels = torch.randint(0, 10, (16,))
  h = workloads.TrainHarness(model, lr=0.05, weight_decay=5e-4, label_smoothing=0.0, frequency=2, end_step=100)
  _compare_step('wrn22_2', model, net, images, labels, h, loss_tol=2e-2, grad_tol=0.25, label_smoothing=0.0)
  _check_update_steps(model, h, images, labels, 4, [0, 2])


def test_mobilenet_v1_step_vs_cpu_oracle():
  torch.manual_seed(2)
  net = cpu.CpuMobileNetV1(sparsity=0.9, seed=13, bf16_weights=True)
  net.bn_init, net.bf16_act = _bn_init(13), True
  model = workloads.MobileNetV1(device=DEV)
  with torch.no_grad():
    model.initial_conv.weight.copy_(net.p['initial_conv'].detach().permute(3, 2, 0, 1).to(DEV))
    for i, blk in enumerate(model.blocks):
      blk.depthwise.weight.copy_(net.p['depthwise_%d' % i].detach().to(DEV))
  images = torch.randn(8, 3, 64, 64).to(torch.bfloat16)
  labels = torch.randint(0, 1000, (8,))
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100)
  _compare_step('mobilenet_v1', model, net, images, labels, h, loss_tol=2e-2, grad_tol=0.6, label_smoothing=0.1,
                last_layers=2)
  _check_update_steps(model, h, images, labels, 4, [0, 2])
