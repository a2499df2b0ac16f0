"""CPU restatement of the reference's sparse ResNet-50 train step -- TEST / BASELINE
INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/rigl_oracle.py header).

What the reference executes per step on its CPU path (TF1 graph; SURVEY 3a):
  masked_weights = mask * weights (dense fp32 tensor, every step)
  fwd: conv(x, masked_weights) for 53 convs + BN/ReLU/pool + masked FC
  bwd: TWO gradient sets -- wrt `weights` (masked) and wrt `masked_weights` (DENSE,
       sparse_optimizers_base.py:478-485; TF1 cond semantics compute it every step)
  then either the Nesterov-momentum step or, on update iterations, the drop/grow
  update (two full sorts per layer, base.py:276-343).
TensorFlow is not installable here, so this is a torch-CPU port of that math
(fp32, dense-executed like TF's Eigen kernels), used as `cpu_baseline` (kind
"port") and by `bench.py --impl reference`.  Parity: unpinned against TF itself.
"""
import time

import numpy as np
import torch
import torch.nn.functional as F

from . import rigl_oracle as orc


def _bf16_round(a):
  return torch.from_numpy(np.asarray(a, np.float32)).to(torch.bfloat16).float()


def max_pool_same(x, k=3, s=2):
  """tf.layers.max_pooling2d(padding='SAME') (resnet_model.py:636-642) on NCHW: TensorFlow pads
  pad_total // 2 before and the rest AFTER (for even inputs and k=3, s=2: nothing before, one after)."""
  h, w = x.shape[2:]
  _, ph0, ph1 = orc.tf_same_padding(h, k, s)
  _, pw0, pw1 = orc.tf_same_padding(w, k, s)
  return F.max_pool2d(F.pad(x, (pw0, pw1, ph0, ph1), value=float('-inf')), k, s, 0)


class _RoundBf16(torch.autograd.Function):
  """x -> bf16(x) in the forward pass, g -> bf16(g) in the backward pass: the storage rounding of an activation
  tensor (and of its gradient) on the bf16 training path of BASELINE C2-C5."""

  @staticmethod
  def forward(ctx, x):
    return x.to(torch.bfloat16).float()

  @staticmethod
  def backward(ctx, g):
    return g.to(torch.bfloat16).float()


class _RoundGradBf16(torch.autograd.Function):
  """identity forward, g -> bf16(g) backward (the fp32 logits: the device casts dL/dlogits to bf16 before the
  classifier's dgrad / wgrad GEMMs)."""

  @staticmethod
  def forward(ctx, x):
    return x.view_as(x)

  @staticmethod
  def backward(ctx, g):
    return g.to(torch.bfloat16).float()


class _CpuNet(object):
  """Shared pieces: masked weights / masks / momentum slots by reference variable scope, batch-norm
  parameters in execution order (`self.bn_order`), dense (un-masked) parameters in `self.p`."""

  def _init_masked(self, layers, sparsities, rng, bf16_weights):
    self.w, self.m, self.mom = {}, {}, {}
    for n, sh in layers:
      fan_in = int(np.prod(sh[:-1]))
      w = (rng.standard_normal(sh) * np.sqrt(2.0 / fan_in)).astype(np.float32)
      self.w[n] = _bf16_round(w) if bf16_weights else torch.from_numpy(w)
      self.m[n] = torch.from_numpy(orc.get_mask_random_numpy(sh, sparsities[n + '/mask:0'], rng).astype(np.float32))
      self.mom[n] = torch.zeros(sh)
    self.bn, self.bn_order, self.p = {}, [], {}
    self.bn_init = None          # optional callable(key, channels) -> (gamma, beta) numpy
    self.trace = None            # optional list: receives (key, BN output) in execution order (debugging)
    # bf16_activations: every activation tensor the GPU path stores (conv outputs, BN / ReLU / residual outputs,
    # pooled features) and its gradient are rounded to bf16 at the same points; arithmetic inside an op stays fp32.
    # This is the bf16 configuration BASELINE.json names; False = the reference's fp32 CPU path (the timing port).
    # A 50-layer batch-normalised network at initialisation amplifies ANY perturbation by ~1.2x per layer
    # (tools/noise_growth.py), so only an oracle that rounds where the device rounds can be
    # compared layer by layer with it.
    self.bf16_act = False

    # record: optional dict name -> (input, stored output) of every masked layer of the last forward pass, both
    # kept with their gradients (tests replay single layers of a real step through the CUDA kernels)
    self.record = None

  def q(self, x):
    return _RoundBf16.apply(x) if self.bf16_act else x

  def mconv(self, x, name, masked, stride, padding):
    """Masked conv `name` on x + storage rounding of its output."""
    y = self.q(_conv_tf(x, masked[name], stride, padding))
    if self.record is not None:
      if x.requires_grad:
        x.retain_grad()
      y.retain_grad()
      self.record[name] = (x, y, stride, padding)
    return y

  def mlinear(self, x, name, masked, bias):
    y = x @ masked[name] + bias
    if self.record is not None:
      if x.requires_grad:
        x.retain_grad()
      y.retain_grad()
      self.record[name] = (x, y, 1, 'LINEAR')
    return y

  def _bn(self, x, key, relu=True, eps=1e-5, store=True):
    """store=False: the BN output is not materialised on the device (it is consumed by a fused residual add)."""
    c = x.shape[1]
    if key not in self.bn:
      g, b = (np.ones(c, np.float32), np.zeros(c, np.float32)) if self.bn_init is None else self.bn_init(key, c)
      self.bn[key] = (torch.tensor(g, requires_grad=True), torch.tensor(b, requires_grad=True))
      self.bn_order.append(key)
    g, b = self.bn[key]
    x = F.batch_norm(x, None, None, g, b, training=True, momentum=0.1, eps=eps)
    x = F.relu(x) if relu else x
    if store:
      x = self.q(x)
    if self.trace is not None:
      self.trace.append((key, x.detach()))
    return x

  def _masked(self):
    return {n: (self.m[n] * self.w[n]).requires_grad_(True) for n in self.w}      # materialised every step

  def _finish(self, logits, labels, masked, label_smoothing):
    if self.bf16_act:
      logits = _RoundGradBf16.apply(logits)
    self.last_masked = masked
    for t in list(self.p.values()) + [v for gb in self.bn.values() for v in gb]:
      t.grad = None
    loss = F.cross_entropy(logits, labels, label_smoothing=label_smoothing)
    loss.backward()
    return float(loss.detach()), {n: masked[n].grad for n in self.w}

  def optimizer_step(self, dense, lr=0.1, momentum=0.9, wd=1e-4):
    for n in self.w:
      g = self.m[n] * dense[n] + wd * self.w[n]              # dL/dweights + l2 on raw weights
      self.mom[n].mul_(momentum).add_(g)
      self.w[n].sub_(lr * (g + momentum * self.mom[n]))

  def mask_update(self, dense, drop_fraction=0.3):
    for n in self.w:
      r = orc.rigl_mask_update(self.m[n].numpy(), self.w[n].numpy(), dense[n].numpy(), drop_fraction,
                               slots=[self.mom[n].numpy()])
      self.m[n] = torch.from_numpy(r['mask'])
      self.w[n] = torch.from_numpy(r['weights'])
      self.mom[n] = torch.from_numpy(r['slots'][0])


def _conv_tf(x, w_hwio, stride, padding):
  """conv with the reference's three paddings on NCHW input / HWIO weights: 'FIXED' = conv2d_fixed_padding
  (resnet_model.py:234-303: explicit (k-1)//2 both sides then VALID), 'SAME' = TensorFlow SAME (asymmetric
  for stride 2 on even inputs; cifar_resnet/resnet_model.py:158-181), 'VALID'."""
  k = w_hwio.shape[0]
  wt = w_hwio.permute(3, 2, 0, 1)
  if padding == 'FIXED':
    return F.conv2d(x, wt, stride=stride, padding=(k - 1) // 2)
  if padding == 'VALID':
    return F.conv2d(x, wt, stride=stride)
  _, ph0, ph1 = orc.tf_same_padding(x.shape[2], k, stride)
  _, pw0, pw1 = orc.tf_same_padding(x.shape[3], k, stride)
  return F.conv2d(F.pad(x, (pw0, pw1, ph0, ph1)), wt, stride=stride)


class CpuResNet50(_CpuNet):

  def __init__(self, sparsity=0.8, seed=0, num_classes=1000, bf16_weights=False):
    rng = np.random.RandomState(seed)
    self.layers = orc.resnet50_masked_layers()
    if num_classes != 1000:
      self.layers[-1] = (self.layers[-1][0], (2048, num_classes)) + tuple(self.layers[-1][2:])
    masks = [orc.FakeMask(n + '/mask:0', sh) for n, sh, _, _ in self.layers]
    sp = orc.get_sparsities(masks, 'erdos_renyi_kernel', sparsity, {})
    self._init_masked([(n, sh) for n, sh, _, _ in self.layers], sp, rng, bf16_weights)
    self.fc_bias = torch.zeros(num_classes)

  def _conv(self, x, name, masked, stride):
    return self.mconv(x, name, masked, stride, 'FIXED')

  def forward_backward(self, images, labels):
    """Returns (loss, dense grads dict).  images [N,3,H,W] fp32."""
    masked = self._masked()
    p = 'resnet_model/'
    x = self._bn(self._conv(images, p + 'initial_conv', masked, 2), 'bn0')
    x = max_pool_same(x, 3, 2)
    for g, (n_blocks, stride) in enumerate(((3, 1), (4, 2), (6, 2), (3, 2)), 1):
      for b in range(n_blocks):
        sfx = ('block_group_projection_block_group%d' % g) if b == 0 else ('block_group%d_%d_1' % (g, b))
        s = stride if b == 0 else 1
        sc = x
        if b == 0:
          sc = self._bn(self._conv(x, p + 'bottleneck_projection_' + sfx, masked, s), sfx + 'p', relu=False)
        y = self._bn(self._conv(x, p + 'bottleneck_1_' + sfx, masked, 1), sfx + '1')
        y = self._bn(self._conv(y, p + 'bottleneck_2_' + sfx, masked, s), sfx + '2')
        y = self._bn(self._conv(y, p + 'bottleneck_3_' + sfx, masked, 1), sfx + '3', relu=False, store=False)
        x = self.q(F.relu(y + sc))              # relu(BN(conv3) + shortcut): ONE fused kernel, one rounding
    x = self.q(x.mean(dim=(2, 3)))
    logits = self.mlinear(x, p + 'final_dense', masked, self.fc_bias)
    return self._finish(logits, labels, masked, 0.1)


class CpuWideResNet(_CpuNet):
  """WRN-(6n+4)-k of cifar_resnet/resnet_model.py:70-235 (BASELINE C5: depth 22, width 2, 95 % ERK): `conv_1`
  dense (prune_first_layer False), pre-activation residual blocks, 3x3 convs TF 'SAME', the 1x1 skip conv 'VALID'
  with the block stride and fed the PRE-ACTIVATED input, BN momentum 0.9 / eps 1e-5; dropout is the caller's
  business (rate 0 here: the parity tests and the timing port run without it)."""

  def __init__(self, depth=22, width=2, sparsity=0.95, seed=0, num_classes=10, bf16_weights=False):
    rng = np.random.RandomState(seed)
    n_blocks = (depth - 4) // 6
    self.blocks, layers, cin = [], [], 16
    for name, size, subsample in (('conv_2', 16 * width, False), ('conv_3', 32 * width, True),
                                  ('conv_4', 64 * width, True)):
      for n in range(n_blocks):
        stride = 2 if (subsample and n == 0) else 1
        skip = None
        if cin != size:
          skip = 'resnet_model/skip_%s' % name
          layers.append((skip, (1, 1, cin, size)))
        a, b = 'resnet_model/%s_%d_1' % (name, n), 'resnet_model/%s_%d_2' % (name, n)
        layers += [(a, (3, 3, cin, size)), (b, (3, 3, size, size))]
        self.blocks.append((skip, a, b, stride))
        cin = size
    layers.append(('resnet_model/logits', (cin, num_classes)))
    masks = [orc.FakeMask(n + '/mask:0', sh) for n, sh in layers]
    sp = orc.get_sparsities(masks, 'erdos_renyi_kernel', sparsity, {})
    self._init_masked(layers, sp, rng, bf16_weights)
    c1 = (rng.standard_normal((3, 3, 3, 16)) * np.sqrt(2.0 / 27)).astype(np.float32)
    self.p['conv_1'] = (_bf16_round(c1) if bf16_weights else torch.from_numpy(c1)).requires_grad_(True)
    self.p['logits_bias'] = torch.zeros(num_classes, requires_grad=True)

  def forward_backward(self, images, labels, label_smoothing=0.0):
    masked = self._masked()
    net = self.q(_conv_tf(images, self.p['conv_1'], 1, 'SAME'))
    for i, (skip_name, a, b, stride) in enumerate(self.blocks):
      skip = net
      net = self._bn(net, 'b%d_a' % i)
      if skip_name is not None:
        skip = self.mconv(net, skip_name, masked, stride, 'VALID')
      net = self.mconv(net, a, masked, stride, 'SAME')
      net = self._bn(net, 'b%d_b' % i)
      net = self.q(self.mconv(net, b, masked, 1, 'SAME') + skip)
    net = self._bn(net, 'final')
    logits = self.mlinear(self.q(net.mean(dim=(2, 3))), 'resnet_model/logits', masked, self.p['logits_bias'])
    return self._finish(logits, labels, masked, label_smoothing)


class CpuMobileNetV1(_CpuNet):
  """MobileNet-v1 as mobilenetv1_model.py:156-342 sparsifies it (BASELINE C4): the 13 pointwise 1x1 convs and
  `final_dense` are masked; `initial_conv` (3x3/2, fixed padding) and the depthwise 3x3 convs are dense."""

  CFG = ((64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1),
         (512, 1), (1024, 2), (1024, 1))

  def __init__(self, sparsity=0.9, seed=0, num_classes=1000, bf16_weights=False):
    rng = np.random.RandomState(seed)
    layers, cin = [], 32
    for i, (f, _) in enumerate(self.CFG):
      layers.append(('resnet_model/contraction_1x1_%d' % i, (1, 1, cin, f)))
      cin = f
    layers.append(('resnet_model/final_dense', (cin, num_classes)))
    sp = {n + '/mask:0': sparsity for n, _ in layers}
    self._init_masked(layers, sp, rng, bf16_weights)
    rnd = (lambda a: _bf16_round(a)) if bf16_weights else (lambda a: torch.from_numpy(a))
    self.p['initial_conv'] = rnd((rng.standard_normal((3, 3, 3, 32)) * np.sqrt(2.0 / 27)).astype(np.float32)) \
        .requires_grad_(True)
    cin = 32
    for i, (f, _) in enumerate(self.CFG):
      self.p['depthwise_%d' % i] = rnd((rng.standard_normal((cin, 1, 3, 3)) * np.sqrt(2.0 / 9)).astype(np.float32)) \
          .requires_grad_(True)                                   # torch depthwise layout [C,1,3,3]
      cin = f
    self.p['final_bias'] = torch.zeros(num_classes, requires_grad=True)

  def forward_backward(self, images, labels, label_smoothing=0.1):
    masked = self._masked()
    x = self._bn(self.q(_conv_tf(images, self.p['initial_conv'], 2, 'FIXED')), 'bn0')
    for i, (f, stride) in enumerate(self.CFG):
      x = self.q(F.conv2d(x, self.p['depthwise_%d' % i], stride=stride, padding=1, groups=x.shape[1]))
      x = self._bn(x, 'dw%d' % i)
      x = self._bn(self.mconv(x, 'resnet_model/contraction_1x1_%d' % i, masked, 1, 'FIXED'), 'pw%d' % i)
    logits = self.mlinear(self.q(x.mean(dim=(2, 3))), 'resnet_model/final_dense', masked, self.p['final_bias'])
    return self._finish(logits, labels, masked, label_smoothing)


def time_train_steps_model(model, batch, steps, warmup=1, image_hw=224, sparsity=0.8, seed=0):
  """Seconds per train step (EVERY timed step, in order) of the CPU port of `model`
  ('resnet50' | 'wrn22_2' | 'mobilenet_v1') at `batch` images; also returns the net and its last dense grads."""
  torch.manual_seed(seed)
  if model == 'resnet50':
    net, classes, kw, opt = CpuResNet50(sparsity=sparsity, seed=seed), 1000, {}, dict(wd=1e-4)
  elif model == 'wrn22_2':
    net, classes, kw, opt = CpuWideResNet(sparsity=sparsity, seed=seed), 10, {}, dict(wd=5e-4)
  elif model == 'mobilenet_v1':
    net, classes, kw, opt = CpuMobileNetV1(sparsity=sparsity, seed=seed), 1000, {}, dict(wd=1e-4)
  else:
    raise ValueError(model)
  images = torch.randn(batch, 3, image_hw, image_hw)
  labels = torch.randint(0, classes, (batch,))
  times = []
  dense = None
  for i in range(warmup + steps):
    t0 = time.perf_counter()
    _, dense = net.forward_backward(images, labels, **kw)
    net.optimizer_step(dense, **opt)
    dt = time.perf_counter() - t0
    if i >= warmup:
      times.append(dt)
  return times, net, dense


def time_train_steps(batch, steps, warmup=1, image_hw=224, sparsity=0.8, seed=0):
  """Median seconds per ResNet-50 train step (kept for callers of the round-1 signature)."""
  times, net, dense = time_train_steps_model('resnet50', batch, steps, warmup, image_hw, sparsity, seed)
  return float(np.median(times)), net, dense


def time_mask_update(net, dense, repeats=1):
  times = []
  for _ in range(repeats):
    t0 = time.perf_counter()
    net.mask_update(dense, 0.3)
    times.append(time.perf_counter() - t0)
  return float(np.median(times))
