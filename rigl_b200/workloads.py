"""Workload definitions for the hot path: the masked-layer graphs of the
reference's models, built on rigl_b200.layers, plus the train-step harness.

Only what BASELINE.json's configs need -- the shapes, variable names and wiring
that the masked conv/linear kernels and the RigL update run on:
  ResNet50   rigl/imagenet_resnet/resnet_model.py:396-731 (v1.5: stride on the 3x3;
             BN after every conv, zero-init gamma on the last BN of a block)
  ResNet     rigl/imagenet_resnet/resnet_model.py:577-805 (resnet_v1_: depths 18-200, width, prune flags)
  MnistFC    rigl/mnist/mnist_train_eval.py:112-160 (784-300-100-10, all masked)
  MobileNetV2 rigl/imagenet_resnet/mobilenetv2_model.py (inverted residual blocks, linear bottlenecks)
  VGG        rigl/imagenet_resnet/vgg.py (vgg_a / vgg_16 / vgg_19: 3x3 convs + ReLU, no BN; ReLU in the conv epilogues)
BN+ReLU(+residual) run on the fused streaming kernels of csrc/bn.cu (SURVEY 8f row 1);
pooling / loss are stock PyTorch kernels over channels_last bf16 tensors.
"""
import math

import numpy as np
import torch
from torch import nn
import torch.nn.functional as F

from . import pruning
from . import sparse_utils
from .layers import SparseConv2d, SparseLinear, variance_scaling_
from .norm import FusedBatchNormReLU, max_pool2x2_relu, max_pool_same, relu_grad_gate
from .sparse_optimizers import SparseRigLOptimizer
from .sparse_optimizers_base import GlobalStep

BATCH_NORM_DECAY = 0.9
BATCH_NORM_EPSILON = 1e-5


class DenseConv2d(nn.Conv2d):
  """An un-masked conv of the reference models (WRN `conv_1`, MobileNet `initial_conv` / depthwise): float32
  master weights like every TF variable, bf16 compute (stock cuDNN kernels -- not a masked op)."""

  def forward(self, x):
    return F.conv2d(x, self.weight.to(torch.bfloat16), None, self.stride, self.padding, self.dilation, self.groups)


def _BNReLU(channels, relu=True, init_zero=False, device='cuda'):
  """batch_norm_relu (resnet_model.py:41-80) on the fused streaming kernels (csrc/bn.cu)."""
  return FusedBatchNormReLU(channels, relu=relu, init_zero=init_zero, eps=BATCH_NORM_EPSILON,
                            decay=BATCH_NORM_DECAY, device=device)


def conv_bn(conv, bn, x, residual=None, fork=False):
  """bn(conv(x), residual) for a SparseConv2d `conv` feeding the FusedBatchNormReLU `bn` (`fork` as
  FusedBatchNormReLU.forward takes it).  In the inference form (conv.bn_fusable(bn): eval mode, no autograd,
  layers.FUSE_BN_INFER) the BN, residual add and ReLU run in the conv's epilogue where its kernel has one; otherwise
  -- training included -- exactly the launches of bn(conv(x), producer=conv), whose epilogue may emit the BN
  statistics.  Both modules are called, so their forward hooks fire."""
  if conv.bn_fusable(bn):
    return bn(conv(x, bn=bn, residual=residual), applied=True, fork=fork)
  return bn(conv(x), residual=residual, producer=conv, fork=fork)


# Block outputs are handed to their two consumers as two handles so that the gradient sum happens
# inside the BN backward kernel (rigl_bn_backward) rather than in a separate elementwise add.
FORK_BLOCK_OUTPUTS = True


class _Bottleneck(nn.Module):

  def __init__(self, cin, filters, strides, use_projection, name, device, registry):
    super(_Bottleneck, self).__init__()
    mk = lambda ci, co, k, s, n: SparseConv2d(ci, co, k, strides=s, padding='FIXED', name='resnet_model/' + n,
                                              device=device, registry=registry)
    self.proj = None
    if use_projection:
      self.proj = mk(cin, 4 * filters, 1, strides, 'bottleneck_projection_%s' % name)
      self.proj_bn = _BNReLU(4 * filters, relu=False, device=device)
    self.conv1 = mk(cin, filters, 1, 1, 'bottleneck_1_%s' % name)
    self.bn1 = _BNReLU(filters, device=device)
    self.conv2 = mk(filters, filters, 3, strides, 'bottleneck_2_%s' % name)
    self.bn2 = _BNReLU(filters, device=device)
    self.conv3 = mk(filters, 4 * filters, 1, 1, 'bottleneck_3_%s' % name)
    for conv in (self.proj, self.conv1, self.conv2, self.conv3):
      if conv is not None:
        conv.collect_bn_stats = True
    # last BN of the block: zero-init gamma; the residual add + final ReLU are fused into it
    self.bn3 = _BNReLU(4 * filters, relu=True, init_zero=True, device=device)

  def forward(self, x, x_skip=None, fork=False):
    """`x` feeds conv1, `x_skip` (the same activation, second handle) the shortcut branch; with
    `fork` the block output comes back as two handles as well (see FusedBatchNormReLU.forward)."""
    # every conv feeds a BN: its epilogue emits that BN's batch statistics (producer=...)
    if x_skip is None:
      x_skip = x
    shortcut = x_skip if self.proj is None else conv_bn(self.proj, self.proj_bn, x_skip)
    y = conv_bn(self.conv1, self.bn1, x)
    y = conv_bn(self.conv2, self.bn2, y)
    return conv_bn(self.conv3, self.bn3, y, residual=shortcut, fork=fork)   # relu(BN(conv3) + shortcut)


class ResNet50(nn.Module):
  """ResNet-50 with every conv and the classifier masked (54 masked tensors,
  names = the reference variable scopes, SURVEY Appendix A)."""

  def __init__(self, num_classes=1000, device='cuda', registry=None):
    super(ResNet50, self).__init__()
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg = self.registry
    self.initial_conv = SparseConv2d(3, 64, 7, strides=2, padding='FIXED', name='resnet_model/initial_conv',
                                     device=device, registry=reg)
    self.initial_bn = _BNReLU(64, device=device)
    self.initial_conv.collect_bn_stats = True
    blocks = []
    cin = 64
    for g, (filters, n_blocks, stride) in enumerate(((64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)), 1):
      blocks.append(_Bottleneck(cin, filters, stride, True, 'block_group_projection_block_group%d' % g,
                                device, reg))
      cin = 4 * filters
      for b in range(1, n_blocks):
        blocks.append(_Bottleneck(cin, filters, 1, False, 'block_group%d_%d_1' % (g, b), device, reg))
    self.blocks = nn.ModuleList(blocks)
    self.final_dense = SparseLinear(
        2048, num_classes, name='resnet_model/final_dense', device=device, registry=reg,
        out_dtype=torch.float32,
        kernel_initializer=lambda w: w.normal_(0., .01))      # resnet_model.py:713

  def forward(self, x):
    x = conv_bn(self.initial_conv, self.initial_bn, x)
    x = max_pool_same(x, 3, 2)                      # 'SAME' 3x3/2 pool, resnet_model.py:636-642
    x_skip, last = x, len(self.blocks) - 1
    for i, blk in enumerate(self.blocks):
      if i < last and FORK_BLOCK_OUTPUTS:
        x, x_skip = blk(x, x_skip, fork=True)
      else:
        x = blk(x, x_skip)
        x_skip = x
    x = x.mean(dim=(2, 3))
    return self.final_dense(x)


class _Residual(nn.Module):
  """residual_block_ (resnet_model.py:306-403), the basic block of ResNet-18 / 34: two 3x3 convs, the first one
  strided, BN after each; the last BN has zero-init gamma and takes the residual add + final ReLU, in the form of
  _Bottleneck.bn3."""

  def __init__(self, cin, filters, strides, use_projection, name, device, registry):
    super(_Residual, self).__init__()
    mk = lambda ci, co, k, s, n: SparseConv2d(ci, co, k, strides=s, padding='FIXED', name='resnet_model/' + n,
                                              device=device, registry=registry)
    self.proj = None
    if use_projection:
      self.proj = mk(cin, filters, 1, strides, 'residual_projection_%s' % name)
      self.proj_bn = _BNReLU(filters, relu=False, device=device)
    self.conv1 = mk(cin, filters, 3, strides, 'residual_1_%s' % name)
    self.bn1 = _BNReLU(filters, device=device)
    self.conv2 = mk(filters, filters, 3, 1, 'residual_2_%s' % name)
    for conv in (self.proj, self.conv1, self.conv2):
      if conv is not None:
        conv.collect_bn_stats = True
    self.bn2 = _BNReLU(filters, relu=True, init_zero=True, device=device)

  def forward(self, x, x_skip=None, fork=False):
    """As _Bottleneck.forward: `x_skip` is the shortcut's handle of the input, `fork` returns two handles."""
    if x_skip is None:
      x_skip = x
    shortcut = x_skip if self.proj is None else conv_bn(self.proj, self.proj_bn, x_skip)
    y = conv_bn(self.conv1, self.bn1, x)
    return conv_bn(self.conv2, self.bn2, y, residual=shortcut, fork=fork)   # relu(BN(conv2) + shortcut)


# resnet_depth -> (block, blocks per group), resnet_model.py:777-802
RESNET_DEPTHS = {18: ('residual', (2, 2, 2, 2)), 34: ('residual', (3, 4, 6, 3)), 50: ('bottleneck', (3, 4, 6, 3)),
                 101: ('bottleneck', (3, 4, 23, 3)), 152: ('bottleneck', (3, 8, 36, 3)),
                 200: ('bottleneck', (3, 24, 36, 3))}


def resnet_plan(depth, width=1.0):
  """Channel plan of resnet_v1_(depth, width): (block kind 'residual' or 'bottleneck', initial_conv filters,
  [(block name, cin, filters, stride, projection)], final_dense inputs).  Block names are block_group's: the first
  block of group g is 'block_group_projection_block_group<g>' (projection shortcut, the group's stride -- group 1
  included, at stride 1), block b > 0 'block_group<g>_<b>_1'.  A bottleneck block's output has 4 * filters channels.
  Every width must be a multiple of 8 (the NHWC kernels move 8 channels per 16-byte vector); ValueError names the
  first layer that is not."""
  if depth not in RESNET_DEPTHS:
    raise ValueError('Not a valid resnet_depth: %r (one of %s)' % (depth, sorted(RESNET_DEPTHS)))
  kind, counts = RESNET_DEPTHS[depth]
  mult = 4 if kind == 'bottleneck' else 1
  prefix = 'bottleneck' if kind == 'bottleneck' else 'residual'

  def need8(c, layer):
    if c % 8:
      raise ValueError('ResNet(%d, width=%g): %s has %d channels, not a multiple of 8' % (depth, width, layer, c))
  c0 = int(64 * width)
  need8(c0, 'resnet_model/initial_conv')
  blocks, cin = [], c0
  for g, (base, n_blocks, stride) in enumerate(zip((64, 128, 256, 512), counts, (1, 2, 2, 2)), 1):
    filters = int(base * width)
    for b in range(n_blocks):
      name = 'block_group_projection_block_group%d' % g if b == 0 else 'block_group%d_%d_1' % (g, b)
      if b == 0:
        need8(mult * filters, 'resnet_model/%s_projection_%s' % (prefix, name))
      need8(filters, 'resnet_model/%s_1_%s' % (prefix, name))
      blocks.append((name, cin, filters, stride if b == 0 else 1, b == 0))
      cin = mult * filters
  return kind, c0, blocks, cin


class ResNet(nn.Module):
  """resnet_v1_(depth, num_classes, width, prune_first_layer, prune_last_layer) (resnet_model.py:577-805): ResNet-18
  / 34 on the basic block (_Residual), ResNet-50 / 101 / 152 / 200 on the bottleneck (_Bottleneck), every width
  int(c * width).  ResNet(50) builds ResNet50's scopes, shapes and modules in the same order, so it draws the same
  initial weights under one seed.  With prune_first_layer=False the 7x7/2 `initial_conv` is a dense conv, with
  prune_last_layer=False `final_dense` a dense fp32 layer with a zero bias; neither is masked, both keep the l2
  regularizer (evaluate.regularized_kernels), as in the reference."""

  def __init__(self, depth, num_classes=1000, width=1.0, prune_first_layer=True, prune_last_layer=True,
               device='cuda', registry=None):
    super(ResNet, self).__init__()
    kind, c0, plan, fc_in = resnet_plan(depth, width)     # (raises before any parameter exists)
    self.depth, self.width = depth, width
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg = self.registry
    self.prune_first_layer = bool(prune_first_layer)
    if self.prune_first_layer:
      self.initial_conv = SparseConv2d(3, c0, 7, strides=2, padding='FIXED', name='resnet_model/initial_conv',
                                       device=device, registry=reg)
      self.initial_conv.collect_bn_stats = True
    else:             # conv2d_fixed_padding with pruning_method 'baseline': not masked
      self.initial_conv = DenseConv2d(3, c0, 7, stride=2, padding=3, bias=False, device=device)
      variance_scaling_(self.initial_conv.weight.data.permute(2, 3, 1, 0))
    self.initial_bn = _BNReLU(c0, device=device)
    block = _Bottleneck if kind == 'bottleneck' else _Residual
    self.blocks = nn.ModuleList([block(cin, filters, stride, proj, name, device, reg)
                                 for name, cin, filters, stride, proj in plan])
    self.prune_last_layer = bool(prune_last_layer)
    if self.prune_last_layer:
      self.final_dense = SparseLinear(fc_in, num_classes, name='resnet_model/final_dense', device=device,
                                      registry=reg, out_dtype=torch.float32,
                                      kernel_initializer=lambda w: w.normal_(0., .01))
    else:             # sparse_fully_connected with sparsity_technique 'baseline' (tf.layers.dense): fp32, zero bias
      self.final_dense = nn.Linear(fc_in, num_classes, device=device)
      with torch.no_grad():
        self.final_dense.weight.normal_(0., .01)
        self.final_dense.bias.zero_()

  def forward(self, x):
    if self.prune_first_layer:
      x = conv_bn(self.initial_conv, self.initial_bn, x)
    else:
      x = self.initial_bn(self.initial_conv(x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)))
    x = max_pool_same(x, 3, 2)
    x_skip, last = x, len(self.blocks) - 1
    for i, blk in enumerate(self.blocks):
      if i < last and FORK_BLOCK_OUTPUTS:
        x, x_skip = blk(x, x_skip, fork=True)
      else:
        x = blk(x, x_skip)
        x_skip = x
    x = x.mean(dim=(2, 3))
    if not self.prune_last_layer:
      x = x.float()
    return self.final_dense(x)


class WideResNet(nn.Module):
  """Pre-activation WideResNet-(6n+4)-k, cifar_resnet/resnet_model.py:70-235 (BASELINE C5:
  depth 22, width 2).  `conv_1` (3x3x3x16) is a plain dense conv unless prune_first_layer
  (resnet_train_eval.py:96); residual 3x3 convs use TF 'SAME', the 1x1 skip convs 'VALID'
  with the block stride; dropout 0.3 between the two convs of a block."""

  def __init__(self, depth=22, width=2, num_classes=10, droprate=0.3, device='cuda', registry=None):
    super(WideResNet, self).__init__()
    if (depth - 4) % 6 != 0:
      raise ValueError('Depth of ResNet specified not sufficient.')
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg, n_blocks = self.registry, (depth - 4) // 6
    self.conv_1 = DenseConv2d(3, 16, 3, padding=1, bias=False, device=device)
    self.droprate = droprate
    blocks, cin = [], 16
    for name, size, subsample in (('conv_2', 16 * width, False), ('conv_3', 32 * width, True),
                                  ('conv_4', 64 * width, True)):
      for n in range(n_blocks):
        stride = 2 if (subsample and n == 0) else 1
        blk = nn.Module()
        blk.bn_a = _BNReLU(cin, device=device)
        blk.skip = None
        if cin != size:
          blk.skip = SparseConv2d(cin, size, 1, strides=stride, padding='VALID',
                                  name='resnet_model/skip_%s' % name, device=device, registry=reg)
        blk.conv_a = SparseConv2d(cin, size, 3, strides=stride, padding='SAME',
                                  name='resnet_model/%s_%d_1' % (name, n), device=device, registry=reg)
        blk.bn_b = _BNReLU(size, device=device)
        blk.conv_b = SparseConv2d(size, size, 3, strides=1, padding='SAME',
                                  name='resnet_model/%s_%d_2' % (name, n), device=device, registry=reg)
        blocks.append(blk)
        cin = size
    self.blocks = nn.ModuleList(blocks)
    self.final_bn = _BNReLU(cin, device=device)
    self.logits = SparseLinear(cin, num_classes, name='resnet_model/logits', device=device, registry=reg,
                               out_dtype=torch.float32)

  def forward(self, x):
    net = self.conv_1(x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
    for blk in self.blocks:
      skip = net
      net = blk.bn_a(net)
      if blk.skip is not None:
        skip = blk.skip(net)
      net = blk.conv_a(net)
      net = F.dropout(blk.bn_b(net), self.droprate, self.training)
      net = blk.conv_b(net) + skip
    net = self.final_bn(net)
    return self.logits(net.mean(dim=(2, 3)))


class MobileNetV1(nn.Module):
  """MobileNet-v1 as the reference sparsifies it (mobilenetv1_model.py:156-342, BASELINE C4):
  only the 13 pointwise 1x1 convs and `final_dense` are masked; `initial_conv` and the
  depthwise 3x3 convs are dense (stock grouped convs)."""

  CFG = ((64, 1), (128, 2), (128, 1), (256, 2), (256, 1), (512, 2), (512, 1), (512, 1), (512, 1), (512, 1),
         (512, 1), (1024, 2), (1024, 1))

  def __init__(self, num_classes=1000, device='cuda', registry=None):
    super(MobileNetV1, self).__init__()
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg = self.registry
    self.initial_conv = DenseConv2d(3, 32, 3, stride=2, padding=1, bias=False, device=device)
    self.initial_bn = _BNReLU(32, device=device)
    blocks, cin = [], 32
    for i, (filters, stride) in enumerate(self.CFG):
      blk = nn.Module()
      blk.depthwise = DepthwiseConv2d(cin, stride=stride, device=device)
      blk.bn_dw = _BNReLU(cin, device=device)
      blk.pointwise = SparseConv2d(cin, filters, 1, strides=1, padding='FIXED',
                                   name='resnet_model/contraction_1x1_%d' % i, device=device, registry=reg)
      blk.bn_pw = _BNReLU(filters, device=device)
      blocks.append(blk)
      cin = filters
    self.blocks = nn.ModuleList(blocks)
    self.final_dense = SparseLinear(cin, num_classes, name='resnet_model/final_dense', device=device,
                                    registry=reg, out_dtype=torch.float32)

  def forward(self, x):
    x = self.initial_bn(self.initial_conv(x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)))
    for blk in self.blocks:
      x = blk.bn_dw(blk.depthwise(x))
      x = conv_bn(blk.pointwise, blk.bn_pw, x)
    return self.final_dense(x.mean(dim=(2, 3)))


def _make_divisible(v, divisor=8, min_value=None):
  """mobilenetv2_model.py:33-40: round to a multiple of `divisor`, never more than 10 % down."""
  if min_value is None:
    min_value = divisor
  new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
  if new_v < 0.9 * v:
    new_v += divisor
  return new_v


def _trunc_variance_scaling_(t, fan_in, scale=1.0):
  """tf.variance_scaling_initializer(scale) with its other defaults: fan_in, truncated normal (|z| <= 2 sigma, the
  untruncated standard deviation divided by 0.8796... so the truncated one is sqrt(scale / fan_in))."""
  std = math.sqrt(scale / max(fan_in, 1)) / .87962566103423978
  with torch.no_grad():
    nn.init.trunc_normal_(t, 0., std, -2. * std, 2. * std)
  return t


def _hwio_init(w):
  return _trunc_variance_scaling_(w, int(np.prod(w.shape[:-1])))


# (filters, stride) of inverted_res_block 0..16, mobilenetv2_model.py:318-340
MOBILENET_V2_BLOCKS = ((16, 1), (24, 2), (24, 1), (32, 2), (32, 1), (32, 1), (64, 2), (64, 1), (64, 1), (64, 1),
                       (96, 1), (96, 1), (96, 1), (160, 2), (160, 1), (160, 1), (320, 1))


def mobilenet_v2_plan(width=1.0, expansion_factor=6.0):
  """Channel plan of mobilenet_v2_generator: (initial_conv filters, [(block_id, cin, expanded width or None,
  stride, cout, identity shortcut)], final_1x1_conv filters).  Every width must be a multiple of 8 (the NHWC
  kernels move 8 channels per 16-byte vector); ValueError names the first layer that is not."""
  def need8(c, layer):
    if c % 8:
      raise ValueError('MobileNetV2(width=%g, expansion_factor=%g): %s has %d channels, not a multiple of 8'
                       % (width, expansion_factor, layer, c))
    return c
  c0 = need8(_make_divisible(32 * width), 'initial_conv')
  blocks, prev = [], c0
  for b, (filters, stride) in enumerate(MOBILENET_V2_BLOCKS):
    expand = need8(int(expansion_factor * prev), 'expand_1x1_%d' % b) if b else None
    cout = need8(_make_divisible(int(width * filters), divisor=8 if b else 1), 'contraction_1x1_%d' % b)
    blocks.append((b, prev, expand, stride, cout, prev == cout and stride == 1))
    prev = cout
  last = need8(max(1280, _make_divisible(1280 * width, 8)), 'final_1x1_conv')
  return c0, blocks, last


class MobileNetV2(nn.Module):
  """MobileNet-v2 as mobilenetv2_model.py:156-398 builds it: plain ReLU (not ReLU6); the masked 1x1 convs
  `expand_1x1_{1..16}`, `contraction_1x1_{0..16}`, `final_1x1_conv` and (prune_last_layer) `final_dense`; dense
  `initial_conv` (3x3/2, 32 * width channels) and depthwise 3x3 convs, fixed padding where strided.  The
  contraction BN has no ReLU ("linear bottleneck"); where the block keeps its depth at stride 1 the input is
  added after it, with no activation after the add (fused into the BN kernel, csrc/bn.cu).  Block outputs whose
  next block has an identity shortcut are handed on as two handles (fork), as in ResNet50."""

  def __init__(self, num_classes=1000, width=1.0, expansion_factor=6.0, prune_last_layer=True, device='cuda',
               registry=None):
    super(MobileNetV2, self).__init__()
    c0, plan, last = mobilenet_v2_plan(width, expansion_factor)     # (raises before any parameter exists)
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg = self.registry

    def mk(ci, co, n):
      conv = SparseConv2d(ci, co, 1, strides=1, padding='FIXED', name='resnet_model/' + n, device=device,
                          registry=reg, kernel_initializer=_hwio_init)
      conv.collect_bn_stats = True        # the epilogue emits the BN statistics where that pays (conv heuristic)
      return conv
    self.initial_conv = DenseConv2d(3, c0, 3, stride=2, padding=1, bias=False, device=device)
    _trunc_variance_scaling_(self.initial_conv.weight, 27)
    self.initial_bn = _BNReLU(c0, device=device)
    blocks = []
    for b, cin, expand, stride, cout, shortcut in plan:
      blk = nn.Module()
      blk.shortcut = shortcut
      blk.expand = None
      mid = cin
      if expand is not None:
        blk.expand = mk(cin, expand, 'expand_1x1_%d' % b)
        blk.bn_expand = _BNReLU(expand, device=device)
        mid = expand
      blk.depthwise = DepthwiseConv2d(mid, stride=stride, device=device)
      # contrib separable_conv2d's default xavier (glorot uniform) init on the [3,3,C,1] depthwise kernel
      bound = math.sqrt(6.0 / (9 * mid + 9))
      with torch.no_grad():
        blk.depthwise.weight.uniform_(-bound, bound)
      blk.bn_dw = _BNReLU(mid, device=device)
      blk.contraction = mk(mid, cout, 'contraction_1x1_%d' % b)
      blk.bn_contraction = _BNReLU(cout, relu=False, device=device)
      blocks.append(blk)
    self.blocks = nn.ModuleList(blocks)
    self.final_conv = mk(plan[-1][4], last, 'final_1x1_conv')
    self.final_bn = _BNReLU(last, device=device)
    self.prune_last_layer = bool(prune_last_layer)
    if self.prune_last_layer:
      self.final_dense = SparseLinear(last, num_classes, name='resnet_model/final_dense', device=device, registry=reg,
                                      out_dtype=torch.float32, kernel_initializer=_hwio_init)
    else:             # tf.layers.dense: not masked, fp32
      self.final_dense = nn.Linear(last, num_classes, device=device)
      with torch.no_grad():
        _trunc_variance_scaling_(self.final_dense.weight, last)
        self.final_dense.bias.zero_()

  def forward(self, x):
    x = self.initial_bn(self.initial_conv(x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)))
    x_skip = x
    for i, blk in enumerate(self.blocks):
      h = x
      if blk.expand is not None:
        h = conv_bn(blk.expand, blk.bn_expand, h)
      h = blk.bn_dw(blk.depthwise(h))
      fork = FORK_BLOCK_OUTPUTS and i + 1 < len(self.blocks) and self.blocks[i + 1].shortcut
      y = conv_bn(blk.contraction, blk.bn_contraction, h, residual=x_skip if blk.shortcut else None, fork=fork)
      x, x_skip = y if fork else (y, y)
    x = conv_bn(self.final_conv, self.final_bn, x)
    x = x.mean(dim=(2, 3))
    if not self.prune_last_layer:
      x = x.float()
    return self.final_dense(x)


# convs per stage (vgg.py network_cfg); the stages have 64, 128, 256, 512 and 512 filters times `width`
VGG_CONFIGS = {'vgg_a': (1, 1, 2, 2, 2), 'vgg_16': (2, 2, 3, 3, 3), 'vgg_19': (2, 2, 4, 4, 4)}
VGG_STAGE_FILTERS = (64, 128, 256, 512, 512)


def vgg_plan(vgg_type, width=1.0):
  """[(scope, cin, cout, pool after)] of the masked 3x3 convs of vgg_net: scopes from tf.variable_scope(vgg_type) and
  contrib layers.repeat (scope 'convS', then 'convS_J' per repetition); a 2x2 max pool follows stages 1-4.  Every
  width must be a multiple of 8 (the NHWC kernels move 8 channels per 16-byte vector); ValueError names the first
  layer that is not."""
  if vgg_type not in VGG_CONFIGS:
    raise ValueError('vgg_type must be one of %s, got %r' % (sorted(VGG_CONFIGS), vgg_type))
  plan, cin = [], 3
  for s, (reps, filters) in enumerate(zip(VGG_CONFIGS[vgg_type], VGG_STAGE_FILTERS), 1):
    cout = int(filters * width)
    for j in range(1, reps + 1):
      scope = '%s/conv%d/conv%d_%d' % (vgg_type, s, s, j)
      if cout % 8:
        raise ValueError('VGG(%s, width=%g): %s has %d channels, not a multiple of 8' % (vgg_type, width, scope, cout))
      plan.append((scope, cin, cout, s < 5 and j == reps))
      cin = cout
  return plan


class VGG(nn.Module):
  """vgg_net (vgg.py) as the ImageNet driver builds it (--model_architecture vgg_a / vgg_16 / vgg_19, init_method
  'baseline'): masked 3x3 / stride-1 'SAME' convs without bias, each followed by a ReLU, the first one included;
  variance_scaling(2.0) (fan_in, truncated normal) init; a 2x2 / stride-2 'VALID' max pool after stages 1-4; then the
  global mean over H and W and `fc8`: with prune_last_layer a masked 1x1 conv to num_classes ([1,1,C,num_classes]
  mask, same init, fp32 logits), otherwise a dense 1x1 conv with xavier init and a zero bias that carries no l2
  regularizer (`l2_regularized = False`, see evaluate.regularized_kernels).

  The ReLUs cost no pass over the activations: every conv writes relu(conv(x)) from its epilogue
  (SparseConv2d.relu_out) and the ReLU's derivative is applied once per edge by the consumer -- the next conv's dgrad
  epilogue (gate_dgrad), the pool's backward (max_pool2x2_relu) or, for the last conv, relu_grad_gate."""

  def __init__(self, vgg_type, num_classes=1000, width=1.0, prune_last_layer=True, device='cuda', registry=None):
    super(VGG, self).__init__()
    plan = vgg_plan(vgg_type, width)            # (raises before any parameter exists)
    self.vgg_type = vgg_type
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    reg = self.registry
    he_init = lambda w: _trunc_variance_scaling_(w, int(np.prod(w.shape[:-1])), scale=2.0)
    convs, self.pool_after, prev_pool = [], [], True
    for scope, cin, cout, pool in plan:
      conv = SparseConv2d(cin, cout, 3, strides=1, padding='SAME', name=scope, device=device, registry=reg,
                          kernel_initializer=he_init)
      conv.relu_out = True
      conv.gate_dgrad = not prev_pool          # input straight from a ReLU conv (not the image, not a pool)
      convs.append(conv)
      self.pool_after.append(pool)
      prev_pool = pool
    self.convs = nn.ModuleList(convs)
    last = plan[-1][2]
    self.prune_last_layer = bool(prune_last_layer)
    if self.prune_last_layer:
      self.fc8 = SparseConv2d(last, num_classes, 1, strides=1, padding='SAME', name=vgg_type + '/fc8', device=device,
                              registry=reg, kernel_initializer=he_init, out_dtype=torch.float32)
    else:             # contrib layers.conv2d 1x1: not masked, fp32, xavier, zero bias, no weight regularizer
      self.fc8 = nn.Linear(last, num_classes, device=device)
      with torch.no_grad():
        nn.init.xavier_uniform_(self.fc8.weight)
        self.fc8.bias.zero_()
      self.fc8.l2_regularized = False

  def forward(self, x):
    x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    for conv, pool in zip(self.convs, self.pool_after):
      x = conv(x)
      if pool:
        x = max_pool2x2_relu(x)
    x = relu_grad_gate(x).mean(dim=(2, 3), keepdim=True)
    if self.prune_last_layer:
      return self.fc8(x).reshape(x.shape[0], -1)
    return self.fc8(x.reshape(x.shape[0], -1).float())


class MnistFC(nn.Module):
  """mnist_network_fc with model_pruning=True: three masked dense layers + ReLU."""

  def __init__(self, hidden=(300, 100), device='cuda', registry=None):
    super(MnistFC, self).__init__()
    self.registry = registry if registry is not None else pruning.MaskedLayerRegistry()
    dims = (784,) + tuple(hidden) + (10,)
    self.layers = nn.ModuleList([
        SparseLinear(dims[i], dims[i + 1], name='layer%d' % (i + 1), device=device,
                     registry=self.registry,
                     out_dtype=torch.float32 if i == len(dims) - 2 else torch.bfloat16)
        for i in range(len(dims) - 1)])

  def forward(self, x):
    for i, l in enumerate(self.layers):
      x = l(x)
      if i + 1 < len(self.layers):
        x = F.relu(x)
    return x


def init_masks(model, method, sparsity, custom_sparsity_map=None, seed=0, erk_power_scale=1.0):
  """Runs the reference's mask-init path (get_mask_init_fn) on a model's masks."""
  np.random.seed(seed)
  fn = sparse_utils.get_mask_init_fn(model.registry.get_masks(), method, sparsity,
                                     custom_sparsity_map or {}, erk_power_scale=erk_power_scale)
  return fn()


class TrainHarness(object):
  """One sparse training step, wired like imagenet_train_eval.py:355-430:
  Nesterov momentum 0.9, weight decay on the raw weights, label smoothing 0.1,
  SparseRigLOptimizer(drop 0.3 cosine, every 100 steps), optional data parallelism."""

  def __init__(self, model, lr=0.1, momentum=0.9, weight_decay=1e-4, label_smoothing=0.1,
               drop_fraction=0.3, drop_fraction_anneal='cosine', begin_step=0, end_step=25000,
               frequency=100, data_parallel=None, optimizer_cls=SparseRigLOptimizer, lr_schedule=None,
               fused_optimizer=None, inner_optimizer='momentum', pruning=None):
    """lr_schedule: optional callable(global_step) -> learning rate, evaluated on the host before every step
    (optim.make_imagenet_lr_fn is the reference's, imagenet_train_eval.py:317-354); `lr` is then only the
    initial value.  fused_optimizer: the inner optimizer is optim.FusedMomentumSGD (one launch, mask * dense_grad
    fused in, device-resident learning rate); default on for CUDA models (RIGL_FUSED_SGD=0 -> torch.optim.SGD).
    inner_optimizer: 'momentum' (the above) or 'adam' -- optim.FusedAdam(lr, weight_decay) with TF's beta1,
    beta2 and epsilon, the reference's `--use_adam` (imagenet_train_eval.py:355-358; there the learning rate is
    the constant base_lr * batch / 256).  'adam' exists only on the fused path: `momentum` is then unused.
    optimizer_cls=None: the inner optimizer alone, one step and one global-step increment per step (the
    reference's scratch / baseline / prune methods: `optimizer.minimize`).  pruning: a pruning.Pruning whose
    conditional_mask_update_op() runs after every step, eager or graphed; it counts this harness's global step."""
    import os
    if inner_optimizer not in ('momentum', 'adam'):
      raise ValueError("inner_optimizer must be 'momentum' or 'adam', got %r" % (inner_optimizer,))
    if inner_optimizer == 'adam' and fused_optimizer is not None and not fused_optimizer:
      raise ValueError("inner_optimizer='adam' needs the fused optimizer: there is no non-fused Adam with "
                       "tf.train.AdamOptimizer's arithmetic")
    self.model = model
    self.label_smoothing = label_smoothing
    self.lr_schedule = lr_schedule
    on_cuda = next(model.parameters()).is_cuda
    if fused_optimizer is None:
      fused_optimizer = inner_optimizer == 'adam' or (on_cuda and os.environ.get('RIGL_FUSED_SGD', '1') != '0')
    self.fused = bool(fused_optimizer)
    if inner_optimizer == 'adam':
      from .optim import FusedAdam
      self.inner = FusedAdam(model.parameters(), lr=lr, weight_decay=weight_decay)
    elif self.fused:
      from .optim import FusedMomentumSGD
      self.inner = FusedMomentumSGD(model.parameters(), lr=lr, momentum=momentum, nesterov=True,
                                    weight_decay=weight_decay)
    else:
      self.inner = torch.optim.SGD(model.parameters(), lr=lr, momentum=momentum, nesterov=True,
                                   weight_decay=weight_decay, foreach=True)
    self.opt = None if optimizer_cls is None else optimizer_cls(
        self.inner, begin_step, end_step, frequency, drop_fraction=drop_fraction,
        drop_fraction_anneal=drop_fraction_anneal, use_tpu=data_parallel is not None).bind(model.registry)
    self.pruning = pruning
    if pruning is not None and pruning.global_step is not None:
      self.global_step = pruning.global_step
    else:
      self.global_step = GlobalStep(0)
    if pruning is not None:
      pruning.global_step = self.global_step
    self.dp = data_parallel
    self._pack_ahead = on_cuda and os.environ.get('RIGL_PACK_AHEAD', '1') != '0'
    if self.dp is not None:
      self.dp.attach(model)
    if self.fused:
      # masked layers: the optimizer reads dense_grad (+ bitmap) directly; under data parallelism the buffers
      # hold the SUM over replicas, the weight update takes the mean (CrossShardOptimizer)
      inv = 1.0 / self.dp.world if self.dp is not None else 1.0
      self.inner.attach_masked_layers(model.registry.layers(), grad_scale=inv, other_grad_scale=inv)
      if self.dp is not None:
        self.dp.masked_grads_in_optimizer = True
        self.dp.other_scale_in_optimizer = True

  def _apply_lr_schedule(self):
    if self.lr_schedule is None:
      return
    lr = float(self.lr_schedule(self.global_step.value))
    if self.fused:
      self.inner.set_lr(lr)
    else:
      if getattr(self, 'graphed', False) and lr != self.inner.param_groups[0]['lr']:
        raise RuntimeError('torch.optim.SGD bakes the learning rate into a captured graph: use the fused optimizer '
                           'with an lr schedule')
      for g in self.inner.param_groups:
        g['lr'] = lr

  # ---- CUDA-graph mode: the forward+backward and the inner optimizer step are captured once and
  # replayed (inter-kernel launch gaps and all host work disappear); the data-parallel
  # all-reduce, the schedule logic and the (rare) mask update stay eager between the replays.
  def enable_cuda_graph(self, images, labels, warmup=3, overlap_wgrad=None):
    """Captures the step for fixed input shapes.  Returns False (and stays eager) if capture fails.
    overlap_wgrad: run the dense wgrad kernels on a forked stream inside the graph (layers.WGRAD_SIDE_STREAM);
    default from RIGL_WGRAD_OVERLAP (on unless '0')."""
    import os
    if overlap_wgrad is None:
      # default on (RIGL_WGRAD_OVERLAP=0 keeps the serial backward)
      overlap_wgrad = os.environ.get('RIGL_WGRAD_OVERLAP', '1') != '0' 
    self._overlap = bool(overlap_wgrad)
    self._sx, self._sy = images.clone(), labels.clone()
    return self._capture(warmup)

  def release_cuda_graph(self):
    """Drops the captured graphs, so the memory their pool holds can be freed; later steps run eagerly."""
    self.graphed = False
    for name in ('_g_fb', '_g_opt', '_sloss'):
      if hasattr(self, name):
        setattr(self, name, None)

  def _capture(self, warmup):
    try:
      side = torch.cuda.Stream()
      side.wait_stream(torch.cuda.current_stream())
      with torch.cuda.stream(side):
        for _ in range(warmup):
          self._forward_backward(self._sx, self._sy, set_to_none=False)
      torch.cuda.current_stream().wait_stream(side)
      torch.cuda.synchronize()
      from . import _cabi
      self._g_fb = torch.cuda.CUDAGraph()
      before = _cabi.launch_count()
      # (thread-local capture mode: the NCCL watchdog thread keeps issuing CUDA calls while we capture)
      with torch.cuda.graph(self._g_fb, capture_error_mode='thread_local'):
        self._sloss = self._forward_backward(self._sx, self._sy, set_to_none=False)
      self.graph_kernel_launches = _cabi.launch_count() - before     # rigl kernels inside one replay
      self.replayed_kernel_launches = 0
      self._g_opt = torch.cuda.CUDAGraph()
      if self.fused:
        self.inner.prepare()                   # slots / device lr / launch plan: allocated OUTSIDE the capture
      with torch.cuda.graph(self._g_opt, pool=self._g_fb.pool(), capture_error_mode='thread_local'):
        self.inner.step()
      self.graphed = True
    except Exception as e:      # stay on the eager path, but say why
      import warnings
      warnings.warn('CUDA-graph capture failed, running eagerly: %r' % (e,))
      torch.cuda.synchronize()
      self.graphed = False
    return self.graphed

  def _forward_backward(self, images, labels, set_to_none):
    from . import layers
    for mw in self.model.registry.get_masked_weights():
      mw.fresh = False
    self.inner.zero_grad(set_to_none=set_to_none)
    if self._pack_ahead:
      # ONE launch packs the operands (mask * W -> bf16, both layouts) of every layer
      layers.pack_all(self.model.registry.layers())
    logits = self.model(images)
    loss = F.cross_entropy(logits.float(), labels, label_smoothing=self.label_smoothing)
    layers.WGRAD_SIDE_STREAM = bool(getattr(self, '_overlap', False))
    layers.MASKED_GRAD_IN_OPTIMIZER = self.fused      # mask * dense_grad is formed inside the optimizer kernel
    try:
      loss.backward()
    finally:
      layers.WGRAD_SIDE_STREAM = False
      layers.MASKED_GRAD_IN_OPTIMIZER = False
      layers.join_side_streams()                # (no-op when nothing was forked)
    return loss

  def _graphed_step(self, images, labels):
    self._apply_lr_schedule()
    self._sx.copy_(images, non_blocking=True)
    self._sy.copy_(labels, non_blocking=True)
    self._g_fb.replay()
    self.replayed_kernel_launches += self.graph_kernel_launches
    if self.dp is not None:
      self.dp.reduce_gradients(self.model)
    gs = self.global_step
    def inner_step():
      self._g_opt.replay()
      gs.increment()
    if self.opt is None:
      inner_step()
    else:
      self.opt.collect_masked_grads()
      self.opt._global_step = gs
      # same decision as SparseRigLOptimizerBase.apply_gradients, with the inner step replayed
      self.opt.cond_mask_update_op(gs, inner_step)
    if self.pruning is not None:
      self.pruning.conditional_mask_update_op()
    return self._sloss

  def step(self, images, labels):
    """images: bf16 [N,3,H,W] channels_last; labels: int64 [N].  Returns the loss tensor."""
    if getattr(self, 'graphed', False):
      return self._graphed_step(images, labels)
    self._apply_lr_schedule()
    # without DP the grads are re-created by autograd (no zero-fill, no accumulate pass);
    # with DP they are views of the flat all-reduce buffer and must persist
    loss = self._forward_backward(images, labels, set_to_none=self.dp is None)
    if self.dp is not None:
      self.dp.reduce_gradients(self.model)
    if self.opt is None:
      self.inner.step()
      self.global_step.increment()
    else:
      self.opt.collect_masked_grads()
      self.opt.apply_gradients(None, global_step=self.global_step)
    if self.pruning is not None:
      self.pruning.conditional_mask_update_op()
    return loss


class _DepthwiseFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, weight, stride):
    from . import _cabi
    n, c, h, w = x.shape
    oh, ow = (h - 1) // stride + 1, (w - 1) // stride + 1
    y = torch.empty((n, c, oh, ow), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    _cabi.check(_cabi.lib().rigl_depthwise3x3_fprop(x.data_ptr(), weight.data_ptr(), n, h, w, c, stride, y.data_ptr(),
                                                    _cabi.stream_ptr()), 'rigl_depthwise3x3_fprop')
    ctx.save_for_backward(x, weight)
    ctx.stride = stride
    return y

  @staticmethod
  def backward(ctx, dy):
    from . import _cabi
    from .layers import _workspace
    x, weight = ctx.saved_tensors
    n, c, h, w = x.shape
    dy = dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dx = dw = None
    if ctx.needs_input_grad[0]:
      dx = torch.empty_like(x, memory_format=torch.channels_last)
      _cabi.check(_cabi.lib().rigl_depthwise3x3_dgrad(dy.data_ptr(), weight.data_ptr(), n, h, w, c, ctx.stride,
                                                      dx.data_ptr(), _cabi.stream_ptr()), 'rigl_depthwise3x3_dgrad')
    if ctx.needs_input_grad[1]:
      dw = torch.empty_like(weight)
      ws = _workspace(x.device, _cabi.lib().rigl_depthwise3x3_workspace_bytes(n, h, w, c, ctx.stride))
      _cabi.check(_cabi.lib().rigl_depthwise3x3_wgrad(x.data_ptr(), dy.data_ptr(), n, h, w, c, ctx.stride, dw.data_ptr(),
                                                      0.0, ws.data_ptr(), ws.numel(), _cabi.stream_ptr()),
                  'rigl_depthwise3x3_wgrad')
    return dx, dw, None


class DepthwiseConv2d(nn.Module):
  """depthwise_conv2d_fixed_padding(kernel_size=3) of the reference's MobileNet-v1 (mobilenetv1_model.py:120-153):
  dense (un-masked), fp32 master weights in the torch depthwise layout [C,1,3,3], bf16 compute on the streaming
  kernels of csrc/depthwise.cu when RIGL_NATIVE_DEPTHWISE=1; default: the stock cuDNN grouped conv (DESIGN.md
  3.4)."""

  def __init__(self, channels, stride=1, device='cuda'):
    super(DepthwiseConv2d, self).__init__()
    import math
    import os
    self.channels, self.stride = int(channels), int(stride)
    self.weight = nn.Parameter(torch.empty(channels, 1, 3, 3, device=device))
    nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
    self.native = os.environ.get('RIGL_NATIVE_DEPTHWISE', '0') == '1'

  def forward(self, x):
    if self.native and x.is_cuda and self.channels % 8 == 0:
      x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
      return _DepthwiseFn.apply(x, self.weight, self.stride)
    return F.conv2d(x, self.weight.to(torch.bfloat16), None, self.stride, 1, 1, self.channels)
