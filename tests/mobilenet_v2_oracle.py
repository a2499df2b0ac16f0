"""CPU restatement of the reference's MobileNet-v2 (rigl/imagenet_resnet/mobilenetv2_model.py) at width 1.0 and
expansion factor 6: its masked-layer table and a train step with the same bf16 rounding points as the other CPU
nets of oracle/cpu_train_step.py.  Test infrastructure, not product code.

The table is written out from the reference's block list (mobilenetv2_model.py:318-340) and its channel rules
(block 0 has no expand conv and its contraction is not rounded to a multiple of 8; expand width = 6 x input depth;
identity shortcut when the depth is kept at stride 1), independently of rigl_b200.workloads.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import cpu_train_step as cpu
from oracle import rigl_oracle as orc

# (filters, stride) of inverted_res_block 0..16 at width 1.0
BLOCKS = ((16, 1), (24, 2), (24, 1), (32, 2), (32, 1), (32, 1), (64, 2), (64, 1), (64, 1), (64, 1),
          (96, 1), (96, 1), (96, 1), (160, 2), (160, 1), (160, 1), (320, 1))
INITIAL, FINAL = 32, 1280


def block_table(image_hw=224):
  """[(block_id, cin, expanded width or None, stride, cout, identity shortcut, input hw, output hw)]."""
  rows, cin, hw = [], INITIAL, (image_hw + 1) // 2
  for b, (cout, stride) in enumerate(BLOCKS):
    out_hw = (hw - 1) // stride + 1
    rows.append((b, cin, 6 * cin if b else None, stride, cout, cin == cout and stride == 1, hw, out_hw))
    cin, hw = cout, out_hw
  return rows


def masked_layers(num_classes=1000, prune_last_layer=True, image_hw=224):
  """[(scope, HWIO / [in,out] shape, stride, output hw)] in the reference's creation order (35 with final_dense)."""
  out = []
  for b, cin, exp, stride, cout, _, hw, out_hw in block_table(image_hw):
    if exp is not None:
      out.append(('resnet_model/expand_1x1_%d' % b, (1, 1, cin, exp), 1, hw))
    out.append(('resnet_model/contraction_1x1_%d' % b, (1, 1, exp or cin, cout), 1, out_hw))
  last_hw = block_table(image_hw)[-1][-1]
  out.append(('resnet_model/final_1x1_conv', (1, 1, BLOCKS[-1][0], FINAL), 1, last_hw))
  if prune_last_layer:
    out.append(('resnet_model/final_dense', (FINAL, num_classes), 1, 1))
  return out


def depthwise_layers(image_hw=224):
  """[(scope, channels, stride, input hw, output hw)] of the 17 dense depthwise 3x3 convs."""
  return [('resnet_model/depthwise_nxn_%d' % b, exp or cin, stride, hw, out_hw)
          for b, cin, exp, stride, _, _, hw, out_hw in block_table(image_hw)]


def macs_per_image(image_hw=224, num_classes=1000):
  """(masked MACs, all MACs) of one image at full density: every conv + the classifier."""
  masked = sum(int(np.prod(sh)) * hw * hw for _, sh, _, hw in masked_layers(num_classes, True, image_hw))
  hw0 = (image_hw + 1) // 2
  dense = 3 * 3 * 3 * INITIAL * hw0 * hw0 + sum(9 * c * ohw * ohw for _, c, _, _, ohw in depthwise_layers(image_hw))
  return masked, masked + dense


class CpuMobileNetV2(cpu._CpuNet):
  """The reference's MobileNet-v2 train step on the CPU (fp32; `bf16_act` rounds every stored activation and its
  gradient where the CUDA path stores bf16).  Masks: uniform `sparsity` (ERK is what the driver uses, but the
  step arithmetic does not depend on how the masks were drawn)."""

  def __init__(self, sparsity=0.8, seed=0, num_classes=1000, bf16_weights=False):
    rng = np.random.RandomState(seed)
    layers = [(n, sh) for n, sh, _, _ in masked_layers(num_classes)]
    self._init_masked(layers, {n + '/mask:0': sparsity for n, _ in layers}, rng, bf16_weights)
    rnd = (lambda a: cpu._bf16_round(a)) if bf16_weights else (lambda a: torch.from_numpy(a))
    self.p['initial_conv'] = rnd((rng.standard_normal((3, 3, 3, INITIAL)) * np.sqrt(1.0 / 27)).astype(np.float32)) \
        .requires_grad_(True)
    for b, c, _, _, _ in depthwise_layers():
      self.p['depthwise_%d' % int(b.rsplit('_', 1)[1])] = rnd(
          (rng.standard_normal((c, 1, 3, 3)) * np.sqrt(2.0 / 9)).astype(np.float32)).requires_grad_(True)
    self.p['final_bias'] = torch.zeros(num_classes, requires_grad=True)

  def forward_backward(self, images, labels, label_smoothing=0.1):
    masked = self._masked()
    p = 'resnet_model/'
    x = self._bn(self.q(cpu._conv_tf(images, self.p['initial_conv'], 2, 'FIXED')), 'bn0')
    for b, _, exp, stride, _, shortcut, _, _ in block_table(images.shape[2]):
      h = x
      if exp is not None:
        h = self._bn(self.mconv(h, p + 'expand_1x1_%d' % b, masked, 1, 'FIXED'), 'e%d' % b)
      h = self.q(F.conv2d(h, self.p['depthwise_%d' % b], stride=stride, padding=1, groups=h.shape[1]))
      h = self._bn(h, 'dw%d' % b)
      h = self.mconv(h, p + 'contraction_1x1_%d' % b, masked, 1, 'FIXED')
      if shortcut:        # BN (no ReLU) + shortcut: ONE fused kernel, one rounding
        x = self.q(self._bn(h, 'c%d' % b, relu=False, store=False) + x)
      else:
        x = self._bn(h, 'c%d' % b, relu=False)
    x = self._bn(self.mconv(x, p + 'final_1x1_conv', masked, 1, 'FIXED'), 'final')
    logits = self.mlinear(self.q(x.mean(dim=(2, 3))), p + 'final_dense', masked, self.p['final_bias'])
    return self._finish(logits, labels, masked, label_smoothing)


def erk_sparsities(sparsity, prune_last_layer=True):
  masks = [orc.FakeMask(n + '/mask:0', sh) for n, sh, _, _ in masked_layers(1000, prune_last_layer)]
  return orc.get_sparsities(masks, 'erdos_renyi_kernel', sparsity, {})
