"""CPU restatement of the reference's VGG (rigl/imagenet_resnet/vgg.py): its masked-layer table and a float64
forward / backward of the reference graph on given weights.  Test infrastructure, not product code.

The table is written out from vgg.py's network_cfg, its filter counts int(64 * width) ... int(512 * width), and the
scopes of tf.variable_scope(vgg_type) + contrib layers.repeat (scope 'convS', repetition J named 'convS_J'),
independently of rigl_b200.workloads.
"""
import numpy as np
import torch
import torch.nn.functional as F

CFG = {'vgg_a': (1, 1, 2, 2, 2), 'vgg_16': (2, 2, 3, 3, 3), 'vgg_19': (2, 2, 4, 4, 4)}
FILTERS = (64, 128, 256, 512, 512)


def masked_layers(vgg_type, num_classes=1000, prune_last_layer=True, width=1.0, image_hw=224):
  """[(scope, HWIO shape, output hw)] in the reference's creation order (fc8 last, with prune_last_layer)."""
  out, cin, hw = [], 3, image_hw
  for s, reps in enumerate(CFG[vgg_type], 1):
    cout = int(FILTERS[s - 1] * width)
    for j in range(1, reps + 1):
      out.append(('%s/conv%d/conv%d_%d' % (vgg_type, s, s, j), (3, 3, cin, cout), hw))
      cin = cout
    if s < 5:
      hw //= 2
  if prune_last_layer:
    out.append(('%s/fc8' % vgg_type, (1, 1, cin, num_classes), 1))
  return out


def macs_per_image(vgg_type, num_classes=1000, image_hw=224):
  """Multiply-adds of one image at full density (every conv + fc8)."""
  return sum(int(np.prod(sh)) * hw * hw for _, sh, hw in masked_layers(vgg_type, num_classes, True, 1.0, image_hw))


def forward(images, weights, vgg_type, fc8_bias=None):
  """float64 logits of the reference graph.  images [N,3,H,W]; weights: list of HWIO tensors (the masked convs, then
  fc8 as [1,1,C,K] -- or, with fc8_bias, the dense fc8 as [K,C]).  Returns (logits, pre-activations of every conv)."""
  x = images.double()
  pre = []
  i = 0
  for s, reps in enumerate(CFG[vgg_type], 1):
    for _ in range(reps):
      w = weights[i].double().permute(3, 2, 0, 1)
      i += 1
      z = F.conv2d(x, w, padding=1)              # 3x3 / stride 1 'SAME'
      pre.append(z)
      x = torch.relu(z)
    if s < 5:
      x = F.max_pool2d(x, 2, 2)                  # 'VALID': floor
  x = x.mean(dim=(2, 3))
  w8 = weights[i].double()
  logits = x @ w8.reshape(-1, w8.shape[-1]) if fc8_bias is None else x @ w8.t() + fc8_bias.double()
  return logits, pre
