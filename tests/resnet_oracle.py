"""CPU restatement of the reference's ResNet family (rigl/imagenet_resnet/resnet_model.py, resnet_v1_): its
masked-layer table for every depth, width and prune flag, and a float64 train-mode forward / backward of the
reference graph on given weights, masks and batch-norm parameters.  Test infrastructure, not product code.

The table is written out from resnet_v1_'s depth table (basic block for 18 / 34, bottleneck for 50 and deeper), the
filter counts int(64 * width) ... int(512 * width) and the scopes of block_group / residual_block_ /
bottleneck_block_, independently of rigl_b200.workloads.
"""
import torch
import torch.nn.functional as F

LAYERS = {18: (2, 2, 2, 2), 34: (3, 4, 6, 3), 50: (3, 4, 6, 3), 101: (3, 4, 23, 3), 152: (3, 8, 36, 3),
          200: (3, 24, 36, 3)}
EPS = 1e-5


def bottleneck(depth):
  return depth >= 50


def blocks(depth, width=1.0):
  """[(block name, cin, filters, stride, projection)] in creation order."""
  out, cin = [], int(64 * width)
  mult = 4 if bottleneck(depth) else 1
  for g, (base, stride) in enumerate(((64, 1), (128, 2), (256, 2), (512, 2)), 1):
    f = int(base * width)
    for b in range(LAYERS[depth][g - 1]):
      name = 'block_group_projection_block_group%d' % g if b == 0 else 'block_group%d_%d_1' % (g, b)
      out.append((name, cin, f, stride if b == 0 else 1, b == 0))
      cin = mult * f
  return out


def block_convs(depth, name, cin, f, stride, proj):
  """[(scope, HWIO shape, stride)] of one block, in creation order (projection first)."""
  if bottleneck(depth):
    p = 'resnet_model/bottleneck_'
    convs = [(p + 'projection_' + name, (1, 1, cin, 4 * f), stride)] if proj else []
    return convs + [(p + '1_' + name, (1, 1, cin, f), 1), (p + '2_' + name, (3, 3, f, f), stride),
                    (p + '3_' + name, (1, 1, f, 4 * f), 1)]
  p = 'resnet_model/residual_'
  convs = [(p + 'projection_' + name, (1, 1, cin, f), stride)] if proj else []
  return convs + [(p + '1_' + name, (3, 3, cin, f), stride), (p + '2_' + name, (3, 3, f, f), 1)]


def fc_inputs(depth, width=1.0):
  return (4 if bottleneck(depth) else 1) * int(512 * width)


def masked_layers(depth, width=1.0, num_classes=1000, prune_first_layer=True, prune_last_layer=True):
  """[(scope, HWIO or [in, out] shape)] of the masked layers in the reference's creation order."""
  out = []
  if prune_first_layer:
    out.append(('resnet_model/initial_conv', (7, 7, 3, int(64 * width))))
  for name, cin, f, stride, proj in blocks(depth, width):
    out += [(s, sh) for s, sh, _ in block_convs(depth, name, cin, f, stride, proj)]
  if prune_last_layer:
    out.append(('resnet_model/final_dense', (fc_inputs(depth, width), num_classes)))
  return out


def _bn(z, gamma, beta):
  mean = z.mean(dim=(0, 2, 3), keepdim=True)
  var = ((z - mean) ** 2).mean(dim=(0, 2, 3), keepdim=True)
  return (z - mean) / torch.sqrt(var + EPS) * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)


def _max_pool_same(x):
  """tf.layers.max_pooling2d(3, 2, 'SAME'): out = ceil(in / 2), the extra padding after the image."""
  h, w = x.shape[2], x.shape[3]
  ph = max((-(-h // 2) - 1) * 2 + 3 - h, 0)
  pw = max((-(-w // 2) - 1) * 2 + 3 - w, 0)
  x = F.pad(x, (pw // 2, pw - pw // 2, ph // 2, ph - ph // 2), value=float('-inf'))
  return F.max_pool2d(x, 3, 2)


def forward(images, weights, bn, depth, width=1.0, fc_bias=None, record=None):
  """float64 train-mode logits of resnet_v1_(depth, width).  weights: scope -> HWIO conv kernel ([in, out] for
  final_dense) -- the effective (masked) values; bn: conv scope -> (gamma, beta) of the batch norm after that conv;
  fc_bias: final_dense's bias or None.  record: if a dict, scope -> (conv input, conv output) of every conv, both
  retaining their gradients after a backward."""
  def conv(x, scope, stride):
    w = weights[scope].double()
    k = w.shape[0]
    z = F.conv2d(x, w.permute(3, 2, 0, 1), stride=stride, padding=(k - 1) // 2)     # conv2d_fixed_padding
    if record is not None:
      if x.requires_grad:
        x.retain_grad()
      z.retain_grad()
      record[scope] = (x, z)
    g, b = bn[scope]
    return _bn(z, g.double(), b.double())

  x = images.double()
  x = torch.relu(conv(x, 'resnet_model/initial_conv', 2))
  x = _max_pool_same(x)
  for name, cin, f, stride, proj in blocks(depth, width):
    convs = block_convs(depth, name, cin, f, stride, proj)
    shortcut = x
    if proj:
      shortcut = conv(x, convs[0][0], stride)
      convs = convs[1:]
    h = x
    for i, (scope, _, s) in enumerate(convs):
      h = conv(h, scope, s)
      if i + 1 < len(convs):
        h = torch.relu(h)
    x = torch.relu(h + shortcut)
  feat = x.mean(dim=(2, 3))
  logits = feat @ weights['resnet_model/final_dense'].double()
  return logits if fc_bias is None else logits + fc_bias.double()
