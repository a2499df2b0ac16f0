"""The layer shapes ResNet-18 / 34 and the width-2 stem add to ResNet-50's, against float64 at batch 256, 224 x 224,
ERK 0.8, with the bounds and controls of test_resnet50_b256_gpu (its module docstring states them).

Covered: the 3x3 stride-2 convs that open block groups 2-4 of the basic block (64 -> 128, 128 -> 256, 256 -> 512),
their 1x1 stride-2 projections, the 1x1 stride-1 64 -> 64 projection of block group 1, final_dense 512 -> 1000, and
ResNet-50's stem at width 2 (3 -> 128: two 64-channel groups of the space-to-depth kernels).  The grouped stem keeps a
64-channel launch's strip-to-CTA assignment in every group, so its wgrad bound and its CTA-0 control are the ones of
the 64-channel stem.  ResNet-34 has no layer shape that ResNet-18 does not.
"""
import pytest
import torch

import test_resnet50_b256_gpu as rb
from test_bench_c4_c5_gpu import _shape_id

gpu = pytest.mark.gpu
_NEW = []


def _entries(model, hw):
  """[entry] (test_resnet50_b256_gpu._table's form) of the model's masked layers, in first-use order."""
  from rigl_b200.layers import SparseConv2d, SparseLinear
  out = []

  def hook(mod, args):
    if isinstance(mod, SparseLinear):
      key, h, w, kind = ('linear', mod.in_channels, mod.out_channels, 1, 1, 1), 1, 1, 'linear'
    else:
      h, w, kind = int(args[0].shape[2]), int(args[0].shape[3]), 'conv'
      key = ('conv', mod.in_channels, mod.out_channels, mod.ksize, mod.stride, h)
    out.append(dict(layer=mod, kind=kind, h=h, w=w, key=key, model=model))

  handles = [m.register_forward_pre_hook(hook) for m in model.modules() if isinstance(m, (SparseConv2d, SparseLinear))]
  model.eval()
  try:
    with torch.no_grad():
      model(torch.zeros((1, 3, hw, hw), device=rb.DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last))
  finally:
    for h in handles:
      h.remove()
    model.train()
  return out


def _new_table():
  """ResNet-18's layers whose key ResNet-50 does not have, plus its block-group-1 projection (a 1x1 64 -> 64 conv
  like ResNet-50's bottleneck_1 of that group, but a projection), then ResNet-50's stem at width 2."""
  if _NEW:
    return _NEW
  from rigl_b200 import workloads
  old = {key for _, key in rb._CASES}
  torch.manual_seed(0)
  r18 = workloads.ResNet(18, device=rb.DEV)
  workloads.init_masks(r18, 'erdos_renyi_kernel', rb.SPARSITY, seed=0)
  seen = set()
  for e in _entries(r18, rb.HW):
    proj1 = e['layer'].scope.endswith('residual_projection_block_group_projection_block_group1')
    if (e['key'] not in old or proj1) and e['key'] not in seen:
      seen.add(e['key'])
      _NEW.append(e)
  torch.manual_seed(0)
  wide = workloads.ResNet(50, width=2.0, device=rb.DEV)
  workloads.init_masks(wide, 'erdos_renyi_kernel', rb.SPARSITY, seed=0)
  _NEW.append(_entries(wide, rb.HW)[0])
  torch.cuda.synchronize()
  return _NEW


_KEYS = [('conv', 64, 64, 1, 1, 56), ('conv', 64, 128, 1, 2, 56), ('conv', 64, 128, 3, 2, 56),
         ('conv', 128, 256, 1, 2, 28), ('conv', 128, 256, 3, 2, 28), ('conv', 256, 512, 1, 2, 14),
         ('conv', 256, 512, 3, 2, 14), ('linear', 512, 1000, 1, 1, 1), ('conv', 3, 128, 7, 2, 224)]
_IDS = ['proj1_64_64', '1x1s2_64_128', '3x3s2_64_128', '1x1s2_128_256', '3x3s2_128_256', '1x1s2_256_512',
        '3x3s2_256_512', 'dense_512_1000', 'stem_w2_128']


def test_new_shapes_from_the_oracle():
  """The shapes the basic block adds, from the reference's tables (no GPU), in first-use order (a block computes
  its shortcut first)."""
  import resnet_oracle as ro
  old = {key for _, key in rb._CASES}
  new = []
  for depth in (18, 34):
    for name, cin, f, stride, proj in ro.blocks(depth):
      g = int(name[-1]) if proj else int(name[len('block_group')])
      in_hw = 56 >> max(g - 2, 0) if proj else 56 >> (g - 1)
      for scope, sh, s in ro.block_convs(depth, name, cin, f, stride, proj):
        key = ('conv', sh[2], sh[3], sh[0], s, in_hw if '_2_' not in scope else 56 >> (g - 1))
        if (key not in old or scope.endswith('projection_block_group_projection_block_group1')) and key not in new:
          new.append(key)
  fc = ro.masked_layers(18)[-1][1]
  assert new + [('linear',) + fc + (1, 1, 1)] == _KEYS[:-1]
  assert _KEYS[-1][:3] == ('conv',) + ro.masked_layers(50, width=2.0)[0][1][2:]
  assert _KEYS[-2] not in old and _KEYS[-1] not in old


@gpu
def test_new_table_matches_the_oracle():
  table = _new_table()
  assert [e['key'] for e in table] == _KEYS
  assert table[-1]['layer'].s2d_mode and table[0]['layer'].scope.endswith('residual_projection_block_group_'
                                                                           'projection_block_group1')
  for e in table:
    p = rb._plan(e)
    print('plan %-52s %s wgrad: %d x %d positions' % (_shape_id(e, rb.BATCH), p['kernel'], p['splits'], p['pps']))


@gpu
@pytest.mark.parametrize('i', range(len(_IDS)), ids=_IDS)
def test_new_layer_b256_against_float64(i):
  table = _new_table()
  saved = list(rb._TABLE)
  rb._TABLE[:] = table
  try:
    rb._case(i)
  finally:
    rb._TABLE[:] = saved
