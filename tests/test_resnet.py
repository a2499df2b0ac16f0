"""ResNet-18 ... 200 on the CPU: the masked-layer table against known answers, the product's plan against it, the
sparsity distribution against fixtures produced by the reference itself, and the space-to-depth stem's channel
limits as the C ABI reports them."""
import json
import os

import numpy as np
import pytest

import resnet_oracle as ro
from rigl_b200 import _cabi, sparse_utils, workloads

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'resnet_sparsities_golden.json')


def test_layer_table_known_answers():
  want = {18: 22, 34: 38, 50: 54, 101: 105, 152: 156, 200: 204}
  for depth, n in want.items():
    assert len(ro.masked_layers(depth)) == n
    assert len(ro.masked_layers(depth, prune_first_layer=False, prune_last_layer=False)) == n - 2
  # ResNet-50's table is the one the rest of the suite already checks
  from oracle import rigl_oracle as orc
  assert ro.masked_layers(50) == [(s, tuple(sh)) for s, sh, _, _ in orc.resnet50_masked_layers()]
  # ResNet-18: the well-known 11,689,512 parameters less 9,600 BN parameters and the 1,000 classifier biases, plus
  # the 64 x 64 projection the reference has on block group 1
  assert sum(int(np.prod(sh)) for _, sh in ro.masked_layers(18)) == 11689512 - 9600 - 1000 + 64 * 64
  names = [s for s, _ in ro.masked_layers(18)]
  assert names[:4] == ['resnet_model/initial_conv',
                       'resnet_model/residual_projection_block_group_projection_block_group1',
                       'resnet_model/residual_1_block_group_projection_block_group1',
                       'resnet_model/residual_2_block_group_projection_block_group1']
  assert names[-2:] == ['resnet_model/residual_2_block_group4_1_1', 'resnet_model/final_dense']
  assert dict(ro.masked_layers(18, width=2.0))['resnet_model/final_dense'] == (1024, 1000)
  assert dict(ro.masked_layers(101, width=0.5))['resnet_model/final_dense'] == (1024, 1000)


def _plan_table(depth, width, first=True, last=True, num_classes=1000):
  """The product's plan written out as the oracle's table."""
  kind, c0, plan, fc_in = workloads.resnet_plan(depth, width)
  out = [('resnet_model/initial_conv', (7, 7, 3, c0))] if first else []
  for name, cin, f, stride, proj in plan:
    if kind == 'bottleneck':
      p = 'resnet_model/bottleneck_'
      if proj:
        out.append((p + 'projection_' + name, (1, 1, cin, 4 * f)))
      out += [(p + '1_' + name, (1, 1, cin, f)), (p + '2_' + name, (3, 3, f, f)), (p + '3_' + name, (1, 1, f, 4 * f))]
    else:
      p = 'resnet_model/residual_'
      if proj:
        out.append((p + 'projection_' + name, (1, 1, cin, f)))
      out += [(p + '1_' + name, (3, 3, cin, f)), (p + '2_' + name, (3, 3, f, f))]
  if last:
    out.append(('resnet_model/final_dense', (fc_in, num_classes)))
  return kind, out


@pytest.mark.parametrize('depth', sorted(ro.LAYERS))
@pytest.mark.parametrize('width', [0.25, 0.5, 1.0, 2.0])
def test_product_plan_matches_the_table(depth, width):
  for first in (True, False):
    for last in (True, False):
      kind, table = _plan_table(depth, width, first, last)
      assert table == ro.masked_layers(depth, width, 1000, first, last)
      assert kind == ('bottleneck' if depth >= 50 else 'residual')
  # strides: the projection and the first conv carrying the group's stride, group 1 at stride 1
  strides = [(name, s) for name, _, _, s, proj in workloads.resnet_plan(depth, width)[2] if proj]
  assert strides == [('block_group_projection_block_group%d' % g, 1 if g == 1 else 2) for g in (1, 2, 3, 4)]
  assert [b[:4] for b in workloads.resnet_plan(depth, width)[2]] == [b[:4] for b in ro.blocks(depth, width)]


def test_bad_depth_and_width_raise_before_any_parameter():
  with pytest.raises(ValueError, match='resnet_depth'):
    workloads.resnet_plan(42)
  with pytest.raises(ValueError, match='resnet_depth'):
    workloads.ResNet(42, device='cuda')
  with pytest.raises(ValueError, match=r'resnet_model/initial_conv has 19 channels'):
    workloads.ResNet(18, width=0.3, device='cuda')
  with pytest.raises(ValueError, match='initial_conv has 20 channels'):
    workloads.resnet_plan(50, 0.3125)
  # a stem of 8 channels and a second group of 17: named by the first layer that has them
  with pytest.raises(ValueError, match=r'residual_projection_block_group_projection_block_group2 has 17 channels'):
    workloads.resnet_plan(18, 17 / 128.)
  with pytest.raises(ValueError, match=r'bottleneck_projection_block_group_projection_block_group2 has 68 channels'):
    workloads.resnet_plan(50, 17 / 128.)


def test_sparsities_bit_exact_vs_reference():
  with open(GOLDEN) as f:
    golden = json.load(f)
  seen = set()
  for case in golden['cases']:
    key = (case['depth'], case['width'], case['prune_first_layer'], case['prune_last_layer'], case['method'],
           case['default_sparsity'])
    seen.add(key)
    _, table = _plan_table(case['depth'], case['width'], case['prune_first_layer'], case['prune_last_layer'])
    assert len(table) == case['n_layers']
    masks = [_Mask(n, sh) for n, sh in table]
    sp = sparse_utils.get_sparsities(masks, case['method'], case['default_sparsity'], {})
    assert set(sp) == {m.name for m in masks}
    for m, hx, nnz in zip(masks, case['sparsities_hex'], case['nnz']):
      assert float(sp[m.name]).hex() == hx, (key, m.name)
      size = int(np.prod(m.shape))
      assert size - sparse_utils.get_n_zeros(size, sp[m.name]) == nnz, (key, m.name)
  # depths 18 / 34 / 101 / 152 / 200; widths 0.5 / 1 / 2; both prune flags on and off; ERK 0.8 / 0.9, random 0.9
  assert len(seen) == 90
  assert {k[0] for k in seen} == {18, 34, 101, 152, 200} and {k[1] for k in seen} == {0.5, 1.0, 2.0}
  assert {k[2:4] for k in seen} == {(True, True), (True, False), (False, True), (False, False)}
  assert {k[4:] for k in seen} == {('erdos_renyi_kernel', 0.8), ('erdos_renyi_kernel', 0.9), ('random', 0.9)}


class _Mask(object):

  def __init__(self, name, shape):
    self.name, self.shape, self.dtype = name + '/mask:0', tuple(shape), np.float32


def _stem_desc(cout, batch=256, hw=224):
  d = _cabi.ConvDesc()
  d.batch, d.in_h, d.in_w, d.cin, d.cout = batch, hw, hw, 3, cout
  d.out_h = d.out_w = hw // 2
  d.ksize, d.stride, d.pad, d.x_pitch = 7, 2, 3, 0
  return d


def test_stem_s2d_channel_limits_and_workspace():
  """cout 8 ... 256 in steps of 8 take the space-to-depth stem, one 64-channel group per grid row; 264 and
  non-multiples of 8 do not.  The wgrad workspace holds one [4][128][64] fp32 partial per CTA and group."""
  lib = _cabi.lib()
  one = lib.rigl_stem_s2d_workspace_bytes(_stem_desc(64))
  assert one > 256 and (one - 256) % (4 * 128 * 64 * 4) == 0
  grid = (one - 256) // (4 * 128 * 64 * 4)
  for cout in range(8, 257, 8):
    d = _stem_desc(cout)
    assert lib.rigl_stem_s2d_supported(d) == 1, cout
    groups = -(-cout // 64)
    assert lib.rigl_stem_s2d_workspace_bytes(d) == grid * groups * 4 * 128 * 64 * 4 + 256, cout
    assert lib.rigl_stem_s2d_packed_bytes(d) == 16 * cout * 32
  for cout in (264, 320, 4, 12, 100, 250):
    d = _stem_desc(cout)
    assert lib.rigl_stem_s2d_supported(d) == 0, cout
    assert lib.rigl_stem_s2d_workspace_bytes(d) == 0, cout
    assert lib.rigl_stem_s2d_folded_bytes(d) == 0, cout
