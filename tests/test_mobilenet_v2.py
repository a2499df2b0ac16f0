"""MobileNet-v2 on the CPU: the layer table against the reference's known answers, the product's sparsity
distribution against fixtures produced by the reference itself, and argument checks that run before any CUDA work."""
import json
import os

import numpy as np
import pytest

import mobilenet_v2_oracle as mo
from rigl_b200 import _cabi, sparse_utils, workloads

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'mobilenet_v2_sparsities_golden.json')


def test_layer_table_matches_the_reference_model():
  layers = mo.masked_layers()
  names = [n for n, _, _, _ in layers]
  assert names == (['resnet_model/contraction_1x1_0'] +
                   [p % b for b in range(1, 17) for p in ('resnet_model/expand_1x1_%d', 'resnet_model/contraction_1x1_%d')] +
                   ['resnet_model/final_1x1_conv', 'resnet_model/final_dense'])
  shapes = dict((n, sh) for n, sh, _, _ in layers)
  assert shapes['resnet_model/contraction_1x1_0'] == (1, 1, 32, 16)
  assert shapes['resnet_model/expand_1x1_1'] == (1, 1, 16, 96)
  assert shapes['resnet_model/contraction_1x1_1'] == (1, 1, 96, 24)
  assert shapes['resnet_model/expand_1x1_16'] == (1, 1, 160, 960)
  assert shapes['resnet_model/contraction_1x1_16'] == (1, 1, 960, 320)
  assert shapes['resnet_model/final_1x1_conv'] == (1, 1, 320, 1280)
  assert shapes['resnet_model/final_dense'] == (1280, 1000)
  assert all(s == 1 for _, _, s, _ in layers)
  out_hw = dict((n, hw) for n, _, _, hw in layers)
  assert out_hw['resnet_model/contraction_1x1_0'] == 112 and out_hw['resnet_model/expand_1x1_1'] == 112
  assert out_hw['resnet_model/contraction_1x1_1'] == 56 and out_hw['resnet_model/contraction_1x1_3'] == 28
  assert out_hw['resnet_model/contraction_1x1_6'] == 14 and out_hw['resnet_model/contraction_1x1_13'] == 7
  assert out_hw['resnet_model/final_1x1_conv'] == 7
  dw = mo.depthwise_layers()
  assert [s for _, _, s, _, _ in dw] == [s for _, s in mo.BLOCKS]
  assert [c for _, c, _, _, _ in dw] == [32, 96, 144, 144, 192, 192, 192, 384, 384, 384, 384, 576, 576, 576, 960,
                                         960, 960]
  # known answers at width 1.0, expansion 6
  assert len(layers) == 35
  assert sum(int(np.prod(sh)) for _, sh, _, _ in layers) == 3404672
  assert mo.macs_per_image() == (269219840, 300774272)
  assert [b for b, _, _, _, _, sc, _, _ in mo.block_table() if sc] == [2, 4, 5, 7, 8, 9, 11, 12, 14, 15]
  assert all(d % 8 == 0 for _, sh, _, _ in layers for d in sh[2:])


def test_product_channel_plan_matches_the_table():
  c0, plan, last = workloads.mobilenet_v2_plan()
  assert (c0, last) == (mo.INITIAL, mo.FINAL)
  assert [p for p in plan] == [r[:6] for r in mo.block_table()]


class _Mask(object):

  def __init__(self, name, shape):
    self.name, self.shape, self.dtype = name + '/mask:0', tuple(shape), np.float32
    self.value = None

  def assign(self, v):
    self.value = np.asarray(v)


def test_sparsities_bit_exact_vs_reference():
  with open(GOLDEN) as f:
    golden = json.load(f)
  tags = set()
  for case in golden['cases']:
    tags.add(case['tag'])
    assert [tuple(sh) for _, sh in case['layers']] == \
        [sh for _, sh, _, _ in mo.masked_layers(1000, len(case['layers']) == 35)]
    masks = [_Mask(n, sh) for n, sh in case['layers']]
    sp = sparse_utils.get_sparsities(masks, case['method'], case['default_sparsity'], case['custom'],
                                     erk_power_scale=case['erk_power_scale'])
    assert set(sp) == set(case['sparsities_hex'])
    for name, hx in case['sparsities_hex'].items():
      assert float(sp[name]).hex() == hx, (case['tag'], name)
    for m in masks:
      size = int(np.prod(m.shape))
      assert size - sparse_utils.get_n_zeros(size, sp[m.name]) == case['nnz'][m.name], (case['tag'], m.name)
  assert len(tags) == 6


@pytest.mark.parametrize('width,expansion,layer', [(0.75, 6.0, 'contraction_1x1_0'), (1.4, 6.0, 'contraction_1x1_0'),
                                                   (1.0, 5.5, 'expand_1x1_2')])
def test_bad_width_raises_before_any_cuda_work(width, expansion, layer):
  with pytest.raises(ValueError, match=layer):
    workloads.MobileNetV2(width=width, expansion_factor=expansion, device='cuda')


def test_half_width_plan_is_all_multiples_of_8():
  c0, plan, last = workloads.mobilenet_v2_plan(0.5)
  assert (c0, last) == (16, 1280)
  assert [cout for _, _, _, _, cout, _ in plan] == [8, 16, 16, 16, 16, 16, 32, 32, 32, 32, 48, 48, 48, 80, 80, 80, 160]


def test_bn_backward_residual_relu_needs_bitmap_before_any_cuda_call():
  """The residual form with a ReLU reads the forward's sign bitmap: a NULL bitmap is refused up front (never a
  launch that dereferences it).  Every pointer here is a non-NULL dummy that must not be touched."""
  lib = _cabi.lib()
  p = 256
  rc = lib.rigl_bn_backward(p, None, p, p, p, p, p, 64, 64, 1, p, p, p, p, p, 1 << 20, None, None)
  assert rc == -1
  assert b'bitmap' in lib.rigl_last_error()
  # the other argument checks still come first
  assert lib.rigl_bn_backward(p, p, p, p, p, p, p, 64, 64, 0, p, None, p, p, p, 1 << 20, None, None) == -1
  assert b'residual form' in lib.rigl_last_error()
  assert lib.rigl_bn_backward(p, None, p, p, p, p, p, 64, 12, 0, p, p, p, p, p, 1 << 20, None, None) == -1
  assert b'multiple of 8' in lib.rigl_last_error()


def test_library_version_matches_the_bindings():
  assert _cabi.lib().rigl_version() >= _cabi.ABI_VERSION == 202
