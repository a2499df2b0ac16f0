"""VGG on the CPU: the layer table against known answers, the product's plan against it, the sparsity distribution
against fixtures produced by the reference itself, and argument checks of the ReLU entry points that run before any
CUDA work."""
import json
import os

import numpy as np
import pytest
import torch
from torch import nn

import vgg_oracle as vo
from rigl_b200 import _cabi, sparse_utils, workloads
from rigl_b200.evaluate import regularized_kernels

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'vgg_sparsities_golden.json')


def test_layer_table_known_answers():
  # (masked tensors with fc8, weights, MACs per 224x224 image) at width 1.0, 1000 classes
  want = {'vgg_a': (9, 9729728, 7485968384), 'vgg_16': (14, 15222464, 15347142656),
          'vgg_19': (17, 20530880, 19508940800)}
  for t, (n, weights, macs) in want.items():
    layers = vo.masked_layers(t)
    assert (len(layers), sum(int(np.prod(sh)) for _, sh, _ in layers), vo.macs_per_image(t)) == want[t]
    assert len(vo.masked_layers(t, prune_last_layer=False)) == n - 1
  # VGG-16's conv kernels: the well-known 14,714,688 parameters less the 4,224 biases the reference does not have
  assert sum(int(np.prod(sh)) for _, sh, _ in vo.masked_layers('vgg_16', prune_last_layer=False)) == 14710464
  names = [n for n, _, _ in vo.masked_layers('vgg_16')]
  assert names[:3] == ['vgg_16/conv1/conv1_1', 'vgg_16/conv1/conv1_2', 'vgg_16/conv2/conv2_1']
  assert names[-2:] == ['vgg_16/conv5/conv5_3', 'vgg_16/fc8']
  assert [hw for _, _, hw in vo.masked_layers('vgg_16')][::3] == [224, 112, 56, 28, 14]


@pytest.mark.parametrize('vgg_type', sorted(vo.CFG))
@pytest.mark.parametrize('width', [1.0, 0.5, 0.125])
def test_product_plan_matches_the_table(vgg_type, width):
  plan = workloads.vgg_plan(vgg_type, width)
  table = vo.masked_layers(vgg_type, width=width, prune_last_layer=False)
  assert [(s, (3, 3, ci, co)) for s, ci, co, _ in plan] == [(n, sh) for n, sh, _ in table]
  # a pool follows the last conv of stages 1-4
  pools = [s for s, _, _, p in plan if p]
  assert pools == ['%s/conv%d/conv%d_%d' % (vgg_type, i, i, vo.CFG[vgg_type][i - 1]) for i in range(1, 5)]


def test_bad_width_raises_naming_the_layer():
  with pytest.raises(ValueError, match='vgg_16/conv1/conv1_1'):
    workloads.VGG('vgg_16', width=0.1, device='cuda')
  with pytest.raises(ValueError, match='vgg_type'):
    workloads.vgg_plan('vgg_11')


class _Mask(object):

  def __init__(self, name, shape):
    self.name, self.shape, self.dtype = name + '/mask:0', tuple(shape), np.float32


def test_sparsities_bit_exact_vs_reference():
  with open(GOLDEN) as f:
    golden = json.load(f)
  tags = set()
  for case in golden['cases']:
    tags.add(case['tag'])
    want = vo.masked_layers(case['vgg_type'], 1000, case['prune_last_layer'])
    assert [(n, tuple(sh)) for n, sh in case['layers']] == [(n, sh) for n, sh, _ in want]
    masks = [_Mask(n, sh) for n, sh in case['layers']]
    sp = sparse_utils.get_sparsities(masks, case['method'], case['default_sparsity'], case['custom'],
                                     erk_power_scale=case['erk_power_scale'])
    assert set(sp) == set(case['sparsities_hex'])
    for name, hx in case['sparsities_hex'].items():
      assert float(sp[name]).hex() == hx, (case['tag'], name)
    for m in masks:
      size = int(np.prod(m.shape))
      assert size - sparse_utils.get_n_zeros(size, sp[m.name]) == case['nnz'][m.name], (case['tag'], m.name)
  assert len(tags) == 18


def test_regularized_kernels_skip_modules_marked_unregularized():
  """VGG's dense fc8 (prune_last_layer=False) is a contrib conv without weights_regularizer: it is marked
  l2_regularized = False; an unmarked nn.Linear (MobileNet's dense head) stays regularized."""
  m = nn.Module()
  m.head = nn.Linear(8, 4, device='cpu')
  m.fc8 = nn.Linear(8, 4, device='cpu')
  m.fc8.l2_regularized = False
  assert [id(k) for k in regularized_kernels(m)] == [id(m.head.weight)]


def _desc(cin=64, cout=64, h=8, stride=1, k=3):
  d = _cabi.ConvDesc()
  d.batch, d.in_h, d.in_w, d.cin, d.cout = 1, h, h, cin, cout
  d.out_h = d.out_w = (h - 1) // stride + 1
  d.ksize, d.stride, d.pad, d.x_pitch = k, stride, (k - 1) // 2, 0
  return d


def test_relu_entry_points_exist_and_version():
  lib = _cabi.lib()
  assert lib.rigl_version() >= 204
  assert _cabi.ABI_VERSION == 202
  for s in ('rigl_masked_conv2d_fprop_relu', 'rigl_masked_conv2d_dgrad_relu', 'rigl_maxpool2x2_relu_forward',
            'rigl_maxpool2x2_relu_backward', 'rigl_relu_gate'):
    assert s in _cabi.SIGNATURES


def test_relu_conv_entry_points_validate_before_any_cuda_call():
  lib = _cabi.lib()
  p = 1 << 20
  f = lib.rigl_masked_conv2d_fprop_relu
  assert f(_desc(), None, p, p, p, 1 << 20, None) == -1
  assert b'null argument' in lib.rigl_last_error()
  assert f(_desc(), p, None, p, p, 1 << 20, None) == -1
  assert f(_desc(), p, p, None, p, 1 << 20, None) == -1
  assert f(_desc(cout=12), p, p, p, p, 1 << 20, None) == -1
  assert b'multiple of 8' in lib.rigl_last_error()
  for x, y in ((p + 8, p), (p, p + 8)):
    assert f(_desc(), x, p, y, p, 1 << 20, None) == -1
    assert b'16-byte aligned' in lib.rigl_last_error()
  bad = _desc()
  bad.out_h = 0
  assert f(bad, p, p, p, p, 1 << 20, None) == -1

  g = lib.rigl_masked_conv2d_dgrad_relu
  for args in ((None, p, p, p), (p, None, p, p), (p, p, None, p), (p, p, p, None)):
    assert g(_desc(), *args, p, 1 << 20, None) == -1
    assert b'null argument' in lib.rigl_last_error()
  assert g(_desc(cin=12), p, p, p, p, p, 1 << 20, None) == -1
  assert b'multiples of 8' in lib.rigl_last_error()
  for dy, x, dx in ((p + 8, p, p), (p, p + 8, p), (p, p, p + 8)):
    assert g(_desc(), dy, p, x, dx, p, 1 << 20, None) == -1
    assert b'16-byte aligned' in lib.rigl_last_error()
  # no gated variant for the stride-2 parity launches: refused before the driver is touched
  assert g(_desc(stride=2), p, p, p, p, p, 1 << 20, None) == -4
  assert b'no gated dgrad' in lib.rigl_last_error()


def test_relu_pool_and_gate_validate_before_any_cuda_call():
  lib = _cabi.lib()
  p = 1 << 20
  fw, bw = lib.rigl_maxpool2x2_relu_forward, lib.rigl_maxpool2x2_relu_backward
  assert fw(None, 1, 4, 4, 8, p, p, None) == -1
  assert fw(p, 1, 4, 4, 8, None, p, None) == -1
  assert fw(p, 1, 4, 4, 8, p, None, None) == -1
  assert b'null tensor' in lib.rigl_last_error()
  assert fw(p, 1, 4, 4, 12, p, p, None) == -1
  assert fw(p, 1, 1, 4, 8, p, p, None) == -1          # no complete window
  assert b'bad geometry' in lib.rigl_last_error()
  assert fw(p + 8, 1, 4, 4, 8, p, p, None) == -1
  assert fw(p, 1, 4, 4, 8, p, p + 4, None) == -1
  assert b'aligned' in lib.rigl_last_error()
  assert bw(None, p, 1, 4, 4, 8, p, None) == -1
  assert bw(p, None, 1, 4, 4, 8, p, None) == -1
  assert bw(p, p, 1, 4, 4, 8, None, None) == -1
  assert bw(p, p, 1, 4, 4, 4, p, None) == -1
  assert bw(p, p, 1, 4, 4, 8, p + 2, None) == -1
  gate = lib.rigl_relu_gate
  assert gate(None, p, 64, p, None) == -1
  assert gate(p, None, 64, p, None) == -1
  assert gate(p, p, 64, None, None) == -1
  assert gate(p, p, 60, p, None) == -1
  assert b'multiple of 8' in lib.rigl_last_error()
  assert gate(p, p, 0, p, None) == -1
  assert gate(p + 2, p, 64, p, None) == -1
  assert b'16-byte aligned' in lib.rigl_last_error()
