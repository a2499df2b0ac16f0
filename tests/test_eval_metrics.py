"""Evaluation metric semantics (rigl_b200.evaluate) on hand-built logits, and the fused conv + BN entry point's
host-side checks; no GPU needed."""
import ctypes as C

import numpy as np
import pytest
import torch
from torch import nn

from rigl_b200 import _cabi
from rigl_b200.evaluate import batch_metrics, reg_loss, regularized_kernels
from rigl_b200.workloads import DenseConv2d, DepthwiseConv2d


def _m(logits, labels, ls=0.0, k=5):
  return batch_metrics(torch.tensor(logits, dtype=torch.float32), torch.tensor(labels), ls, k).tolist()


def _np_cross(logits, labels, ls):
  z = np.asarray(logits, np.float64)
  logp = z - z.max(1, keepdims=True)
  logp = logp - np.log(np.exp(logp).sum(1, keepdims=True))
  soft = np.eye(z.shape[1])[labels] * (1 - ls) + ls / z.shape[1]
  return float(-(soft * logp).sum(1).mean())


def test_argmax_ties_pick_the_lowest_index():
  logits = [[1., 3., 3., 0.], [2., 2., 2., 2.], [0., 5., 1., 5.]]
  top1, _, _ = _m(logits, [1, 0, 3], k=1)
  assert top1 == 2          # rows 0 and 1 hit; row 2's argmax is class 1, not 3


def test_in_top_k_counts_boundary_ties_as_in():
  # target 0 has 4 classes strictly above it and 3 tied with it: in the top 5 (fewer than 5 strictly higher)
  row = [1., 2., 2., 2., 2., 1., 1., 1.]
  assert _m([row], [0], k=5)[1] == 1
  # 5 strictly higher: out
  assert _m([[1., 2., 2., 2., 2., 2., 1., 1.]], [0], k=5)[1] == 0
  # k = 1 with a tie at the top: both tied classes are in
  assert _m([[3., 3., 0.]], [1], k=1)[1] == 1


def test_in_top_k_non_finite_rows_miss():
  nan, inf = float('nan'), float('inf')
  logits = [[9., 0., 0., 0., 0., 0., nan], [inf, 0., 0., 0., 0., 0., 0.], [0., 1., 2., 3., 4., 5., 6.],
            [-inf, 1., 2., 3., 4., 5., 6.]]
  _, top5, _ = _m(logits, [0, 0, 6, 6], k=5)
  assert top5 == 1          # only the finite row 2 counts


def test_out_of_range_labels_miss():
  top1, top5, _ = _m([[1., 0.], [0., 1.]], [2, -1], k=1)
  assert top1 == 0 and top5 == 0


@pytest.mark.parametrize('ls', [0.0, 0.1, 0.3])
def test_label_smoothed_cross_entropy(ls):
  rng = np.random.RandomState(0)
  logits = rng.randn(6, 10).astype(np.float32) * 3
  labels = rng.randint(0, 10, 6)
  _, _, cross = _m(logits, labels.tolist(), ls)
  assert cross == pytest.approx(6 * _np_cross(logits, labels, ls), rel=1e-5)


def test_cross_loss_is_the_batch_size_weighted_mean_of_batch_means():
  rng = np.random.RandomState(1)
  batches = [(rng.randn(n, 7).astype(np.float32), rng.randint(0, 7, n)) for n in (5, 2, 9)]
  total = sum(_m(z, y.tolist(), 0.1)[2] for z, y in batches)
  want = sum(len(y) * _np_cross(z, y, 0.1) for z, y in batches) / 16.0
  assert total / 16.0 == pytest.approx(want, rel=1e-5)
  assert total / 16.0 != pytest.approx(np.mean([_np_cross(z, y, 0.1) for z, y in batches]), rel=1e-3)


def test_reg_loss_covers_conv_and_dense_kernels_but_not_depthwise():
  torch.manual_seed(0)
  m = nn.Module()
  m.conv = DenseConv2d(3, 8, 3, bias=False, device='cpu')
  m.dw = DepthwiseConv2d(8, device='cpu')
  m.fc = nn.Linear(8, 4, device='cpu')
  ks = regularized_kernels(m)
  assert [id(k) for k in ks] == [id(m.conv.weight), id(m.fc.weight)]
  want = 1e-4 * 0.5 * (m.conv.weight.detach().double().pow(2).sum() + m.fc.weight.detach().double().pow(2).sum())
  assert float(reg_loss(m, 1e-4)) == pytest.approx(float(want), rel=1e-5)


def _desc(cin=64, cout=64, h=8):
  d = _cabi.ConvDesc()
  d.batch, d.in_h, d.in_w, d.cin, d.out_h, d.out_w, d.cout = 1, h, h, cin, h, h, cout
  d.ksize, d.stride, d.pad, d.x_pitch = 1, 1, 0, 0
  return d


def test_fused_bn_entry_point_and_version():
  lib = _cabi.lib()
  assert lib.rigl_version() >= 203
  assert 'rigl_masked_conv2d_fprop_bnapply' in _cabi.SIGNATURES


def test_fused_bn_entry_point_validates_before_any_cuda_call():
  lib = _cabi.lib()
  f = lib.rigl_masked_conv2d_fprop_bnapply
  p = 1 << 20
  assert f(_desc(), None, p, None, p, p, 1, p, p, 1 << 20, None) == -1
  assert b'null argument' in lib.rigl_last_error()
  assert f(_desc(), p, p, None, None, p, 1, p, p, 1 << 20, None) == -1
  assert f(_desc(), p, p, None, p, None, 1, p, p, 1 << 20, None) == -1
  assert f(_desc(), p, p, None, p, p, 1, None, p, 1 << 20, None) == -1
  assert f(_desc(cout=12), p, p, None, p, p, 1, p, p, 1 << 20, None) == -1
  assert b'multiple of 8' in lib.rigl_last_error()
  for x, y, r in ((p + 8, p, None), (p, p + 8, None), (p, p, p + 8)):
    assert f(_desc(), x, p, r, p, p, 0, y, p, 1 << 20, None) == -1
    assert b'16-byte aligned' in lib.rigl_last_error()
  bad = _desc()
  bad.out_h = 0
  assert f(bad, p, p, None, p, p, 1, p, p, 1 << 20, None) == -1
