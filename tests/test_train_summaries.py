"""Training summaries without a GPU: argument validation of the C entry points, which parameters the l2 term and the
`fw_*` scalars cover, the key set, and the host arithmetic from per-parameter rows (rigl_b200.summaries)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch
from torch import nn

from rigl_b200 import _cabi, evaluate, sparse_utils, summaries
from rigl_b200.workloads import DenseConv2d, DepthwiseConv2d


def test_plan_create_and_run_validate_before_any_cuda_call():
  lib = _cabi.lib()
  plan = C.c_void_p(None)
  assert lib.rigl_summary_plan_create(None, 1, C.byref(plan)) == -1
  assert b'rigl_summary_plan_create: bad arguments' in lib.rigl_last_error()
  descs = (_cabi.SummaryDesc * 2)()
  descs[0].param, descs[0].grad, descs[0].n = 16, 32, 4
  descs[1].param, descs[1].grad, descs[1].n = 16, None, 4
  assert lib.rigl_summary_plan_create(descs, 2, C.byref(plan)) == -1
  assert b'parameter 1: null tensor or bad size' in lib.rigl_last_error()
  descs[1].grad, descs[1].n = 32, 1 << 31
  assert lib.rigl_summary_plan_create(descs, 2, C.byref(plan)) == -1
  assert b'parameter 1: null tensor or bad size' in lib.rigl_last_error()
  descs[1].n, descs[1].grad = 4, 34
  assert lib.rigl_summary_plan_create(descs, 2, C.byref(plan)) == -1
  assert b'parameter 1: tensors must be float-aligned' in lib.rigl_last_error()
  assert lib.rigl_summary_plan_create(descs, 0, C.byref(plan)) == -1
  assert lib.rigl_summary_plan_run(None, None, None) == -1
  assert b'rigl_summary_plan_run: null argument' in lib.rigl_last_error()
  assert plan.value is None
  assert lib.rigl_summary_plan_destroy(None) == 0


class _Fc8(nn.Module):
  """A dense layer the reference builds without weights_regularizer (VGG's fc8)."""
  l2_regularized = False

  def __init__(self):
    super(_Fc8, self).__init__()
    self.weight = nn.Parameter(torch.zeros(4, 8))


def _fake_masked(scope, shape):
  """Stands in for a masked layer: its weight and its mask's scope and size (the masks need a GPU to build)."""
  return types.SimpleNamespace(weight=nn.Parameter(torch.zeros(shape)),
                               mask=types.SimpleNamespace(scope=scope, size=int(np.prod(shape))))


def _cpu_model():
  m = nn.Module()
  m.stem = DenseConv2d(3, 8, 3, bias=False, device='cpu')
  m.bn = nn.BatchNorm2d(8)
  m.dw = DepthwiseConv2d(8, device='cpu')
  m.fc = nn.Linear(8, 4)
  m.fc8 = _Fc8()
  return m


def test_layout_regularizes_kernels_only_and_takes_the_first_masked_layer_in_registry_order():
  m = _cpu_model()
  masked = [_fake_masked('layer1', (784, 300)), _fake_masked('layer2', (300, 100)), _fake_masked('layer3', (100, 10))]
  # plan order: the optimizer's parameter order, masked weights interleaved with the rest
  params = [m.stem.weight, masked[1].weight, m.bn.weight, m.bn.bias, masked[0].weight, m.dw.weight, m.fc.weight,
            m.fc.bias, m.fc8.weight, masked[2].weight]
  regularized = evaluate.regularized_kernels(m) + [l.weight for l in masked]
  lay = summaries.summary_layout(params, masked, regularized)
  assert lay.reg == [True, True, False, False, True, False, True, False, False, True]
  assert lay.masked == [('layer1', 784 * 300, 4), ('layer2', 300 * 100, 1), ('layer3', 100 * 10, 9)]
  with pytest.raises(ValueError, match='no gradient in the optimizer plan'):
    summaries.summary_layout([p for p in params if p is not m.fc.weight], masked, regularized)
  with pytest.raises(ValueError, match='no gradient in the optimizer plan'):
    summaries.summary_layout([p for p in params if p is not masked[2].weight], masked, regularized)


def test_key_set():
  masked = [_fake_masked('a', (3, 3, 8, 8)), _fake_masked('b', (8, 4))]
  lay = summaries.summary_layout([l.weight for l in masked], masked, [])
  base = ['global_step', 'loss', 'cross_loss', 'reg_loss', 'learning_rate']
  rest = ['grad_norm', 'var_norm', 'fw_nz_weight', 'fw_nz_mask', 'fw_l1_weight', 'global_sparsity',
          'pruning/a/mask/sparsity', 'pruning/b/mask/sparsity']
  assert summaries.summary_keys(lay, dst=True) == base + ['drop_fraction'] + rest
  assert summaries.summary_keys(lay, dst=False) == base + rest
  rows = np.ones((2, 5))
  assert list(summaries.summary_dict(rows, lay, 1.0, 0, 0.1, 1e-4, np.float32(0.3))) == \
      summaries.summary_keys(lay, dst=True)
  assert list(summaries.summary_dict(rows, lay, 1.0, 0, 0.1, 1e-4)) == summaries.summary_keys(lay, dst=False)


def test_summary_dict_arithmetic():
  masked = [_fake_masked('a', (10,)), _fake_masked('b', (7,))]
  other = nn.Parameter(torch.zeros(3))
  params = [other, masked[1].weight, masked[0].weight]
  lay = summaries.summary_layout(params, masked, [l.weight for l in masked])
  rows = np.array([[2.0, 3.0, 1.5, 3, 0],        # other: not regularized, no bitmap
                   [5.0, 7.0, 2.5, 6, 4],        # b
                   [11.0, 13.0, 4.5, 9, 8]])     # a: the first masked layer
  s = summaries.summary_dict(rows, lay, 2.25, 17, 0.05, 1e-4, np.float32(0.125))
  assert s['global_step'] == 17 and s['learning_rate'] == 0.05 and s['drop_fraction'] == 0.125
  assert s['reg_loss'] == 1e-4 * 0.5 * (5.0 + 11.0)
  assert s['cross_loss'] == 2.25 and s['loss'] == 2.25 + s['reg_loss']
  assert s['grad_norm'] == np.sqrt(3.0 + 7.0 + 13.0)
  assert s['var_norm'] == np.sqrt(2.0 + 5.0 + 11.0)
  assert (s['fw_nz_weight'], s['fw_nz_mask'], s['fw_l1_weight']) == (9.0, 8.0, 4.5)
  assert s['pruning/a/mask/sparsity'] == 1.0 - 8 / 10.0
  assert s['pruning/b/mask/sparsity'] == 1.0 - 4 / 7.0
  assert all(type(v) in (int, float) for v in s.values())


def test_global_sparsity_from_counts_is_calculate_sparsity_bit_for_bit():
  rng = np.random.RandomState(0)
  shapes = [(7, 7, 3, 64), (1, 1, 64, 256), (3, 3, 128, 128), (2048, 1000), (5,)]
  masks = [(rng.rand(*s) < rng.uniform(0.02, 0.9)).astype(np.float32) for s in shapes]
  fake = [_fake_masked('l%d' % i, s) for i, s in enumerate(shapes)]
  lay = summaries.summary_layout([l.weight for l in fake], fake, [])
  rows = np.zeros((len(shapes), 5))
  rows[:, summaries.ONES] = [m.sum() for m in masks]
  got = summaries.summary_dict(rows, lay, 0.0, 0, 0.0, 0.0)['global_sparsity']
  want = sparse_utils.calculate_sparsity(masks)
  assert np.float64(got).tobytes() == np.float64(want).tobytes()


def test_summaries_need_the_fused_inner_optimizer():
  m = _cpu_model()
  m.registry = types.SimpleNamespace(layers=lambda: [])
  with pytest.raises(ValueError, match='fused inner optimizer'):
    summaries.TrainSummaries(m, torch.optim.SGD(m.parameters(), lr=0.1))
