"""optim.FusedAdam on the CPU: the numpy restatement of tf.train.AdamOptimizer's update (tests/adam_oracle.py)
against a float64 evaluation of the formula and against torch.optim.Adam, and argument validation of the
constructor, the harness option and the C ABI (all before any CUDA call)."""
import ctypes as C

import numpy as np
import pytest
import torch

from rigl_b200 import _cabi
import adam_oracle as ao

F32 = np.float32


def _state(rng, n, tiny_v=False):
  w = rng.standard_normal(n).astype(F32)
  m = (0.1 * rng.standard_normal(n)).astype(F32)
  v = (1e-14 if tiny_v else 1e-2) * rng.rand(n).astype(F32)
  g = rng.standard_normal(n).astype(F32)
  return w, m, v.astype(F32), g


def test_oracle_matches_float64_formula():
  rng = np.random.RandomState(0)
  w, m, v, g = _state(rng, 4096)
  lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
  p1, p2 = F32(b1), F32(b2)
  for _ in range(5):
    wg, mg, vg = ao.adam_step(w, m, v, g, lr, b1, b2, eps, p1, p2)
    alpha = lr * np.sqrt(1 - np.float64(p2)) / (1 - np.float64(p1))
    m64 = m.astype(np.float64) + (g.astype(np.float64) - m) * (1 - np.float64(F32(b1)))
    v64 = v.astype(np.float64) + (np.float64(1) * g * g - v) * (1 - np.float64(F32(b2)))
    w64 = w.astype(np.float64) - m64 * alpha / (np.sqrt(v64) + eps)
    assert wg.dtype == mg.dtype == vg.dtype == F32
    # (absolute floors: the float32 rounding of g - m, g * g and w, where the result cancels to near zero)
    np.testing.assert_allclose(mg, m64, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(vg, v64, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(wg - w, w64 - w, rtol=1e-3, atol=3e-7)      # the update itself, not just w
    w, m, v = wg, mg, vg
    p1, p2 = ao.advance_powers(p1, p2, b1, b2)
  assert p1 == F32(F32(F32(F32(F32(F32(0.9) * F32(0.9)) * F32(0.9)) * F32(0.9)) * F32(0.9)) * F32(0.9))


def _torch_adam_run(w, m, v, grads, lr, b1, b2, eps, wd):
  p = torch.nn.Parameter(torch.from_numpy(w.copy()))
  opt = torch.optim.Adam([p], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
  for g in grads:
    p.grad = torch.from_numpy(g.copy())
    opt.step()
  st = opt.state[p]
  return p.detach().numpy(), st['exp_avg'].numpy(), st['exp_avg_sq'].numpy()


def _oracle_run(w, m, v, grads, lr, b1, b2, eps, wd):
  p1, p2 = F32(b1), F32(b2)
  for g in grads:
    w, m, v = ao.adam_step(w, m, v, ao.optimizer_grad(w, g, weight_decay=wd), lr, b1, b2, eps, p1, p2)
    p1, p2 = ao.advance_powers(p1, p2, b1, b2)
  return w, m, v


def test_oracle_agrees_with_torch_adam_without_epsilon():
  """eps = 0: TF's eps-hat form and torch's are the same algorithm up to float32 rounding.  The betas are exact in
  float32 (as is 1 - beta): TF forms 1 - beta from the float32 beta, torch in double, which for 0.999 alone moves
  v by 1.3e-5 relative."""
  rng = np.random.RandomState(1)
  n = 2048
  w = rng.standard_normal(n).astype(F32)
  zeros = np.zeros(n, F32)
  grads = [rng.standard_normal(n).astype(F32) for _ in range(4)]
  b1, b2 = 0.875, 1 - 2.0 ** -9
  got = _oracle_run(w, zeros, zeros, grads, 1e-2, b1, b2, 0.0, 1e-2)
  want = _torch_adam_run(w, zeros, zeros, grads, 1e-2, b1, b2, 0.0, 1e-2)
  for a, b in zip(got, want):
    np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6 * np.abs(b).max())     # (floor: values near zero)
  np.testing.assert_allclose(got[0] - w, want[0] - w, rtol=1e-4, atol=1e-7)


def test_oracle_differs_from_torch_adam_where_v_is_tiny():
  """eps = 1e-8 and |g| ~ 1e-6 (a masked-out weight under weight decay, a regrown connection): TF adds eps to
  sqrt(v) before the bias correction, i.e. an effective eps / sqrt(1 - beta2^t) ~ 30x larger at t = 1."""
  rng = np.random.RandomState(2)
  n = 1024
  w = rng.standard_normal(n).astype(F32)
  zeros = np.zeros(n, F32)
  grads = [(1e-6 * rng.standard_normal(n)).astype(F32)]
  got = _oracle_run(w, zeros, zeros, grads, 1e-3, 0.9, 0.999, 1e-8, 0.0)
  want = _torch_adam_run(w, zeros, zeros, grads, 1e-3, 0.9, 0.999, 1e-8, 0.0)
  # the moments agree (up to 1 - beta formed in float32 vs double) ...
  np.testing.assert_allclose(got[1], want[1], rtol=5e-5)
  np.testing.assert_allclose(got[2], want[2], rtol=5e-5)
  step_tf, step_torch = np.abs(got[0] - w), np.abs(want[0] - w)
  ratio = np.median(step_tf[step_torch > 0] / step_torch[step_torch > 0])
  assert ratio < 0.9                                     # ... the steps do not: TF's is measurably smaller
  # with gradients far from zero the two forms agree again
  grads = [(rng.choice([-1., 1.], n) * (0.5 + rng.rand(n))).astype(F32)]
  got = _oracle_run(w, zeros, zeros, grads, 1e-3, 0.9, 0.999, 1e-8, 0.0)
  want = _torch_adam_run(w, zeros, zeros, grads, 1e-3, 0.9, 0.999, 1e-8, 0.0)
  np.testing.assert_allclose(got[0] - w, want[0] - w, rtol=1e-3, atol=3e-7)


@pytest.mark.parametrize('kwargs', [dict(lr=-1e-3), dict(beta1=1.0), dict(beta1=-0.1), dict(beta2=1.0),
                                    dict(epsilon=-1e-8), dict(weight_decay=-1.0), dict(lr=float('nan'))])
def test_fused_adam_rejects_bad_hyper_parameters(kwargs):
  from rigl_b200.optim import FusedAdam
  with pytest.raises(ValueError):
    FusedAdam([torch.nn.Parameter(torch.zeros(4))], **kwargs)


def test_fused_adam_rejects_bad_parameters_before_any_cuda_call():
  from rigl_b200.optim import FusedAdam
  with pytest.raises(ValueError):
    FusedAdam([torch.nn.Parameter(torch.zeros(4))])                               # not on a CUDA device
  with pytest.raises(ValueError):
    FusedAdam([{'params': [torch.nn.Parameter(torch.zeros(4))]},
               {'params': [torch.nn.Parameter(torch.zeros(4))]}])                  # two groups
  with pytest.raises(ValueError):
    FusedAdam([])


def test_harness_adam_needs_the_fused_path():
  from rigl_b200 import workloads
  model = torch.nn.Linear(2, 2)
  with pytest.raises(ValueError):
    workloads.TrainHarness(model, inner_optimizer='adam', fused_optimizer=False)
  with pytest.raises(ValueError):
    workloads.TrainHarness(model, inner_optimizer='rmsprop')


def test_adam_abi_validates_before_any_cuda_call():
  lib = _cabi.lib()
  plan = C.c_void_p(None)
  assert lib.rigl_adam_plan_create(None, 1, C.byref(plan)) == -1
  d = (_cabi.AdamDesc * 1)()
  d[0].param, d[0].m, d[0].v, d[0].grad, d[0].n = 16, None, 16, 16, 4        # no first moment 
  assert lib.rigl_adam_plan_create(d, 1, C.byref(plan)) == -1
  assert b'null tensor' in lib.rigl_last_error()
  d[0].m, d[0].param = 16, 18                                                 # not float-aligned
  assert lib.rigl_adam_plan_create(d, 1, C.byref(plan)) == -1
  assert lib.rigl_adam_plan_run(None, 16, 16, 0.9, 0.999, 1e-8, None) == -1
  assert lib.rigl_adam_plan_run(16, 16, None, 0.9, 0.999, 1e-8, None) == -1
  # a plan pointer that is never dereferenced: the hyper-parameters are checked first
  assert lib.rigl_adam_plan_run(16, 16, 16, 1.0, 0.999, 1e-8, None) == -1
  assert lib.rigl_adam_plan_run(16, 16, 16, 0.9, 0.999, -1.0, None) == -1
  assert b'beta1' in lib.rigl_last_error()
