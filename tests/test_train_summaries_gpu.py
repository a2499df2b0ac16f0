"""Training summaries on the H100: the batched reduction (rigl_summary_plan_run) against float64 numpy on synthetic
plans, and TrainHarness(summaries=True) against a float64 torch recomputation from the state before each step."""
import ctypes as C
import gc

import numpy as np
import pytest
import torch

from rigl_b200 import _cabi, evaluate, sparse_utils, summaries, workloads
from rigl_b200.evaluate import Evaluator
from rigl_b200.masks import MaskVariable
from rigl_b200.sparse_optimizers_base import host_drop_fraction

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
CHUNK = 8192


@pytest.fixture(autouse=True)
def _free_device_memory():
  """The harness tests capture CUDA graphs over ResNet-50 state: free it, and return the allocator's cache to the
  driver, before the next test, so the tests after these see the device as they would without them."""
  yield
  gc.collect()
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


# ---- the kernel on synthetic plans

def _param(n, masked, gscale, rd, seed, offset=0, special=False):
  """One parameter: weights (optionally 4 bytes off 16-byte alignment), dense gradient with NaN at masked-out
  positions, a random bitmap or none."""
  rng = np.random.RandomState(seed)
  w = rng.standard_normal(n).astype(np.float32)
  w[rng.rand(n) < 0.1] = 0.0
  if special:
    w[::7] = -0.0
    w[3::11] = np.nan
  g = (rng.standard_normal(n) * 1e-2).astype(np.float32)
  on = rng.rand(n) < 0.3 if masked else np.ones(n, bool)
  g[~on] = np.nan
  wt = torch.zeros(n + offset, device=DEV)
  wt[offset:] = torch.from_numpy(w).to(DEV)
  gt = torch.zeros(n + offset, device=DEV)
  gt[offset:] = torch.from_numpy(g).to(DEV)
  mask = MaskVariable('p%d' % seed, (n,), DEV).assign(on.astype(np.float32)) if masked else None
  return dict(w=w, g=g, on=on, masked=masked, gscale=np.float32(gscale), rd=np.float32(rd),
              wt=wt[offset:], gt=gt[offset:], mask=mask)


def _expected(p):
  """float64 [5]: sum w^2, sum g^2, sum |w|, nnz(w), set bits."""
  w = p['w'].astype(np.float64)
  gm = np.where(p['on'], p['g'].astype(np.float64) * np.float64(p['gscale']), 0.0)
  ge = gm + np.float64(p['rd']) * w
  ones = float(p['on'].sum()) if p['masked'] else 0.0
  return np.array([np.sum(w * w), np.sum(ge * ge), np.sum(np.abs(w)), float(np.count_nonzero(p['w'])), ones])


def _bound(p, want):
  """|got - want| allowed per column.  Float64 accumulation over n terms: n * 2^-52 of the sum of |terms|; sum g^2
  also carries the float32 rounding of g (one rounding of an exact product and one fma: 2^-24 of |g| each, so
  2^-22 of g^2)."""
  n = len(p['w'])
  acc = (n + 64) * 2.0 ** -52
  return np.array([acc * want[0], (acc + 2.0 ** -22) * want[1], acc * want[2], 0.0, 0.0])


def _run(params, out=None):
  descs = (_cabi.SummaryDesc * len(params))()
  for d, p in zip(descs, params):
    d.param, d.grad, d.n = p['wt'].data_ptr(), p['gt'].data_ptr(), p['wt'].numel()
    d.mask_bits = p['mask'].bits.data_ptr() if p['mask'] is not None else None
    d.grad_scale, d.reg_decay = float(p['gscale']), float(p['rd'])
  plan = C.c_void_p(None)
  lib = _cabi.lib()
  _cabi.check(lib.rigl_summary_plan_create(descs, len(params), C.byref(plan)), 'rigl_summary_plan_create')
  try:
    out = torch.full((len(params), 5), -1.0, dtype=torch.float64, device=DEV)
    before = _cabi.launch_count()
    _cabi.check(lib.rigl_summary_plan_run(plan, out.data_ptr(), _cabi.stream_ptr()), 'rigl_summary_plan_run')
    assert _cabi.launch_count() - before == 2
    return out.cpu().numpy()
  finally:
    lib.rigl_summary_plan_destroy(plan)


SIZES = [1, 3, 8191, 8192, 8193, 3 * CHUNK + 5]


def _synthetic_plan():
  params, seed = [], 0
  for n in SIZES:
    for masked in (False, True):
      params.append(_param(n, masked, (1.0, 0.5)[seed % 2], (0.0, 1e-4)[(seed // 2) % 2], seed))
      seed += 1
  params.append(_param(8193, True, 0.5, 1e-4, seed, offset=1))            # scalar path
  params.append(_param(3 * CHUNK + 5, True, 1.0, 1e-4, seed + 1, offset=3))
  params.append(_param(3 * CHUNK + 5, False, 1.0, 0.0, seed + 2, special=True))  # -0.0 and NaN weights
  return params


def test_summary_kernel_against_float64():
  params = _synthetic_plan()
  assert any(p['wt'].data_ptr() % 16 for p in params) and any(p['wt'].data_ptr() % 16 == 0 for p in params)
  got = _run(params)
  for i, p in enumerate(params):
    want = _expected(p)
    assert got[i, 3] == want[3] and got[i, 4] == want[4], (i, got[i], want)        # counts exactly
    if np.isnan(p['w']).any():
      # a NaN weight reaches every sum of its parameter, as in float64
      assert np.isnan(got[i, :3]).all()
      continue
    assert np.isfinite(got[i]).all(), i      # NaN dense gradients at masked-out positions are never read into g
    err = np.abs(got[i, :3] - want[:3])
    assert (err <= _bound(p, want)[:3]).all(), (i, err, _bound(p, want))
  # control: one task row fewer must fail the bound
  i = next(k for k, p in enumerate(params) if len(p['w']) == 3 * CHUNK + 5 and not np.isnan(p['w']).any())
  p = params[i]
  part = dict(p, w=p['w'][:CHUNK], g=p['g'][:CHUNK], on=p['on'][:CHUNK])
  short = got[i, :3] - _expected(part)[:3]
  assert (np.abs(short - _expected(p)[:3]) > 100 * _bound(p, _expected(p))[:3]).all()


def test_summary_kernel_is_bit_identical_run_to_run():
  params = _synthetic_plan()
  a, b = _run(params), _run(params)
  assert a.tobytes() == b.tobytes()


# ---- TrainHarness(summaries=True)

def _images(n, size, seed):
  g = torch.Generator(device=DEV).manual_seed(seed)
  return torch.randn(n, 3, size, size, device=DEV, generator=g).to(torch.bfloat16).contiguous(
      memory_format=torch.channels_last)


def _resnet(seed=0):
  torch.manual_seed(seed)
  model = workloads.ResNet50(device=DEV)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=seed)
  model.train()
  return model


def _lr_fn(gs):
  return 0.05 / (1.0 + gs)


def _harness(model, mode, summaries_on=True):
  h = workloads.TrainHarness(model, lr=0.05, frequency=2, end_step=100, lr_schedule=_lr_fn,
                             inner_optimizer='adam' if mode == 'adam' else 'momentum', summaries=summaries_on)
  if mode == 'half_scale':       # the dense gradients as a two-replica SUM would hold them
    h.inner.attach_masked_layers(model.registry.layers(), grad_scale=0.5, other_grad_scale=0.5)
  return h


def _snapshot(model, h):
  ev = Evaluator(model, weight_decay=h.inner.param_groups[0]['weight_decay'], mask_summaries=True)
  ev.reset()
  layers = model.registry.layers()
  return dict(params={id(p): p.detach().double().clone() for p in model.parameters()},
              masks={id(l.weight): l.mask.to_dense().reshape(-1).double().clone() for l in layers},
              gs=h.global_step.value,
              reg_loss=float(evaluate.reg_loss(model, h.inner.param_groups[0]['weight_decay'])),
              evaluator=ev.result(),
              global_sparsity=float(sparse_utils.calculate_sparsity(model.registry.get_masks())))


def _recompute(model, h, snap, loss):
  wd = h.inner.param_groups[0]['weight_decay']
  regularized = {id(w) for w in evaluate.regularized_kernels(model)}
  g2 = w2 = reg = 0.0
  for p, grad, bits, scale in h.inner.plan_params():
    w = snap['params'][id(p)].reshape(-1)
    g = grad.detach().double().reshape(-1) * float(np.float32(scale))
    if bits is not None:
      g = torch.where(snap['masks'][id(p)] != 0, g, torch.zeros_like(g))
    if id(p) in regularized:
      g = g + float(np.float32(wd)) * w
    g2 += float((g * g).sum())
    w2 += float((w * w).sum())
    reg += float((w * w).sum()) if id(p) in regularized else 0.0
  first = model.registry.layers()[0]
  fw = snap['params'][id(first.weight)]
  reg *= wd * 0.5
  # reg_loss against evaluate.reg_loss (float32 sums) and, tighter, against float64
  want = dict(global_step=snap['gs'], cross_loss=float(loss.detach()), reg_loss=snap['reg_loss'], reg_loss_f64=reg,
              loss=float(loss.detach()) + reg, learning_rate=_lr_fn(snap['gs']),
              grad_norm=np.sqrt(g2), var_norm=np.sqrt(w2),
              fw_nz_weight=float(torch.count_nonzero(fw)), fw_l1_weight=float(fw.abs().sum()),
              fw_nz_mask=float(snap['masks'][id(first.weight)].sum()), global_sparsity=snap['global_sparsity'])
  for k, v in snap['evaluator'].items():
    if k.startswith('pruning/'):
      want[k] = v
  return want


_EXACT = ('global_step', 'cross_loss', 'learning_rate', 'fw_nz_weight', 'fw_nz_mask', 'global_sparsity')
_RTOL = dict(reg_loss=1e-5, loss=1e-9, grad_norm=1e-6, var_norm=1e-9, fw_l1_weight=1e-9)


@pytest.mark.parametrize('mode', ['eager', 'graph', 'adam', 'half_scale'])
def test_harness_summaries_match_a_float64_recomputation(mode):
  model = _resnet(seed=3)
  h = _harness(model, mode)
  x, y = _images(4, 64, 1), torch.randint(0, 1000, (4,), device=DEV)
  if mode == 'graph':
    assert h.enable_cuda_graph(x, y)
  with pytest.raises(RuntimeError, match='before the first step'):
    h.summaries()
  updates = 0
  for step in range(5):
    x, y = _images(4, 64, 10 + step), torch.randint(0, 1000, (4,), device=DEV)
    snap = _snapshot(model, h)
    loss = h.step(x, y)
    s = h.summaries()
    want = _recompute(model, h, snap, loss)
    update = h.opt.last_update_was_mask_update
    updates += update
    want['drop_fraction'] = float(host_drop_fraction('cosine', 0.3, snap['gs'], 0, 100)) if update else 0.0
    assert abs(s['reg_loss'] - want.pop('reg_loss_f64')) <= 1e-9 * s['reg_loss']
    assert sorted(s) == sorted(want)
    for k, v in want.items():
      if k in _EXACT or k.startswith('pruning/') or k == 'drop_fraction':
        assert s[k] == v, (mode, step, k, s[k], v)
      else:
        assert abs(s[k] - v) <= _RTOL[k] * abs(v), (mode, step, k, s[k], v)
    assert s['grad_norm'] > 0 and s['fw_nz_mask'] < s['fw_nz_weight']
  assert updates >= 2        # mask-update steps are summarised with their pre-update masks


def test_mnist_fc_key_set_and_first_layer():
  model = workloads.MnistFC(device=DEV)
  workloads.init_masks(model, 'random', 0.9, {'layer2': 0.81, 'layer3': 0.0}, seed=0)
  h = workloads.TrainHarness(model, lr=0.1, frequency=4, end_step=1000, summaries=True)
  x = torch.randn(64, 784, device=DEV)
  h.step(x, x[:, :10].argmax(1).long())
  s = h.summaries()
  lay = h._summaries.layout
  assert list(s) == summaries.summary_keys(lay, dst=True)
  assert [scope for scope, _, _ in lay.masked] == ['layer1', 'layer2', 'layer3']
  assert s['fw_nz_mask'] == float(model.registry.get_masks()[0].count_ones())
  # every masked kernel is regularized; the biases are not
  params = [p for p, _, _, _ in h.inner.plan_params()]
  kernels = {id(l.weight) for l in model.registry.layers()}
  assert lay.reg == [id(p) in kernels for p in params]


def test_capture_after_eager_steps_with_summaries():
  model = _resnet(seed=6)
  h = _harness(model, 'eager')
  x, y = _images(4, 64, 1), torch.randint(0, 1000, (4,), device=DEV)
  h.step(x, y)
  h.step(x, y)
  assert h.enable_cuda_graph(x, y)
  h.step(x, y)
  assert np.isfinite(h.summaries()['grad_norm'])


def test_summaries_are_off_by_default():
  x, y = _images(4, 64, 1), torch.randint(0, 1000, (4,), device=DEV)
  off, on = _harness(_resnet(seed=4), 'eager', False), _harness(_resnet(seed=4), 'eager', True)
  with pytest.raises(RuntimeError, match='without summaries'):
    off.summaries()
  for step in range(3):
    counts = []
    for h in (off, on):
      before = _cabi.launch_count()
      h.step(x, y)
      torch.cuda.synchronize()
      counts.append(_cabi.launch_count() - before)
    assert counts[1] == counts[0] + 2, counts
  g_off, g_on = _harness(_resnet(seed=5), 'eager', False), _harness(_resnet(seed=5), 'eager', True)
  assert g_off.enable_cuda_graph(x, y) and g_on.enable_cuda_graph(x, y)
  assert g_off.graph_kernel_launches == g_on.graph_kernel_launches
  la, lb = g_off.step(x, y), g_on.step(x, y)
  assert torch.equal(la, lb)
  for pa, pb in zip(g_off.model.parameters(), g_on.model.parameters()):
    assert torch.equal(pa, pb)
