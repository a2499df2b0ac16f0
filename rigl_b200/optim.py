"""The wrapped ("inner") optimizers of the reference's training scripts, each on one fused launch.

`FusedMomentumSGD` is tf.train.MomentumOptimizer(learning_rate, momentum, use_nesterov) + the l2 term on the raw
weights, as imagenet_train_eval.py:355-365 / cifar resnet_train_eval.py build it under the sparse wrapper;
`FusedAdam` is tf.train.AdamOptimizer + the same l2 term (imagenet_train_eval.py:355-358 `--use_adam`,
mnist_train_eval.py:247-261, rigl_tf2/utils.py get_optimizer).  Each updates every parameter of a model in ONE
kernel (csrc/sgd.cu).  For masked layers the gradient it consumes is `mask * dense_grad` formed while loading the
dense gradient (sparse_optimizers_base.py:478-485), so the masked gradient tensor is never materialised.  The
learning rate lives in device memory: `set_lr` (or assigning param_groups[...]['lr'] between steps) takes effect in
CUDA-graph replays without re-capture.

They are `torch.optim.Optimizer`s: the sparse wrappers only call `.step()`, `.zero_grad()`, `.state` (slot names
'momentum_buffer', as torch.optim.SGD; 'exp_avg' / 'exp_avg_sq', as torch.optim.Adam) and `.param_groups`.
"""
import ctypes as C

import torch

from . import _cabi


class _FusedInnerOptimizer(torch.optim.Optimizer):
  """What the fused optimizers share: masked-layer gradients, the device learning rate, the launch plan (built
  for the current gradient / slot buffers, reused while they stay the same) and `step` under stream capture.
  A subclass names its C entry points and supplies `_slots(p)` (its per-parameter slot tensors, in plan order),
  `_create_plan(ents)` and `_run_plan()`."""

  _name = None
  _plan_destroy = None

  def __init__(self, params, defaults):
    super(_FusedInnerOptimizer, self).__init__(params, defaults)
    if len(self.param_groups) != 1:
      raise ValueError('%s supports a single parameter group' % self._name)
    self._masked = {}            # id(weight) -> masked layer (dense gradient + bitmap replace weight.grad)
    self._grad_scale = 1.0
    self._plan, self._key = C.c_void_p(None), None
    self._lr_dev, self._lr_uploaded = None, None

  def __del__(self):
    try:
      self._destroy()
    except Exception:
      pass

  def _destroy(self):
    if self._plan and self._plan.value:
      getattr(_cabi.lib(), self._plan_destroy)(self._plan)
      self._plan = C.c_void_p(None)

  # ---- masked layers: consume mask * dense_grad (* grad_scale) instead of weight.grad
  def attach_masked_layers(self, layers, grad_scale=1.0, other_grad_scale=1.0):
    """grad_scale multiplies the masked layers' dense gradients, other_grad_scale every other gradient
    (1 / replicas when the buffers hold cross-replica SUMS)."""
    self._masked = {id(l.weight): l for l in layers}
    self._grad_scale = float(grad_scale)
    self._other_scale = float(other_grad_scale)
    self._key = None
    return self

  # ---- learning rate in device memory
  def set_lr(self, lr):
    """Sets the learning rate (eagerly: call it OUTSIDE graph capture / between replays)."""
    lr = float(lr)
    self.param_groups[0]['lr'] = lr
    self._upload_lr()

  def _upload_lr(self):
    g = self.param_groups[0]
    dev = g['params'][0].device
    if self._lr_dev is None or self._lr_dev.device != dev:
      self._lr_dev = torch.zeros(1, dtype=torch.float32, device=dev)
      self._lr_uploaded = None
    lr = float(g['lr'])
    if self._lr_uploaded != lr:
      self._lr_dev.fill_(lr)
      self._lr_uploaded = lr

  def _plan_extra_key(self):
    """Device buffers the plan's launches read besides the per-parameter ones."""
    return ()

  def plan_params(self):
    """(param, grad, bitmap or None, grad_scale) of every parameter the next step updates, in plan order: a masked
    layer's weight with its dense gradient and bitmap, every other parameter that has a `.grad`."""
    out = []
    for p in self.param_groups[0]['params']:
      layer = self._masked.get(id(p))
      if layer is not None:
        grad, bits, scale = layer.masked_weights.dense_grad, layer.mask.bits, self._grad_scale
      else:
        if p.grad is None:
          continue
        grad, bits, scale = p.grad, None, getattr(self, '_other_scale', 1.0)
      if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous() or grad.dtype != torch.float32 \
          or not grad.is_contiguous():
        raise ValueError('%s needs contiguous float32 CUDA parameters and gradients' % self._name)
      out.append((p, grad, bits, float(scale)))
    return out

  @torch.no_grad()
  def prepare(self):
    """Creates the slots, the device learning rate and the launch plan for the CURRENT gradient
    buffers.  Allocates, so it cannot run under stream capture: call it once before capturing `step()`
    (TrainHarness.enable_cuda_graph does)."""
    g = self.param_groups[0]
    self._upload_lr()
    ents = []
    for p, grad, bits, scale in self.plan_params():
      ents.append((p.data_ptr(), tuple(s.data_ptr() for s in self._slots(p)), grad.data_ptr(),
                   0 if bits is None else bits.data_ptr(), p.numel(), float(g['weight_decay']), scale))
    key = (tuple(ents), self._plan_extra_key())
    if key != self._key:
      self._destroy()
      if ents:
        self._plan = self._create_plan(ents)
      self._key = key

  def _current_key_matches(self):
    """Cheap check under capture: the gradient buffers are the ones the plan was built for."""
    if self._key is None:
      return False
    ents = self._key[0]
    i = 0
    for p in self.param_groups[0]['params']:
      layer = self._masked.get(id(p))
      grad = layer.masked_weights.dense_grad if layer is not None else p.grad
      if grad is None:
        continue
      if i >= len(ents) or ents[i][0] != p.data_ptr() or ents[i][2] != grad.data_ptr():
        return False
      i += 1
    return i == len(ents)

  @torch.no_grad()
  def step(self, closure=None):
    loss = None
    if closure is not None:
      with torch.enable_grad():
        loss = closure()
    if torch.cuda.is_current_stream_capturing():
      if not self._current_key_matches():
        raise RuntimeError('%s.step() under stream capture needs prepare() with the same gradient '
                           'buffers first' % self._name)
    else:
      self.prepare()
    if self._plan and self._plan.value:
      self._run_plan()
    return loss


class FusedMomentumSGD(_FusedInnerOptimizer):

  _name = 'FusedMomentumSGD'
  _plan_destroy = 'rigl_sgd_plan_destroy'

  def __init__(self, params, lr=0.1, momentum=0.9, nesterov=True, weight_decay=0.0):
    if momentum < 0 or lr < 0 or weight_decay < 0:
      raise ValueError('lr, momentum and weight_decay must be non-negative')
    super(FusedMomentumSGD, self).__init__(params, dict(lr=lr, momentum=momentum, nesterov=nesterov,
                                                        weight_decay=weight_decay))

  def _slots(self, p):
    st = self.state[p]
    if 'momentum_buffer' not in st:
      st['momentum_buffer'] = torch.zeros_like(p, memory_format=torch.preserve_format)
    return (st['momentum_buffer'],)

  def _create_plan(self, ents):
    descs = (_cabi.SgdDesc * len(ents))()
    for d, (pp, (mp,), gp, bp, n, wd, sc) in zip(descs, ents):
      d.param, d.momentum, d.grad, d.mask_bits, d.n, d.weight_decay, d.grad_scale = pp, mp, gp, bp or None, n, wd, sc
    plan = C.c_void_p(None)
    _cabi.check(_cabi.lib().rigl_sgd_plan_create(descs, len(ents), C.byref(plan)), 'rigl_sgd_plan_create')
    return plan

  def _run_plan(self):
    g = self.param_groups[0]
    _cabi.check(_cabi.lib().rigl_sgd_plan_run(self._plan, self._lr_dev.data_ptr(), float(g['momentum']),
                                              int(bool(g['nesterov'])), _cabi.stream_ptr()), 'rigl_sgd_plan_run')


class FusedAdam(_FusedInnerOptimizer):
  """tf.train.AdamOptimizer(learning_rate, beta1, beta2, epsilon) + the l2 term on the raw weights: TF 1.x
  ApplyAdam, which adds epsilon to sqrt(v) BEFORE the bias correction,
    w -= lr * sqrt(1 - beta2^t) / (1 - beta1^t) * m / (sqrt(v) + epsilon),
  where torch.optim.Adam adds it after.  The two differ where v is tiny -- in RigL training that is every
  masked-out weight (its gradient is only weight_decay * w) and every regrown connection (m = v = 0).

  Slots `state[p]['exp_avg']` (TF 'm') and `state[p]['exp_avg_sq']` (TF 'v') exist from construction on, as TF
  creates them with the graph: a RigL update at global_step 0 resets them like any later one.  That reset
  (base.py:555-564) writes dense_grad * initial_acc_scale into BOTH slots, so with initial_acc_scale > 0 the second
  moment is negative wherever the gradient is, and those weights become NaN at the next step, as in the reference:
  use initial_acc_scale = 0 with Adam.  The bias
  correction powers beta1^t, beta2^t are one device float32[2] (`non_slot_variables()`), initialised to
  (beta1, beta2) and advanced on the device after every step, so captured steps replay with no host work."""

  _name = 'FusedAdam'
  _plan_destroy = 'rigl_adam_plan_destroy'

  def __init__(self, params, lr=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, weight_decay=0.0):
    if not (lr >= 0 and weight_decay >= 0 and epsilon >= 0):
      raise ValueError('lr, epsilon and weight_decay must be non-negative')
    if not (0 <= beta1 < 1 and 0 <= beta2 < 1):
      raise ValueError('beta1 and beta2 must lie in [0, 1)')
    super(FusedAdam, self).__init__(params, dict(lr=lr, beta1=beta1, beta2=beta2, epsilon=epsilon,
                                                 weight_decay=weight_decay))
    params = self.param_groups[0]['params']
    if not params:
      raise ValueError('FusedAdam got an empty parameter list')
    for p in params:
      if not p.is_cuda or p.dtype != torch.float32 or not p.is_contiguous():
        raise ValueError('FusedAdam needs contiguous float32 CUDA parameters')
    dev = params[0].device
    if any(p.device != dev for p in params):
      raise ValueError('FusedAdam needs every parameter on one device')
    for p in params:
      st = self.state[p]
      st['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
      st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
    self._powers = torch.tensor([beta1, beta2], dtype=torch.float32, device=dev)

  def non_slot_variables(self):
    """{'beta1_power', 'beta2_power'}: one-element views of the device powers (TF's variable names)."""
    return {'beta1_power': self._powers[0:1], 'beta2_power': self._powers[1:2]}

  def state_dict(self):
    sd = super(FusedAdam, self).state_dict()
    sd['powers'] = self._powers.detach().clone()
    return sd

  def load_state_dict(self, state_dict):
    state_dict = dict(state_dict)
    powers = state_dict.pop('powers', None)
    super(FusedAdam, self).load_state_dict(state_dict)
    if powers is not None:
      with torch.no_grad():
        self._powers.copy_(torch.as_tensor(powers, dtype=torch.float32))       # in place: captured graphs stay valid

  def _slots(self, p):
    st = self.state[p]
    return st['exp_avg'], st['exp_avg_sq']

  def _plan_extra_key(self):
    return (self._powers.data_ptr(),)

  def _create_plan(self, ents):
    descs = (_cabi.AdamDesc * len(ents))()
    for d, (pp, (mp, vp), gp, bp, n, wd, sc) in zip(descs, ents):
      d.param, d.m, d.v, d.grad, d.mask_bits, d.n, d.weight_decay, d.grad_scale = \
          pp, mp, vp, gp, bp or None, n, wd, sc
    plan = C.c_void_p(None)
    _cabi.check(_cabi.lib().rigl_adam_plan_create(descs, len(ents), C.byref(plan)), 'rigl_adam_plan_create')
    return plan

  def _run_plan(self):
    g = self.param_groups[0]
    _cabi.check(_cabi.lib().rigl_adam_plan_run(self._plan, self._lr_dev.data_ptr(), self._powers.data_ptr(),
                                               float(g['beta1']), float(g['beta2']), float(g['epsilon']),
                                               _cabi.stream_ptr()), 'rigl_adam_plan_run')


def imagenet_lr_schedule(current_epoch, base_learning_rate=0.1, train_batch_size=4096, architecture='resnet',
                         training_steps_multiplier=1.0):
  """lr_schedule of imagenet_train_eval.py:317-330 (step schedule, no SGDR) with set_lr_schedule :280-299:
  (multiplier, start epoch) pairs, linear ramp from 0 to the first multiplier over the first start epoch."""
  if architecture in ('mobilenet_v1', 'mobilenet_v2'):
    sched = [(1.0, 8), (0.1, 40), (0.01, 75), (0.001, 95), (.0003, 120)]
  elif architecture == 'resnet' or architecture.startswith('vgg'):
    sched = [(1.0, 0), (0.1, 30), (0.01, 70), (0.001, 90), (.0001, 120)]
  else:
    raise ValueError('Unknown architecture ' + architecture)
  if training_steps_multiplier != 1.0:
    sched = [(x, y * training_steps_multiplier) for x, y in sched]
  scaled_lr = base_learning_rate * (train_batch_size / 256.0)
  # the ramp term is only selected while current_epoch < first start epoch (tf.where), so a zero-length ramp
  # (ResNet) is never read
  rate = scaled_lr * sched[0][0] * current_epoch / sched[0][1] if sched[0][1] > 0 else scaled_lr * sched[0][0]
  for mult, start_epoch in sched:
    if not current_epoch < start_epoch:
      rate = scaled_lr * mult
  return rate


def make_imagenet_lr_fn(base_learning_rate=0.1, train_batch_size=4096, num_train_images=1281167,
                        architecture='resnet', training_steps_multiplier=1.0):
  """global_step -> learning rate, as train_function computes it (imagenet_train_eval.py:350-354)."""
  steps_per_epoch = num_train_images / float(train_batch_size)

  def lr_fn(global_step):
    return imagenet_lr_schedule(float(int(global_step)) / steps_per_epoch, base_learning_rate, train_batch_size,
                                architecture, training_steps_multiplier)
  return lr_fn
