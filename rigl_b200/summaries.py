"""Per-step training summaries: the scalars the reference's `train_function` logs on every step
(imagenet_train_eval.py:431-470, through utils.host_call_fn / utils.mask_summaries, utils.py:59-90).

    harness = TrainHarness(model, ..., summaries=True)
    loss = harness.step(images, labels)
    s = harness.summaries()        # dict of floats; one device synchronisation

A summary describes the state the step's loss was computed at: the weights and masks before the step's optimizer
or mask update, the gradients after the data-parallel exchange and scaling, and the global step, learning rate and
drop fraction the step used.  The per-parameter sums come from one batched reduction over every parameter of the
fused inner optimizer's plan (csrc/sgd.cu `rigl_summary_plan_run`, two launches, no synchronisation); the host
only adds a few hundred float64 rows.  DESIGN.md 5 pins each key.
"""
import collections
import ctypes as C
import math

import numpy as np
import torch

from . import _cabi
from . import evaluate
from . import sparse_utils

# Columns of a result row (csrc/sgd.cu).
SUM_W2, SUM_G2, SUM_ABS_W, NNZ_W, ONES = range(5)
_COLS = 5

# reg: per plan row, whether the parameter is an l2-regularized kernel; masked: (scope, size, plan row) of every
# masked layer in registry order (the first one is the reference's `fw_*` layer).
Layout = collections.namedtuple('Layout', ['reg', 'masked'])


def summary_layout(params, masked_layers, regularized):
  """Host-only.  params: the plan's parameters in order; masked_layers: the registry's layers in order (each with
  `.weight` and `.mask.scope` / `.mask.size`); regularized: evaluate.regularized_kernels(model).  Raises ValueError
  when a masked layer or a regularized kernel is not in the plan (its terms would be missing)."""
  rows = {id(p): i for i, p in enumerate(params)}
  reg_ids = {id(w) for w in regularized}
  missing = [w for w in regularized if id(w) not in rows] + [l.weight for l in masked_layers if id(l.weight) not in rows]
  if missing:
    raise ValueError('training summaries: %d regularized or masked weight(s) have no gradient in the optimizer plan'
                     % len(missing))
  return Layout(reg=[id(p) in reg_ids for p in params],
                masked=[(l.mask.scope, int(l.mask.size), rows[id(l.weight)]) for l in masked_layers])


def summary_keys(layout, dst):
  """The keys of a summary dict, in order (dst: the sparse optimizer is a drop/grow one and logs drop_fraction)."""
  keys = ['global_step', 'loss', 'cross_loss', 'reg_loss', 'learning_rate']
  if dst:
    keys.append('drop_fraction')
  keys += ['grad_norm', 'var_norm']
  if layout.masked:
    keys += ['fw_nz_weight', 'fw_nz_mask', 'fw_l1_weight', 'global_sparsity']
  keys += ['pruning/%s/mask/sparsity' % scope for scope, _, _ in layout.masked]
  return keys


class _Counted(object):
  """A mask as sparse_utils.calculate_sparsity reads it, from a popcount already taken."""

  def __init__(self, ones, size):
    self._ones, self.size = ones, size

  def count_ones(self):
    return self._ones


def summary_dict(rows, layout, cross_loss, global_step, learning_rate, weight_decay, drop_fraction=None):
  """Host-only: the summary dict from the per-parameter rows (float64 [n_params][5], plan order) and the step's host
  values.  drop_fraction None: the key is absent (not a drop/grow optimizer)."""
  rows = np.asarray(rows, dtype=np.float64).reshape(-1, _COLS)
  w2_reg = 0.0
  for r, reg in zip(rows, layout.reg):
    if reg:
      w2_reg += float(r[SUM_W2])
  reg_loss = float(weight_decay) * 0.5 * w2_reg
  out = {
      'global_step': int(global_step),
      'loss': float(cross_loss) + reg_loss,
      'cross_loss': float(cross_loss),
      'reg_loss': reg_loss,
      'learning_rate': float(learning_rate),
  }
  if drop_fraction is not None:
    out['drop_fraction'] = float(drop_fraction)
  out['grad_norm'] = math.sqrt(sum(float(r[SUM_G2]) for r in rows))
  out['var_norm'] = math.sqrt(sum(float(r[SUM_W2]) for r in rows))
  if layout.masked:
    first = rows[layout.masked[0][2]]
    out['fw_nz_weight'] = float(first[NNZ_W])
    out['fw_nz_mask'] = float(first[ONES])
    out['fw_l1_weight'] = float(first[SUM_ABS_W])
    out['global_sparsity'] = float(sparse_utils.calculate_sparsity(
        [_Counted(float(rows[i][ONES]), size) for _, size, i in layout.masked]))
  for scope, size, i in layout.masked:
    # Evaluator.result()'s formula with mask_summaries=True
    out['pruning/%s/mask/sparsity' % scope] = 1.0 - float(rows[i][ONES]) / float(size)
  return out


class TrainSummaries(object):
  """The batched summary reduction over the parameters of a fused inner optimizer (optim.FusedMomentumSGD /
  optim.FusedAdam): the same (param, grad, bitmap, grad_scale) entries as its plan, plus reg_decay =
  weight_decay on evaluate.regularized_kernels(model) and 0 elsewhere.  The launch plan is rebuilt whenever one
  of those buffers changes, the optimizer's own rule.  Owns one device result buffer float64 [n_params][5]."""

  def __init__(self, model, inner):
    from .optim import _FusedInnerOptimizer
    if not isinstance(inner, _FusedInnerOptimizer):
      raise ValueError('training summaries need the fused inner optimizer (optim.FusedMomentumSGD or '
                       'optim.FusedAdam), got %s' % type(inner).__name__)
    self.model, self.inner = model, inner
    self._masked_layers = model.registry.layers()
    self._regularized = evaluate.regularized_kernels(model)
    self._plan, self._key = C.c_void_p(None), None
    self.layout, self.out = None, None

  def __del__(self):
    try:
      self._destroy()
    except Exception:
      pass

  def _destroy(self):
    if self._plan and self._plan.value:
      _cabi.lib().rigl_summary_plan_destroy(self._plan)
      self._plan = C.c_void_p(None)

  @property
  def weight_decay(self):
    return float(self.inner.param_groups[0]['weight_decay'])

  def prepare(self):
    """Builds the plan for the CURRENT gradient buffers (allocates and copies: not under stream capture)."""
    ents = self.inner.plan_params()
    wd = self.weight_decay
    layout = summary_layout([p for p, _, _, _ in ents], self._masked_layers, self._regularized)
    key = tuple((p.data_ptr(), g.data_ptr(), 0 if b is None else b.data_ptr(), p.numel(), s, reg)
                for (p, g, b, s), reg in zip(ents, layout.reg)) + (wd,)
    if key == self._key:
      return
    self._destroy()
    descs = (_cabi.SummaryDesc * len(ents))()
    for d, (p, g, b, s), reg in zip(descs, ents, layout.reg):
      d.param, d.grad, d.mask_bits, d.n = p.data_ptr(), g.data_ptr(), None if b is None else b.data_ptr(), p.numel()
      d.grad_scale, d.reg_decay = s, wd if reg else 0.0
    plan = C.c_void_p(None)
    _cabi.check(_cabi.lib().rigl_summary_plan_create(descs, len(ents), C.byref(plan)), 'rigl_summary_plan_create')
    self._plan, self._key, self.layout = plan, key, layout
    dev = ents[0][0].device
    if self.out is None or self.out.shape[0] != len(ents) or self.out.device != dev:
      self.out = torch.empty((len(ents), _COLS), dtype=torch.float64, device=dev)

  def run(self):
    """Launches the reduction on the current stream into `out` (no synchronisation)."""
    self.prepare()
    _cabi.check(_cabi.lib().rigl_summary_plan_run(self._plan, self.out.data_ptr(), _cabi.stream_ptr()),
                'rigl_summary_plan_run')

  def read(self, cross_loss, global_step, learning_rate, drop_fraction=None):
    """The dict of the last run; `cross_loss` (a 0-d device tensor) comes back in the same copy."""
    flat = torch.cat([self.out.view(-1), cross_loss.detach().double().reshape(1)]).cpu().numpy()
    return summary_dict(flat[:-1], self.layout, flat[-1], global_step, learning_rate, self.weight_decay,
                        drop_fraction)
