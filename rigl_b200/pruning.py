"""Stand-in for `tensorflow.contrib.model_pruning.python.pruning`.

The registry of masked layers replaces the graph collections the reference reads through
`pruning.get_masks() / get_weights() / get_masked_weights()` (rigl/sparse_optimizers.py:46-56; collection names
visible at rigl/mnist/mnist_train_eval.py:236).  Entries are returned in creation order.

`get_pruning_hparams()` and `Pruning` are gradual magnitude pruning (Zhu & Gupta), the `prune` training method of
cifar_resnet/resnet_train_eval.py:249-275 and mnist/mnist_train_eval.py:320-335, with contrib's TF 1.14/1.15
semantics (DESIGN.md 5).  The host computes the sparsity schedule and every layer's k; one batched launch sequence
(`rigl_mask_prune_run`) then updates every layer's threshold and mask.
"""
import re

import numpy as np


class MaskedLayerRegistry(object):

  def __init__(self):
    self._layers = []

  def register(self, layer):
    if layer not in self._layers:
      self._layers.append(layer)

  def clear(self):
    del self._layers[:]

  def layers(self):
    return list(self._layers)

  def get_masks(self):
    return [l.mask for l in self._layers]

  def get_weights(self):
    return [l.weight for l in self._layers]

  def get_masked_weights(self):
    return [l.masked_weights for l in self._layers]

  def get_thresholds(self):
    return [l.threshold for l in self._layers]

  def get_weight_sparsity(self):
    """Fraction of zeros of every mask (contrib's get_weight_sparsity: zero_fraction(mask)), float32."""
    return [np.float32(l.mask.sparsity()) for l in self._layers]

  @classmethod
  def from_module(cls, module):
    """Registry holding the masked layers found in `module`, in module order."""
    reg = cls()
    for m in module.modules():
      if getattr(m, 'is_rigl_masked_layer', False):
        reg.register(m)
    return reg


_DEFAULT = MaskedLayerRegistry()


def default_registry():
  return _DEFAULT


def reset_default_registry():
  """Analogue of tf.reset_default_graph() for the mask collections."""
  _DEFAULT.clear()


def get_masks():
  return _DEFAULT.get_masks()


def get_weights():
  return _DEFAULT.get_weights()


def get_masked_weights():
  return _DEFAULT.get_masked_weights()


def get_thresholds():
  return _DEFAULT.get_thresholds()


def get_weight_sparsity():
  return _DEFAULT.get_weight_sparsity()


# one `name=value` token (value: a bracketed list or anything up to the next comma) and its separator
_HPARAM_TOKEN = re.compile(r'\s*(\w+)\s*=\s*(\[[^\]]*\]|[^,\[\]=]*)\s*(?:,|$)')


class HParams(object):
  """The subset of tf.contrib.training.HParams that the drivers use: `parse('k=v,...')`, `set_hparam`, attribute
  access.  Values keep the type of their default; an unknown name raises ValueError."""

  def __init__(self, **defaults):
    object.__setattr__(self, '_values', dict(defaults))

  def __getattr__(self, name):
    values = self.__dict__.get('_values')     # (absent while copy / pickle rebuild the object)
    if values is None or name not in values:
      raise AttributeError(name)
    return values[name]

  def __setattr__(self, name, value):
    self.set_hparam(name, value)

  def values(self):
    return dict(self._values)

  def set_hparam(self, name, value):
    if name not in self._values:
      raise ValueError('Unknown hyperparameter: %s' % name)
    default = self._values[name]
    if isinstance(default, list):
      if not isinstance(value, (list, tuple)):
        raise ValueError('%s takes a list, got %r' % (name, value))
      value = [str(v) for v in value]
    elif isinstance(default, bool):
      if isinstance(value, str):
        if value.lower() not in ('true', 'false', '1', '0'):
          raise ValueError('%s takes a bool, got %r' % (name, value))
        value = value.lower() in ('true', '1')
      value = bool(value)
    elif isinstance(default, int):
      f = float(value)
      if f != int(f):
        raise ValueError('%s takes an integer, got %r' % (name, value))
      value = int(f)
    elif isinstance(default, float):
      value = float(value)
    else:
      value = str(value)
    self._values[name] = value

  def parse(self, values):
    """Sets scalars from 'name=value,name=value'; a list value is written '[a,b]'.  Returns self."""
    values = values or ''
    pos = 0
    while pos < len(values):
      m = _HPARAM_TOKEN.match(values, pos)
      if m is None:
        raise ValueError('Malformed hyperparameter string at %r: %r' % (values[pos:], values))
      pos = m.end()
      name, value = m.group(1), m.group(2).strip()
      if value.startswith('['):
        value = [v.strip() for v in value[1:-1].split(',') if v.strip()]
      self.set_hparam(name, value)
    return self

  def __repr__(self):
    return 'HParams(%s)' % ', '.join('%s=%r' % kv for kv in sorted(self._values.items()))


def get_pruning_hparams():
  """contrib's documented defaults.  nbins and use_tpu are accepted and ignored (the threshold is exact, not a
  histogram CDF); block_height / block_width other than 1 are rejected by Pruning (no block pooling)."""
  return HParams(name='model_pruning', begin_pruning_step=0, end_pruning_step=-1, weight_sparsity_map=[''],
                 threshold_decay=0.0, pruning_frequency=10, nbins=256, block_height=1, block_width=1,
                 block_pooling_function='AVG', initial_sparsity=0.0, target_sparsity=0.5,
                 sparsity_function_begin_step=0, sparsity_function_end_step=100, sparsity_function_exponent=3,
                 use_tpu=False)


def schedule_sparsity(spec, gs):
  """Target sparsity at global step gs, float32 at every operation (pow in float64 on the float32 base, rounded
  once)."""
  f = np.float32
  sfb, sfe = int(spec.sparsity_function_begin_step), int(spec.sparsity_function_end_step)
  p = f(f(int(gs) - sfb) / f(sfe - sfb))
  p = min(f(1.0), max(f(0.0), p))
  base = f(f(1.0) - p)
  decay = f(np.float64(base) ** int(spec.sparsity_function_exponent))
  # (initial - target) is one constant: contrib subtracts the two Python floats before it becomes a float32 tensor
  return f(f(float(spec.initial_sparsity) - float(spec.target_sparsity)) * decay + f(spec.target_sparsity))


def keep_count(n, sparsity):
  """k = int32(round_half_even(f32(n) * f32(1 - s))), clamped to [1, n].  The clamp at 1 follows tfmot: contrib
  gathers element k - 1 = -1 of the sorted magnitudes, which is undefined."""
  f = np.float32
  k = int(np.rint(f(f(n) * f(f(1.0) - f(sparsity)))))
  return min(max(k, 1), int(n))


class Pruning(object):
  """contrib's Pruning(spec, global_step): `conditional_mask_update_op()` after every optimizer step (it reads the
  incremented step) updates, every `pruning_frequency` steps inside [begin_pruning_step, end_pruning_step], each
  layer's threshold and mask from the raw weights:

    k   = keep_count(n, layer sparsity);  cur = the k-th largest |w|
    thr = cur * (1 - threshold_decay) + threshold * threshold_decay;  mask = |w| >= thr

  Weights and optimizer slots are not touched, and a mask re-opens where |w| climbs back above the threshold.
  registry: the masked layers (default: the global registry).  Every layer's `threshold` becomes a view of one flat
  device tensor that a single batched run reads and writes."""

  def __init__(self, spec=None, global_step=None, registry=None):
    from .masks import MaskUpdateEngine
    self.spec = spec if spec is not None else get_pruning_hparams()
    sp = self.spec
    if int(sp.block_height) != 1 or int(sp.block_width) != 1:
      raise ValueError('block_height / block_width other than 1 (block pooling) are not supported')
    if int(sp.sparsity_function_end_step) <= int(sp.sparsity_function_begin_step):
      raise ValueError('sparsity_function_end_step must be greater than sparsity_function_begin_step')
    self._weight_sparsity_map = []
    for entry in sp.weight_sparsity_map:
      if entry:
        name, _, value = entry.rpartition(':')
        if float(value) >= 1.0:
          raise ValueError('Weight sparsity can not exceed 1.0')
        self._weight_sparsity_map.append((re.compile(name), float(value)))
    self.global_step = global_step
    self._registry = registry if registry is not None else _DEFAULT
    self.last_update_step = 0
    self._engine = MaskUpdateEngine()
    layers = self._registry.layers()
    self._layer_ratio = [self._ratio_for(l.scope + '/weights') for l in layers]
    self.thresholds = None
    if layers:
      import torch
      self.thresholds = torch.stack([l.threshold.detach().reshape(()).float() for l in layers]).contiguous()
      for i, l in enumerate(layers):
        l.threshold = self.thresholds[i]

  def _ratio_for(self, weight_name):
    hits = [v for rx, v in self._weight_sparsity_map if rx.search(weight_name)]
    if len(hits) > 1:
      raise ValueError('Multiple matches in weight_sparsity_map for weight %s' % weight_name)
    return None if not hits else np.float32(hits[0] / float(self.spec.target_sparsity))

  def _step(self):
    if self.global_step is None:
      from .sparse_optimizers_base import get_or_create_global_step
      return int(get_or_create_global_step())
    return int(self.global_step)

  def sparsity(self, gs=None):
    """The schedule's float32 sparsity at global step gs (default: the current step)."""
    return schedule_sparsity(self.spec, self._step() if gs is None else gs)

  def layer_sparsities(self, gs=None):
    s = self.sparsity(gs)
    return [s if r is None else np.float32(s * r) for r in self._layer_ratio]

  def keep_counts(self, gs=None):
    return [keep_count(l.mask.size, s) for l, s in zip(self._registry.layers(), self.layer_sparsities(gs))]

  def is_update_step(self, gs):
    sp = self.spec
    in_window = gs >= int(sp.begin_pruning_step) and (gs <= int(sp.end_pruning_step) or int(sp.end_pruning_step) < 0)
    return in_window and self.last_update_step + int(sp.pruning_frequency) <= gs

  def mask_update_op(self):
    """Updates every layer's threshold and mask at the current step's sparsity (asynchronous on the current
    stream)."""
    layers = self._registry.layers()
    if not layers:
      return
    from . import _cabi
    specs = []
    for l in layers:
      flat = l.weight.data.view(-1)
      specs.append(dict(mask=l.mask, weights=flat, score_grow=flat,     # (score_grow is not ranked: nothing grows)
                        flags=_cabi.LAYER_DROP_ONLY | _cabi.LAYER_ALL_ACTIVE))
    self._engine.prune(specs, self.keep_counts(), self.thresholds, float(self.spec.threshold_decay))

  def conditional_mask_update_op(self):
    """Runs mask_update_op when the (already incremented) global step is an update step; returns whether it did."""
    gs = self._step()
    if not self.is_update_step(gs):
      return False
    self.mask_update_op()
    self.last_update_step = gs
    return True
