"""Checkpoints with the reference's partial-restore semantics.

The reference trains from TF checkpoints and supports loading only a subset of variables from a
previous run -- masks only (lottery-ticket / "scratch" experiments) or parameters only --
selected by NAME SUFFIX (`utils.initialize_parameters_from_ckpt`,
rigl/imagenet_resnet/utils.py:93-125; flags `--initial_value_checkpoint`, `--load_mask_dir` of
imagenet_train_eval.py).  Variable names follow the reference's scopes: `<scope>/mask`,
`<scope>/weights`, optimizer slots `<scope>/weights/<slot>`, everything else by module path.

Format: one `.npz` per step (`model.ckpt-<step>.npz`), float32 arrays in the reference layouts (masks
as 0/1 float32, HWIO / [in,out] weights) + `global_step`.  Host-side only; the arrays are staged
through numpy.
"""
import collections
import glob
import os
import re

import numpy as np


class Handle(object):
  """get() -> ndarray, set(ndarray) for one variable."""

  def __init__(self, get, set_):
    self.get, self.set = get, set_


def _tensor_handle(t):
  def get():
    return t.detach().float().cpu().numpy()

  def set_(a):
    import torch
    with torch.no_grad():
      t.copy_(torch.from_numpy(np.ascontiguousarray(a)).to(t.device).to(t.dtype).reshape(t.shape))
  return Handle(get, set_)


def _scalar_handle(get, set_):
  return Handle(lambda: np.asarray(get(), dtype=np.float64), lambda a: set_(np.asarray(a).reshape(-1)[0]))


def variables_of(model, optimizer=None, sparse_optimizer=None, ckpt_path=None, pruning=None):
  """OrderedDict name -> Handle for a rigl_b200 model: masks, masked weights, the remaining
  parameters / buffers, (optionally) the inner optimizer's per-parameter state tensors and the sparse
  optimizer's own state.

  optimizer: its slots become `<scope>/weights/<slot>`; what its `non_slot_variables()` returns (if it has
    one) keeps its own name, e.g. `beta1_power`, `beta2_power` of optim.FusedAdam.
  sparse_optimizer: adds `last_mask_update_step` -- a non-trainable global variable in the reference
    (sparse_optimizers_base.py:166-171), so it lives in its checkpoints; without it a resumed run would
    re-initialise it to -frequency and fire an off-schedule mask update -- and, for
    SparseMomentumOptimizer, the EMA shadows `<scope>/weights/ExponentialMovingAverage`.
  pruning: a pruning.Pruning; adds every layer's `<scope>/threshold` and `<name>/last_mask_update_step`
    (e.g. `model_pruning/last_mask_update_step`), the variables contrib's Pruning keeps in its checkpoints.
  ckpt_path: a checkpoint about to be restored.  A freshly built torch optimizer has an EMPTY state, so
    its slots (`<scope>/weights/momentum_buffer` ...) would be skipped silently; every slot the file holds
    for a known parameter is materialised (zeros) in `optimizer.state` here so that restore() fills it."""
  import torch
  out = collections.OrderedDict()
  masked = {}
  for l in model.registry.layers():
    out[l.scope + '/mask'] = Handle(l.mask.numpy, l.mask.assign)
    out[l.scope + '/weights'] = _tensor_handle(l.weight)
    masked[id(l.weight)] = l.scope + '/weights'
  for name, p in list(model.named_parameters()) + list(model.named_buffers()):
    if id(p) not in masked:
      out[name.replace('.', '/')] = _tensor_handle(p)
  if optimizer is not None:
    names = {id(p): (masked.get(id(p)) or n.replace('.', '/')) for n, p in model.named_parameters()}
    if ckpt_path is not None:
      by_name = {v: p for p in (q for g in optimizer.param_groups for q in g['params'])
                 for v in [names.get(id(p))] if v is not None}
      with np.load(ckpt_path) as z:
        for key in z.files:
          base, _, slot = key.rpartition('/')
          p = by_name.get(base)
          if p is not None and key not in out and z[key].size == p.numel() and slot not in optimizer.state[p]:
            optimizer.state[p][slot] = torch.zeros_like(p)
    for p, st in optimizer.state.items():
      for k, v in st.items():
        if hasattr(v, 'shape') and tuple(v.shape) == tuple(p.shape):
          out['%s/%s' % (names.get(id(p), 'param%d' % id(p)), k)] = _tensor_handle(v)
    # optimizer variables that belong to no parameter (optim.FusedAdam's beta1_power / beta2_power), under
    # TF's names; restored in place, so a captured step keeps reading them
    non_slot = getattr(optimizer, 'non_slot_variables', None)
    if non_slot is not None:
      for name, v in non_slot().items():
        out[name] = _tensor_handle(v)
  if sparse_optimizer is not None:
    so = sparse_optimizer
    out['last_mask_update_step'] = _scalar_handle(
        so._last_update_value, lambda v: setattr(so, '_last_update_step', int(v)))
    if hasattr(so, '_ema'):
      for l in model.registry.layers():
        name = l.weight.name
        if name not in so._ema:
          so._ema[name] = torch.zeros(l.weight.numel(), dtype=torch.float32, device=l.weight.device)
        out[l.scope + '/weights/ExponentialMovingAverage'] = _tensor_handle(so._ema[name])
  if pruning is not None:
    for l in model.registry.layers():
      out[l.scope + '/threshold'] = _tensor_handle(l.threshold)
    out[pruning.spec.name + '/last_mask_update_step'] = _scalar_handle(
        lambda: pruning.last_update_step, lambda v: setattr(pruning, 'last_update_step', int(v)))
  return out


def save(model_dir, variables, global_step):
  """Writes model.ckpt-<step>.npz; returns its path."""
  os.makedirs(model_dir, exist_ok=True)
  path = os.path.join(model_dir, 'model.ckpt-%d.npz' % int(global_step))
  arrays = {k: (lambda a: a if a.dtype == np.float64 else a.astype(np.float32))(np.asarray(h.get()))
            for k, h in variables.items()}
  arrays['global_step'] = np.asarray(int(global_step), dtype=np.int64)
  tmp = path + '.tmp.npz'
  np.savez(tmp, **arrays)
  os.replace(tmp, path)
  return path


def latest_checkpoint(model_dir):
  """Path of the checkpoint with the highest step in `model_dir`, or None (tf.train.latest_checkpoint)."""
  if not model_dir or not os.path.isdir(model_dir):
    return None
  best, best_step = None, -1
  for p in glob.glob(os.path.join(model_dir, 'model.ckpt-*.npz')):
    m = re.search(r'model\.ckpt-(\d+)\.npz$', p)
    if m and int(m.group(1)) > best_step:
      best, best_step = p, int(m.group(1))
  return best


def restore(path, variables, strict=True):
  """Full restore; returns the stored global step.  strict: every variable must be present with
  the right number of elements."""
  with np.load(path) as z:
    if strict:
      # optimizer slots / EMA shadows the file holds for a known variable but the caller has no handle for
      # (a freshly built optimizer's state is empty): refuse to drop them silently
      orphans = [k for k in z.files if k not in variables and k.rpartition('/')[0] in variables
                 and k.rpartition('/')[0].endswith('weights')]
      if orphans:
        raise KeyError('checkpoint %s holds %d optimizer-slot variables with no handle (e.g. %s): build the '
                       'variables with variables_of(..., ckpt_path=path)' % (path, len(orphans), orphans[0]))
    for k, h in variables.items():
      if k not in z.files:
        if strict:
          raise KeyError('variable %s not in checkpoint %s' % (k, path))
        continue
      a = z[k]
      if strict and a.size != np.asarray(h.get()).size:
        raise ValueError('variable %s: checkpoint has %d elements, model %d' % (k, a.size, np.asarray(h.get()).size))
      h.set(a)
    return int(z['global_step']) if 'global_step' in z.files else 0


def initialize_parameters_from_ckpt(ckpt_path, model_dir, param_suffixes, variables, log=None):
  """utils.py:93-125: load from `ckpt_path` ONLY the variables whose name ends with one of
  `param_suffixes` (str or tuple, e.g. 'mask' or ('weights', 'gamma')), and only if training has
  not already started in `model_dir`.  Variables with a matching suffix that the checkpoint lacks
  are skipped (logged).  Returns the list of loaded names."""
  log = log or (lambda *a: None)
  if latest_checkpoint(model_dir) is not None:
    log('Training already started on this model, not loading from previously trained model')
    return []
  suffixes = (param_suffixes,) if isinstance(param_suffixes, str) else tuple(param_suffixes)
  loaded = []
  with np.load(ckpt_path) as z:
    present = {n for n in z.files if n.endswith(suffixes)}
    for name, h in variables.items():
      if name in present:
        log('Loading parameter variable from checkpoint: %s' % name)
        h.set(z[name])
        loaded.append(name)
      elif name.endswith(suffixes):
        log('Cannot find parameter variable in checkpoint, skipping: %s' % name)
  return loaded
