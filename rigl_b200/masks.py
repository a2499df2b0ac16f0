"""Device-resident mask variables and the batched mask-update engine.

`MaskVariable` is the PyTorch-side stand-in for the float32 `mask` variable that
tf.contrib.model_pruning's masked layers create (reference call sites
rigl/imagenet_resnet/pruning_layers.py:140-157,223-233): same `.name`
('<scope>/mask:0'), `.shape`, `.dtype`, readable as a 0/1 float tensor and
assignable, but stored as a 1-bit bitmap in HBM.

`MaskUpdateEngine` drives the batched CUDA mask update (csrc/mask_update.cu)
for a fixed list of (mask, weights, score_grow, ...) layers -- the replacement
for the per-layer `_get_update_op` graph of sparse_optimizers_base.py:276-343.
"""
import ctypes as C

import numpy as np
import torch

from . import _cabi


def mask_words(n):
  return int(_cabi.lib().rigl_mask_words(int(n)))


class MaskVariable(object):
  """A binary mask of a weight tensor, flat index = C order of `shape`."""

  def __init__(self, scope, shape, device):
    self.scope = scope
    self.name = scope + '/mask:0'
    self.shape = tuple(int(s) for s in shape)
    self.size = int(np.prod(self.shape))
    self.dtype = torch.float32
    self.device = torch.device(device)
    # all-ones initial mask, like the contrib layers (SURVEY Appendix C)
    self.bits = torch.zeros(mask_words(self.size), dtype=torch.int32, device=self.device)
    self.assign(np.ones(self.shape, np.float32))

  # -- reference-style access -------------------------------------------------
  def assign(self, value):
    """mask <- (value != 0); `value` is array-like / tensor of `shape`."""
    t = torch.as_tensor(np.asarray(value) if not torch.is_tensor(value) else value)
    if tuple(t.shape) != self.shape:
      raise ValueError('mask %s: shape %s != %s' % (self.name, tuple(t.shape), self.shape))
    t = t.to(device=self.device, dtype=torch.float32).contiguous().view(-1)
    _cabi.check(_cabi.lib().rigl_mask_pack_f32(t.data_ptr(), self.size, self.bits.data_ptr(),
                                               _cabi.stream_ptr()), 'rigl_mask_pack_f32')
    return self

  def to_dense(self, out=None):
    """The mask as a float32 0/1 tensor of `shape` (the reference's mask value)."""
    if out is None:
      out = torch.empty(self.size, dtype=torch.float32, device=self.device)
    _cabi.check(_cabi.lib().rigl_mask_unpack_f32(self.bits.data_ptr(), self.size, out.data_ptr(),
                                                 _cabi.stream_ptr()), 'rigl_mask_unpack_f32')
    return out.view(self.shape)

  def numpy(self):
    return self.to_dense().cpu().numpy()

  def count_ones(self):
    cnt = torch.zeros(1, dtype=torch.int32, device=self.device)
    _cabi.check(_cabi.lib().rigl_mask_popcount(self.bits.data_ptr(), self.size, cnt.data_ptr(),
                                               _cabi.stream_ptr()), 'rigl_mask_popcount')
    return int(cnt.item())

  def sparsity(self):
    return 1.0 - self.count_ones() / float(self.size)

  def apply_to(self, src, out=None, scale=1.0):
    """out <- mask * src * scale (float32, flat C order)."""
    src = src.contiguous()
    if out is None:
      out = torch.empty_like(src)
    _cabi.check(_cabi.lib().rigl_apply_mask_f32(src.data_ptr(), self.bits.data_ptr(), self.size,
                                                out.data_ptr(), float(scale), _cabi.stream_ptr()),
                'rigl_apply_mask_f32')
    return out

  def __repr__(self):
    return 'MaskVariable(%s, shape=%s)' % (self.name, self.shape)


def _ptr(t):
  return None if t is None else t.data_ptr()


class MaskUpdateEngine(object):
  """Batched drop/grow for a list of layers.

  Each layer is a dict with tensors (float32, contiguous, same numel):
    weights, score_grow, mask (MaskVariable), and optional noise, slots (list of
    up to 2 tensors), grow_values, score_drop, n_prune (int override), grad (the gradient the
    grad_* grow inits and the slot reset read when it is not score_grow itself), flags
    (_cabi.LAYER_GROW_SCORE_SIGNED: rank score_grow verbatim instead of |score_grow|; LAYER_DROP_ONLY;
    LAYER_ALL_ACTIVE) and noise_key (per-layer key of the in-kernel noise, see `run(noise_std=...)`).
  The C plan captures raw pointers, so it is rebuilt whenever any pointer changes.
  """

  def __init__(self):
    self._plan = C.c_void_p(None)
    self._key = None
    self._ws = None
    self._n_layers = 0

  def __del__(self):
    try:
      self._destroy()
    except Exception:  # interpreter shutdown
      pass

  def _destroy(self):
    if self._plan and self._plan.value:
      _cabi.lib().rigl_mask_plan_destroy(self._plan)
      self._plan = C.c_void_p(None)

  @staticmethod
  def _layer_key(ly):
    slots = list(ly.get('slots') or [])[:2]
    return (ly['weights'].data_ptr(), ly['score_grow'].data_ptr(), ly['mask'].bits.data_ptr(),
            _ptr(ly.get('noise')), tuple(s.data_ptr() for s in slots), _ptr(ly.get('grow_values')),
            _ptr(ly.get('score_drop')), int(ly['mask'].size), int(ly.get('n_prune', -1)),
            _ptr(ly.get('grad')), int(ly.get('flags', 0)), int(ly.get('noise_key', 0)))

  def prepare(self, layers):
    key = tuple(self._layer_key(ly) for ly in layers)
    if key == self._key:
      return
    self._destroy()
    descs = (_cabi.LayerDesc * len(layers))()
    for d, ly in zip(descs, layers):
      n = ly['mask'].size
      for name in ('weights', 'score_grow', 'noise', 'grow_values', 'score_drop', 'grad'):
        t = ly.get(name)
        if t is not None:
          if t.dtype != torch.float32 or not t.is_contiguous() or t.numel() != n or not t.is_cuda:
            raise ValueError('%s of %s must be a contiguous float32 CUDA tensor of %d elements'
                             % (name, ly['mask'].name, n))
      slots = list(ly.get('slots') or [])[:2]        # slots beyond two are reset on the host side (see run)
      d.weights = ly['weights'].data_ptr()
      d.score_grow = ly['score_grow'].data_ptr()
      d.mask_bits = ly['mask'].bits.data_ptr()
      d.noise = _ptr(ly.get('noise'))
      for i, s in enumerate(slots):
        if s.dtype != torch.float32 or not s.is_contiguous() or s.numel() != n:
          raise ValueError('optimizer slot of %s must be contiguous float32' % ly['mask'].name)
        d.slots[i] = s.data_ptr()
      d.grow_values = _ptr(ly.get('grow_values'))
      d.score_drop = _ptr(ly.get('score_drop'))
      d.grad = _ptr(ly.get('grad'))
      d.flags = int(ly.get('flags', 0))
      d.noise_key = int(ly.get('noise_key', 0)) & 0xffffffff
      d.n = n
      d.n_prune_override = int(ly.get('n_prune', -1))
    plan = C.c_void_p(None)
    _cabi.check(_cabi.lib().rigl_mask_plan_create(descs, len(layers), C.byref(plan)),
                'rigl_mask_plan_create')
    self._plan = plan
    self._key = key
    self._n_layers = len(layers)
    need = int(_cabi.lib().rigl_mask_plan_workspace_bytes(plan))
    if self._ws is None or self._ws.numel() < need:
      self._ws = torch.empty(need, dtype=torch.uint8, device=layers[0]['weights'].device)

  def run(self, layers, drop_fraction, grow_mode=_cabi.GROW_ZEROS, grow_divisor=1.0, acc_scale=0.0,
          reinit_when_same=False, plan_key=None, noise_std=0.0, noise_seed=0):
    """One mask update of every layer; asynchronous on the current stream.  plan_key: a caller-side key that
    changes whenever any tensor of `layers` is reallocated; when it equals the key of the previous run the
    per-layer validation / plan lookup is skipped (the host cost then does not scale with the layer count)."""
    if plan_key is None or plan_key != getattr(self, '_caller_key', None) or not (self._plan and self._plan.value):
      self.prepare(layers)
      self._caller_key = plan_key
    # The kernels reset up to two optimizer slots per weight in place (SGD momentum; Adam's two moments).  Further
    # slots (amsgrad's max_exp_avg_sq, LAMB ...) are reset after the update from the bitmaps: new connections =
    # new mask & ~old mask (base.py:332-333, 345-353, 555-564 reset EVERY slot).
    extra = [(ly, list(ly['slots'])[2:], ly['mask'].bits.clone()) for ly in layers if len(ly.get('slots') or []) > 2]
    if extra and reinit_when_same:
      raise ValueError('reinit_when_same with more than 2 optimizer slots per weight is not supported')
    self._launch(drop_fraction, grow_mode, grow_divisor, acc_scale, reinit_when_same, noise_std, noise_seed)
    for ly, slots, old_bits in extra:
      n = ly['mask'].size
      grown_bits = ly['mask'].bits & ~old_bits
      grown = torch.empty(n, dtype=torch.float32, device=grown_bits.device)
      _cabi.check(_cabi.lib().rigl_mask_unpack_f32(grown_bits.data_ptr(), n, grown.data_ptr(), _cabi.stream_ptr()),
                  'rigl_mask_unpack_f32')
      grown = grown > 0
      g = ly.get('grad')
      g = ly['score_grow'] if g is None else g
      value = g * float(acc_scale)        # (always the product: acc_scale = 0 gives the SIGNED zeros the kernels and
      for sl in slots:                    #  the reference's `masked_grad * initial_acc_scale` give)
        flat = sl.view(-1)
        flat.copy_(torch.where(grown, value, flat))

  def _launch(self, drop_fraction, grow_mode, grow_divisor, acc_scale, reinit_when_same, noise_std, noise_seed):
    if noise_std:
      # drop-score noise drawn in-kernel for the layers without a `noise` tensor (keyed by noise_seed and each
      # layer's `noise_key`; rigl_mask_noise_fill reproduces it)
      _cabi.check(_cabi.lib().rigl_mask_update_run_noise(
          self._plan, float(drop_fraction), int(grow_mode), float(grow_divisor), float(acc_scale),
          int(bool(reinit_when_same)), float(noise_std), int(noise_seed) & 0xffffffffffffffff, self._ws.data_ptr(),
          self._ws.numel(), _cabi.stream_ptr()), 'rigl_mask_update_run_noise')
      return
    _cabi.check(_cabi.lib().rigl_mask_update_run(
        self._plan, float(drop_fraction), int(grow_mode), float(grow_divisor), float(acc_scale),
        int(bool(reinit_when_same)), self._ws.data_ptr(), self._ws.numel(), _cabi.stream_ptr()),
                'rigl_mask_update_run')

  def prune(self, layers, keep, thresholds, threshold_decay):
    """Gradual magnitude pruning of every layer (rigl_mask_prune_run): layers as for `run`, each with flags
    LAYER_DROP_ONLY | LAYER_ALL_ACTIVE; keep[l] = the layer's k; thresholds: float32 [n_layers] on the device, read
    as the old thresholds and overwritten with the new ones.  Asynchronous on the current stream."""
    self.prepare(layers)
    if (thresholds.dtype != torch.float32 or not thresholds.is_contiguous() or thresholds.numel() != len(layers)
        or not thresholds.is_cuda):
      raise ValueError('thresholds must be a contiguous float32 CUDA tensor of %d elements' % len(layers))
    k = (C.c_int32 * len(layers))(*[int(v) for v in keep])
    _cabi.check(_cabi.lib().rigl_mask_prune_run(self._plan, k, thresholds.data_ptr(), thresholds.data_ptr(),
                                                float(threshold_decay), self._ws.data_ptr(), self._ws.numel(),
                                                _cabi.stream_ptr()), 'rigl_mask_prune_run')

  def stats(self):
    """[(n_ones, n_prune, n_keep, drop_candidates, grow_candidates, drop_bin, grow_bin)] per layer."""
    out = (C.c_int32 * (8 * self._n_layers))()
    _cabi.check(_cabi.lib().rigl_mask_plan_read_stats(self._plan, self._ws.data_ptr(), out,
                                                      _cabi.stream_ptr()), 'rigl_mask_plan_read_stats')
    return [tuple(out[8 * i:8 * i + 7]) for i in range(self._n_layers)]

  @property
  def workspace_bytes(self):
    return 0 if self._ws is None else self._ws.numel()


def noise_fill(n, noise_key, noise_std, noise_seed, device):
  """The noise tensor `MaskUpdateEngine.run(noise_std=..., noise_seed=...)` adds in-kernel to the drop scores of a
  layer with `noise_key` (float32 [n]); for tests / the oracle -- the product path never materialises it."""
  out = torch.empty(int(n), dtype=torch.float32, device=device)
  _cabi.check(_cabi.lib().rigl_mask_noise_fill(out.data_ptr(), int(n), int(noise_key) & 0xffffffff, float(noise_std),
                                               int(noise_seed) & 0xffffffffffffffff, _cabi.stream_ptr()),
              'rigl_mask_noise_fill')
  return out
