"""CPU oracle for the RigL hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

This module restates, in plain numpy, the algorithm of google-research/rigl for
the path this repository accelerates.  Only `tests/`, `__graft_entry__.smoke()`
and `bench.py`'s cpu_baseline / `--impl reference` legs may import it; the
product package `rigl_b200` never does (see tests/test_no_oracle_in_product.py).

Parity pinning status (see DESIGN.md "Oracle"):
  * mask utilities (get_n_zeros, get_mask_random_numpy, ERK / uniform
    sparsities): PINNED -- checked bit-for-bit against the reference's own
    `rigl/sparse_utils.py` imported in the build container (generator:
    tools/make_golden.py, fixtures: tests/golden/sparse_utils_golden.json) and
    against the known-answer counts in rigl/sparse_utils_test.py:47-55.
  * schedule / step semantics: PINNED against the explicit vectors in
    rigl/sparse_optimizers_test.py:85,108,349-352.
  * drop/grow mask update (`get_update_op`, `rigl_mask_update`, grow tensors, slot reset): restates
    rigl/sparse_optimizers_base.py:276-353,523-564 with TF `top_k` == stable descending argsort.
    PINNED TO THE REFERENCE'S CODE, TF PRIMITIVES STUBBED: tools/make_golden_update_op.py imports
    the reference module unmodified and EXECUTES its `_get_update_op` / `generic_mask_update` /
    `reset_momentum` / `get_grow_tensor` over a numpy-backed stand-in for the ~20 TF ops they call;
    tests/test_update_op_golden.py checks masks, weights and slots bit-for-bit on 13 cases (ties,
    reinit, grad_scale / grad_sign grow, accumulator scale, conv shapes).  What remains unpinned is
    only the behaviour of the TF primitives themselves (top_k tie order, float->int cast), taken
    from their documentation; TensorFlow is not installable here.  Additional cross-check: the
    independent TF2 statement rigl/rigl_tf2/mask_updaters.py:99-154 (`tf2_generic_mask_update`).
  * masked conv / linear numerics: third-party (tf.contrib.model_pruning,
    un-vendored); restated as y = op(x, mask*w).  "parity unpinned".

All citations are file:line into /root/reference (google-research/rigl @ d39fc7d).
"""
from __future__ import annotations

import math
import re

import numpy as np

F32 = np.float32


# --------------------------------------------------------------------------
# rigl/sparse_utils.py
# --------------------------------------------------------------------------
def mask_extract_name_fn(mask_name):
  """sparse_utils.py:31-32."""
  return re.findall('(.+)/mask:0', mask_name)[0]


def get_n_zeros(size, sparsity):
  """sparse_utils.py:35-36 -- float64 multiply, floor, python int."""
  return int(np.floor(sparsity * size))


def get_mask_random_numpy(mask_shape, sparsity, random_state=None):
  """sparse_utils.py:48-68 -- float64 ones, first n_zeros zeroed, one shuffle."""
  flat = np.ones(mask_shape).flatten()
  flat[:get_n_zeros(flat.size, sparsity)] = 0
  (random_state if random_state else np.random).shuffle(flat)
  return flat.reshape(mask_shape)


def calculate_sparsity(masks):
  """sparse_utils.py:39-45 -- float32 accumulation of sizes and sums."""
  dense = F32(0.)
  sparse = F32(0.)
  for m in masks:
    dense = F32(dense + F32(m.size))
    sparse = F32(sparse + F32(np.sum(m.astype(F32), dtype=F32)))
  return F32(1.) - sparse / dense


class FakeMask(object):
  """Stands in for a TF mask variable: `.name` ('<scope>/mask:0') and `.shape`."""

  def __init__(self, name, shape):
    self.name = name
    self.shape = tuple(int(s) for s in shape)


def get_sparsities_erdos_renyi(all_masks, default_sparsity, custom_sparsity_map,
                               include_kernel, extract_name_fn=mask_extract_name_fn,
                               erk_power_scale=1.0):
  """sparse_utils.py:90-207.  Same float64 operation order as the reference."""
  dense_layers = set()
  while True:
    divisor = 0
    rhs = 0
    raw = {}
    for mask in all_masks:
      var_name = extract_name_fn(mask.name)
      shape_list = list(mask.shape)
      n_param = np.prod(shape_list)
      n_zeros = get_n_zeros(n_param, default_sparsity)
      if var_name in dense_layers:
        rhs -= n_zeros                                   # :152-154
      elif var_name in custom_sparsity_map:
        pass                                             # :155-157
      else:
        rhs += n_param - n_zeros                         # :161-162
        if include_kernel:
          raw[mask.name] = (np.sum(shape_list) / np.prod(shape_list)) ** erk_power_scale
        else:
          n_in, n_out = shape_list[-2:]
          raw[mask.name] = (n_in + n_out) / (n_in * n_out)
        divisor += raw[mask.name] * n_param              # :172
    eps = rhs / divisor                                  # :175
    max_prob = np.max(list(raw.values()))
    if max_prob * eps > 1:                               # :179-186
      for mask_name, p in raw.items():
        if p == max_prob:
          dense_layers.add(extract_name_fn(mask_name))
    else:
      break
  sparsities = {}
  for mask in all_masks:
    var_name = extract_name_fn(mask.name)
    if var_name in custom_sparsity_map:
      sparsities[mask.name] = custom_sparsity_map[var_name]
    elif var_name in dense_layers:
      sparsities[mask.name] = 0.
    else:
      sparsities[mask.name] = 1. - eps * raw[mask.name]
  return sparsities


def get_sparsities_uniform(all_masks, default_sparsity, custom_sparsity_map,
                           extract_name_fn=mask_extract_name_fn):
  """sparse_utils.py:210-235."""
  out = {}
  for mask in all_masks:
    var_name = extract_name_fn(mask.name)
    out[mask.name] = custom_sparsity_map.get(var_name, default_sparsity)
  return out


def get_sparsities(all_masks, method, default_sparsity, custom_sparsity_map,
                   extract_name_fn=mask_extract_name_fn, erk_power_scale=1.0):
  """sparse_utils.py:258-316 (the 'str' table is data, not algorithm; omitted)."""
  found = set(extract_name_fn(m.name) for m in all_masks
              if extract_name_fn(m.name) in custom_sparsity_map)
  given = set(custom_sparsity_map.keys())
  if found != given:
    raise ValueError('No masks are found for the following names: %s' % str(given - found))
  if method in ('erdos_renyi', 'erdos_renyi_kernel'):
    return get_sparsities_erdos_renyi(
        all_masks, default_sparsity, custom_sparsity_map,
        include_kernel=(method == 'erdos_renyi_kernel'),
        extract_name_fn=extract_name_fn, erk_power_scale=erk_power_scale)
  if method == 'random':
    return get_sparsities_uniform(all_masks, default_sparsity, custom_sparsity_map,
                                  extract_name_fn=extract_name_fn)
  raise ValueError('Method: %s is not valid mask initialization method' % method)


# --------------------------------------------------------------------------
# rigl/sparse_optimizers_base.py -- schedule
# --------------------------------------------------------------------------
def extract_number(token):
  """base.py:45-59."""
  m = re.compile(r'.*_(\d*\.?\d*)$').search(token)
  return float(m.group(1)) if m else 1.


def is_mask_update_iter(global_step, last_update_step, begin_step, end_step, frequency):
  """base.py:198-230 (integer comparisons)."""
  in_range = (global_step >= begin_step) and (global_step <= end_step or end_step < 0)
  return bool(in_range and (last_update_step + frequency <= global_step))


def get_drop_fraction(anneal, initial_value, global_step, begin_step, end_step,
                      is_update_iter):
  """base.py:232-258.  Returns np.float32.

  Canonical float32 evaluation (TF's Eigen cosf/powf are not available here and
  are not bit-portable): every elementary op rounds to float32; cos and pow are
  evaluated in float64 on the float32-rounded argument and rounded once.
  cosine: tf.train.cosine_decay(lr, gs, decay_steps=end-begin) with the RAW
  global_step (base.py:237-242); alpha=0.
  """
  init = F32(float(initial_value))
  if anneal == 'constant':
    frac = init
  elif anneal == 'cosine':
    decay_steps = F32(end_step - begin_step)
    gs = F32(min(F32(global_step), decay_steps))
    completed = F32(gs / decay_steps)
    arg = F32(F32(math.pi) * completed)
    cos_v = F32(math.cos(float(arg)))
    cosine_decayed = F32(F32(0.5) * F32(F32(1.0) + cos_v))
    frac = F32(init * cosine_decayed)
  elif anneal.startswith('exponential'):
    exponent = extract_number(anneal)
    power = F32(F32(global_step - begin_step) / F32(end_step - begin_step))
    base = F32(F32(1.0) - power)
    frac = F32(init * F32(math.pow(float(base), float(F32(exponent)))))
  else:
    raise ValueError('drop_fraction_anneal: %s is not valid' % anneal)
  return frac if is_update_iter else F32(0.)


class ScheduleSim(object):
  """Step/skip semantics of RigL (base.py:487-521) and SET (base.py:118-146).

  `step()` returns (did_mask_update, did_optimizer_step).
  """

  def __init__(self, kind, begin_step, end_step, frequency):
    self.kind, self.begin, self.end, self.freq = kind, begin_step, end_step, frequency
    self.global_step = 0
    self.last_update = -frequency                        # base.py:164-171

  def step(self):
    if self.kind == 'rigl':
      if is_mask_update_iter(self.global_step, self.last_update, self.begin, self.end, self.freq):
        self.last_update = self.global_step
        return True, False                               # no optimizer step, gs frozen
      self.global_step += 1
      return False, True
    # SET: optimizer first (gs += 1), cond evaluated on the incremented gs.
    self.global_step += 1
    if is_mask_update_iter(self.global_step, self.last_update, self.begin, self.end, self.freq):
      self.last_update = self.global_step
      return True, True
    return False, True


# --------------------------------------------------------------------------
# rigl/sparse_optimizers_base.py -- the mask update
# --------------------------------------------------------------------------
def _top_k_indices_all(x):
  """nn_ops.top_k(x, k=n_total).indices: descending, ties -> lower index first."""
  return np.argsort(-x.astype(F32), kind='stable')


def n_prune_keep(mask, drop_fraction):
  """base.py:284-290: float32 sum, float32 multiply, truncation."""
  n_ones = int(np.int32(np.sum(mask.astype(F32).ravel(), dtype=np.float64)))
  n_prune = int(np.int32(F32(F32(n_ones) * F32(drop_fraction))))
  return n_ones, n_prune, n_ones - n_prune


def get_update_op(score_drop, score_grow, mask, weights, drop_fraction,
                  grow_tensor=None, reinit_when_same=False, slots=(), slot_reset=None):
  """base.py:276-343.  All arrays share `mask.shape`; flat index = C order.

  Returns dict(mask, weights, slots, mask1, mask2, new_connections, n_prune, n_keep).
  `slot_reset`: None -> zeros (SET, base.py:345-353) or an array (RigL:
  grad * initial_acc_scale, base.py:555-564).
  """
  shape = mask.shape
  mask_f = mask.astype(F32).ravel()
  n_total = mask_f.size
  _, n_prune, n_keep = n_prune_keep(mask_f, drop_fraction)

  order = _top_k_indices_all(score_drop.astype(F32).ravel())         # :293-294
  mask1 = np.zeros(n_total, F32)
  mask1[order[:n_keep]] = 1                                          # :297-302

  sg = score_grow.astype(F32).ravel()
  lifted = np.where(mask1 == 1, F32(F32(sg.min()) - F32(1)), sg)     # :307-310
  order2 = _top_k_indices_all(lifted)                                # :311
  mask2 = np.zeros(n_total, F32)
  mask2[order2[:n_prune]] = 1                                        # :313-318
  assert float(np.sum(mask1 * mask2)) == 0., 'masks not disjoint (base.py:320-321)'

  if reinit_when_same:
    new_conn = mask2 == 1                                            # :328-330
  else:
    new_conn = (mask2 == 1) & (mask_f == 0)                          # :332-333
  w = weights.astype(F32).ravel().copy()
  grow = np.zeros(n_total, F32) if grow_tensor is None else grow_tensor.astype(F32).ravel()
  w = np.where(new_conn, grow, w)                                    # :334-335
  new_slots = []
  for s in slots:                                                    # :345-353 / :555-564
    sv = s.astype(F32).ravel()
    rv = np.zeros(n_total, F32) if slot_reset is None else slot_reset.astype(F32).ravel()
    new_slots.append(np.where(new_conn, rv, sv).reshape(shape))
  return dict(mask=(mask1 + mask2).reshape(shape), weights=w.reshape(shape),
              slots=new_slots, mask1=mask1.reshape(shape), mask2=mask2.reshape(shape),
              new_connections=new_conn.reshape(shape), n_prune=n_prune, n_keep=n_keep)


def rigl_scores(mask, weights, dense_grad, noise=None):
  """base.py:523-538: score_drop = |float(mask)*w| + noise; score_grow = |dense grad|."""
  sd = np.abs(mask.astype(F32) * weights.astype(F32))
  if noise is not None:
    sd = (sd + noise.astype(F32)).astype(F32)
  return sd.astype(F32), np.abs(dense_grad.astype(F32))


def rigl_grow_tensor(method, weights, dense_grad):
  """base.py:540-553 (+ 'zeros' of :372-373).  random_* need an RNG stream the
  reference seeds with a per-process salted hash (base.py:270,388,397) and are
  supplied by the caller as explicit tensors instead."""
  if not isinstance(method, str):
    raise ValueError('Grow-Init: %s is not a string' % method)
  if method == 'zeros':
    return np.zeros_like(weights, dtype=F32)
  if method.startswith('grad_scale'):
    return (dense_grad.astype(F32) / F32(extract_number(method))).astype(F32)
  if method.startswith('grad_sign'):
    return (np.sign(dense_grad.astype(F32)) / F32(extract_number(method))).astype(F32)
  raise ValueError('Grow-Init: %s is not a valid option.' % method)


def rigl_mask_update(mask, weights, dense_grad, drop_fraction, noise=None,
                     grow_init='zeros', initial_acc_scale=0., slots=()):
  """generic_mask_update + _get_update_op for SparseRigLOptimizer."""
  sd, sg = rigl_scores(mask, weights, dense_grad, noise)
  grow = rigl_grow_tensor(grow_init, weights, dense_grad)
  reset = (dense_grad.astype(F32) * F32(initial_acc_scale)).astype(F32)
  return get_update_op(sd, sg, mask, weights, drop_fraction, grow_tensor=grow,
                       slots=slots, slot_reset=reset)


def set_mask_update(mask, weights, random_grow_scores, drop_fraction, noise=None, slots=()):
  """SET: base.py:260-274 -- grow score is a uniform draw supplied by the caller."""
  sd = np.abs(mask.astype(F32) * weights.astype(F32))
  if noise is not None:
    sd = (sd + noise.astype(F32)).astype(F32)
  return get_update_op(sd, random_grow_scores, mask, weights, drop_fraction, slots=slots)


# --------------------------------------------------------------------------
# rigl/sparse_optimizers.py -- the remaining optimizers on the same select primitive
# (SURVEY 8(f) row 2: the oracle of the GPU product path for them)
# --------------------------------------------------------------------------
def momentum_ema_update(ema, masked_grad, momentum):
  """SparseMomentumOptimizer._before_apply_gradients (sparse_optimizers.py:172,195-197):
  tf.train.ExponentialMovingAverage(decay=momentum).apply on a Tensor: the shadow starts at zero (no
  zero-debias: the constructor default) and is updated by moving_averages.assign_moving_average,
  shadow -= (shadow - value) * (1 - decay), in float32; `average()` returns that shadow.  The
  reference's own test pins this trajectory (sparse_optimizers_test.py:276-295)."""
  e, g = ema.astype(F32), masked_grad.astype(F32)
  return (e - (e - g) * F32(1.0 - momentum)).astype(F32)


def momentum_mask_update(mask, weights, ema_grad, drop_fraction, noise=None, slots=()):
  """SparseMomentumOptimizer.generic_mask_update (sparse_optimizers.py:199-214): drop by
  |mask*w| (+noise), grow by |EMA of the dense gradient|; new connections zero-initialised."""
  sd = np.abs(mask.astype(F32) * weights.astype(F32))
  if noise is not None:
    sd = (sd + noise.astype(F32)).astype(F32)
  return get_update_op(sd, np.abs(ema_grad.astype(F32)), mask, weights, drop_fraction, slots=slots)


def top_k_keep_mask(score, sparsity):
  """snip_fn / dnw_fn (sparse_optimizers.py:293-315 and 427-452): keep the n_keep =
  n_total - get_n_zeros(n_total, sparsity) highest scores; tf.nn.top_k over the WHOLE flattened
  array, so equal scores keep the lower flat index."""
  flat = score.astype(F32).ravel()
  n_total = flat.size
  n_keep = n_total - get_n_zeros(n_total, sparsity)
  order = _top_k_indices_all(flat)
  mask = np.zeros(n_total, F32)
  mask[order[:n_keep]] = 1
  return mask.reshape(score.shape)


def snip_mask(grad, weights, sparsity):
  """SparseSnipOptimizer.snip_fn: score = |g * w| (sparse_optimizers.py:293)."""
  return top_k_keep_mask(np.abs(grad.astype(F32) * weights.astype(F32)), sparsity)


def dnw_mask(weights, sparsity):
  """SparseDNWOptimizer.dnw_fn: score = |w| of the weights AFTER the optimizer step (:408-431)."""
  return top_k_keep_mask(np.abs(weights.astype(F32)), sparsity)


class SnipSim(object):
  """Control flow of SparseSnipOptimizer.apply_gradients (sparse_optimizers.py:317-337): the first
  call at global_step 0 snips (no weight update, step counter NOT incremented), every later call is a
  plain optimizer step."""

  def __init__(self):
    self.is_snipped = False

  def is_snip_iter(self, global_step):
    return global_step == 0 and not self.is_snipped


def tf2_generic_mask_update(mask, weights, score_drop, score_grow, drop_fraction):
  """Independent second statement: rigl/rigl_tf2/mask_updaters.py:99-154.

  n_prune = int32(float32(n_ones) * drop_fraction); keep top-(n_ones-n_prune) of
  score_drop over ALL positions; grow top-n_prune of score_grow where the lifted
  score of kept positions is min-1.  Same tie rule (tf.math.top_k).  Written from
  that file, used only to cross-check `get_update_op`.
  """
  m = mask.astype(F32).ravel()
  n_total = m.size
  n_ones = int(m.sum(dtype=np.float64))
  n_prune = int(np.int32(F32(F32(n_ones) * F32(drop_fraction))))
  n_keep = n_ones - n_prune
  keep_idx = np.argsort(-score_drop.astype(F32).ravel(), kind='stable')[:n_keep]
  mask1 = np.zeros(n_total, F32)
  mask1[keep_idx] = 1
  sg = score_grow.astype(F32).ravel()
  lifted = np.where(mask1 == 1, F32(sg.min() - F32(1)), sg)
  grow_idx = np.argsort(-lifted, kind='stable')[:n_prune]
  mask2 = np.zeros(n_total, F32)
  mask2[grow_idx] = 1
  new_conn = (mask2 == 1) & (m == 0)
  w = np.where(new_conn, F32(0), weights.astype(F32).ravel())
  return (mask1 + mask2).reshape(mask.shape), w.reshape(mask.shape)


# --------------------------------------------------------------------------
# Masked layers (tf.contrib.model_pruning semantics, SURVEY Appendix C)
# --------------------------------------------------------------------------
def masked_linear_fwd(x, w_io, mask_io, bias=None):
  """y = x @ (mask*w) + b; w is [in, out] (mnist_train_eval.py:116-132)."""
  y = x.astype(np.float64) @ (mask_io.astype(np.float64) * w_io.astype(np.float64))
  if bias is not None:
    y = y + bias.astype(np.float64)
  return y


def masked_linear_bwd(x, w_io, mask_io, dy):
  """Returns (dx, dense dW, masked dW): dL/d(mask*w) is dense, dL/dw = mask*dense."""
  wm = mask_io.astype(np.float64) * w_io.astype(np.float64)
  dx = dy.astype(np.float64) @ wm.T
  dw_dense = x.astype(np.float64).T @ dy.astype(np.float64)
  return dx, dw_dense, dw_dense * mask_io


def tf_same_padding(size, k, stride):
  """TensorFlow 'SAME': (output extent, pad_before, pad_after)."""
  out = -(-size // stride)
  total = max((out - 1) * stride + k - size, 0)
  return out, total // 2, total - total // 2


def conv2d_nhwc_general(x, w_hwio, stride, pad_before, out_hw):
  """float64 NHWC conv with `pad_before` zeros before the image and as many after as the
  requested output size needs (covers TF 'SAME' stride-2 asymmetry)."""
  n, h, w, c = x.shape
  kh, kw, ci, co = w_hwio.shape
  ho, wo = out_hw
  ph = max((ho - 1) * stride + kh - h - pad_before, 0)
  pw = max((wo - 1) * stride + kw - w - pad_before, 0)
  xp = np.zeros((n, h + pad_before + ph, w + pad_before + pw, c), np.float64)
  xp[:, pad_before:pad_before + h, pad_before:pad_before + w, :] = x
  y = np.zeros((n, ho, wo, co), np.float64)
  for i in range(kh):
    for j in range(kw):
      patch = xp[:, i:i + stride * (ho - 1) + 1:stride, j:j + stride * (wo - 1) + 1:stride, :]
      y += patch.reshape(-1, c).dot(w_hwio[i, j].astype(np.float64)).reshape(n, ho, wo, co)
  return y


def conv2d_nhwc_general_bwd(x, w_hwio, dy, stride, pad_before):
  n, h, w, c = x.shape
  kh, kw, ci, co = w_hwio.shape
  ho, wo = dy.shape[1:3]
  ph = max((ho - 1) * stride + kh - h - pad_before, 0)
  pw = max((wo - 1) * stride + kw - w - pad_before, 0)
  xp = np.zeros((n, h + pad_before + ph, w + pad_before + pw, c), np.float64)
  xp[:, pad_before:pad_before + h, pad_before:pad_before + w, :] = x
  dxp = np.zeros_like(xp)
  dw = np.zeros(w_hwio.shape, np.float64)
  dyf = dy.reshape(-1, co).astype(np.float64)
  for i in range(kh):
    for j in range(kw):
      sl = (slice(None), slice(i, i + stride * (ho - 1) + 1, stride),
            slice(j, j + stride * (wo - 1) + 1, stride), slice(None))
      dw[i, j] = xp[sl].reshape(-1, c).T.dot(dyf)
      dxp[sl] += dyf.dot(w_hwio[i, j].astype(np.float64).T).reshape(n, ho, wo, c)
  return dxp[:, pad_before:pad_before + h, pad_before:pad_before + w, :], dw


def conv2d_nhwc_fwd(x, w_hwio, stride, pad):
  """Plain-loop-free float64 NHWC conv, symmetric zero pad `pad`, square stride.

  Equivalent to the reference call conv(x, mask*W) (pruning_layers.py:140-157)
  with conv2d_fixed_padding semantics (resnet_model.py:234-303): explicit pad
  (k-1)//2 then VALID for stride>1, SAME for stride 1 (identical for odd k).
  """
  n, h, w, c = x.shape
  kh, kw, ci, co = w_hwio.shape
  assert ci == c
  xp = np.zeros((n, h + 2 * pad, w + 2 * pad, c), np.float64)
  xp[:, pad:pad + h, pad:pad + w, :] = x
  ho = (h + 2 * pad - kh) // stride + 1
  wo = (w + 2 * pad - kw) // stride + 1
  y = np.zeros((n, ho, wo, co), np.float64)
  for i in range(kh):
    for j in range(kw):
      patch = xp[:, i:i + stride * (ho - 1) + 1:stride, j:j + stride * (wo - 1) + 1:stride, :]
      y += patch.reshape(-1, c) .dot(w_hwio[i, j].astype(np.float64)).reshape(n, ho, wo, co)
  return y


def conv2d_nhwc_bwd(x, w_hwio, dy, stride, pad):
  """Returns (dx, dW dense) for conv2d_nhwc_fwd, float64."""
  n, h, w, c = x.shape
  kh, kw, ci, co = w_hwio.shape
  ho, wo = dy.shape[1:3]
  xp = np.zeros((n, h + 2 * pad, w + 2 * pad, c), np.float64)
  xp[:, pad:pad + h, pad:pad + w, :] = x
  dxp = np.zeros_like(xp)
  dw = np.zeros(w_hwio.shape, np.float64)
  dyf = dy.reshape(-1, co).astype(np.float64)
  for i in range(kh):
    for j in range(kw):
      sl = (slice(None), slice(i, i + stride * (ho - 1) + 1, stride),
            slice(j, j + stride * (wo - 1) + 1, stride), slice(None))
      dw[i, j] = xp[sl].reshape(-1, c).T.dot(dyf)
      dxp[sl] += dyf.dot(w_hwio[i, j].astype(np.float64).T).reshape(n, ho, wo, c)
  return dxp[:, pad:pad + h, pad:pad + w, :], dw


# --------------------------------------------------------------------------
# Optimizer arithmetic used by the train-step parity tests (SURVEY Appendix C)
# --------------------------------------------------------------------------
def momentum_step(w, acc, g, lr, momentum, nesterov):
  """tf.train.MomentumOptimizer: acc = m*acc + g; w -= lr*(g + m*acc) | lr*acc."""
  acc = (F32(momentum) * acc.astype(F32) + g.astype(F32)).astype(F32)
  if nesterov:
    w = (w.astype(F32) - F32(lr) * (g.astype(F32) + F32(momentum) * acc)).astype(F32)
  else:
    w = (w.astype(F32) - F32(lr) * acc).astype(F32)
  return w, acc


# --------------------------------------------------------------------------
# Workload tables (SURVEY Appendix A/B; derived from resnet_model.py:396-731)
# --------------------------------------------------------------------------
def resnet50_masked_layers():
  """(scope, HWIO shape, stride, out_hw) in pruning.get_masks() creation order."""
  layers = [('resnet_model/initial_conv', (7, 7, 3, 64), 2, 112)]
  cfg = [(1, 64, 3, 1, 56), (2, 128, 4, 2, 28), (3, 256, 6, 2, 14), (4, 512, 3, 2, 7)]
  cin = 64
  for g, f, blocks, stride, out_hw in cfg:
    in_hw = out_hw * stride
    sfx = 'block_group_projection_block_group%d' % g
    layers.append(('resnet_model/bottleneck_projection_' + sfx, (1, 1, cin, 4 * f), stride, out_hw))
    layers.append(('resnet_model/bottleneck_1_' + sfx, (1, 1, cin, f), 1, in_hw))
    layers.append(('resnet_model/bottleneck_2_' + sfx, (3, 3, f, f), stride, out_hw))
    layers.append(('resnet_model/bottleneck_3_' + sfx, (1, 1, f, 4 * f), 1, out_hw))
    cin = 4 * f
    for b in range(1, blocks):
      sfx = 'block_group%d_%d_1' % (g, b)
      layers.append(('resnet_model/bottleneck_1_' + sfx, (1, 1, cin, f), 1, out_hw))
      layers.append(('resnet_model/bottleneck_2_' + sfx, (3, 3, f, f), 1, out_hw))
      layers.append(('resnet_model/bottleneck_3_' + sfx, (1, 1, f, 4 * f), 1, out_hw))
  layers.append(('resnet_model/final_dense', (2048, 1000), 1, 1))
  return layers
