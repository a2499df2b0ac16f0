"""numpy restatement of tf.train.AdamOptimizer's update -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

TF 1.x ApplyAdam (training_ops.cc, use_nesterov=false) plus the l2 term the reference adds to the loss, in
float32, one rounding per operation and in the kernel's order (csrc/sgd.cu), so the two agree bit for bit.
TensorFlow is not installable here, so the parity with TF itself is unpinned, like the other TF primitives the
oracle restates from their documentation.
"""
import numpy as np

F32 = np.float32


def adam_step(w, m, v, g, lr, beta1, beta2, eps, beta1_power, beta2_power):
  """One step on one tensor; `g` is the gradient the optimizer sees (mask * dense_grad * scale + wd * w).
  Returns (w, m, v); the caller advances the powers (beta1_power * beta1, beta2_power * beta2 in float32)."""
  w, m, v, g = (np.asarray(a, F32) for a in (w, m, v, g))
  one = F32(1)
  alpha = F32(F32(F32(lr) * np.sqrt(one - F32(beta2_power))) / F32(one - F32(beta1_power)))
  m = (m + (g - m) * F32(one - F32(beta1))).astype(F32)
  v = (v + (g * g - v) * F32(one - F32(beta2))).astype(F32)
  with np.errstate(invalid='ignore'):            # v < 0 (a RigL slot reset with initial_acc_scale > 0): NaN, as TF
    w = (w - (m * alpha) / (np.sqrt(v) + F32(eps))).astype(F32)
  return w, m, v


def optimizer_grad(w, grad, bits=None, grad_scale=1.0, weight_decay=0.0):
  """g = (bit ? grad * grad_scale : 0) + weight_decay * w, float32, as the fused kernels form it."""
  w, grad = np.asarray(w, F32), np.asarray(grad, F32)
  gs = grad * F32(grad_scale)
  if bits is not None:
    gs = np.where(np.asarray(bits, bool), gs, F32(0))
  return (gs + F32(weight_decay) * w).astype(F32)


def advance_powers(beta1_power, beta2_power, beta1, beta2):
  return F32(F32(beta1_power) * F32(beta1)), F32(F32(beta2_power) * F32(beta2))
