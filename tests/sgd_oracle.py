"""numpy restatement of the fused momentum step -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

csrc/sgd.cu sgd_one, per element, in float32 with three fused multiply-adds (one rounding each):
  ge = fma(wd, p, bit ? f32(g * grad_scale) : 0)
  m  = fma(momentum, m, ge)
  p  = fma(-lr, nesterov ? fma(momentum, m, ge) : m, p)
numpy has no fma and Python 3.12 has no math.fma, so `fma32` forms one: the product of two float32 values is
exact in float64 (48 significant bits), TwoSum gives the exact error of the float64 sum, and the one case where
rounding that sum to float32 is not the rounding of the exact value -- the float64 sum lies exactly halfway
between two float32 values -- is resolved by the sign of that error.  (Every float32 halfway point is a float64
value, so the float64 sum never crosses one; and every quantity here is a multiple of 2^-298, so nothing
underflows in float64.)
"""
import numpy as np

F32, F64 = np.float32, np.float64


def fma32(a, b, c):
  """float32 a * b + c with a single rounding (to nearest, ties to even), elementwise."""
  a, b, c = (np.asarray(t, F32) for t in (a, b, c))
  with np.errstate(invalid='ignore', over='ignore'):
    p = a.astype(F64) * b.astype(F64)              # exact
    cc = c.astype(F64)
    s = p + cc
    bb = s - p                                     # TwoSum: p + cc == s + e exactly
    e = (p - (s - bb)) + (cc - bb)
    r = s.astype(F32)                              # to nearest, ties to even
    d = s - r.astype(F64)                          # exact: s and r are within a factor of two
    o = np.nextafter(r, np.where(d > 0, F32(np.inf), F32(-np.inf)).astype(F32))   # the other neighbour of s
    half = (d != 0) & ((r.astype(F64) + o.astype(F64)) * 0.5 == s)
    # a tie in float64 that is not a tie in exact arithmetic: the error says which neighbour is nearer
    return np.where(half & (e * d > 0), o, r).astype(F32)


def masked_grad(g, on, grad_scale):
  """bit ? f32(g * grad_scale) : 0 (on = None: every bit set)."""
  gs = np.asarray(g, F32) * F32(grad_scale)
  return gs if on is None else np.where(np.asarray(on, bool), gs, F32(0)).astype(F32)


def sgd_step(p, m, g, on, grad_scale, weight_decay, lr, momentum, nesterov):
  """One step of sgd_one on one tensor: returns (p, m)."""
  p, m = np.asarray(p, F32), np.asarray(m, F32)
  mom = F32(momentum)
  ge = fma32(F32(weight_decay), p, masked_grad(g, on, grad_scale))
  m = fma32(mom, m, ge)
  upd = fma32(mom, m, ge) if nesterov else m
  return fma32(-F32(lr), upd, p), m
