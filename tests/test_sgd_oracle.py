"""sgd_oracle.fma32 against exact rational arithmetic (no GPU): the single-rounding float32 fma the bit-exact test of
the fused momentum step relies on."""
from fractions import Fraction

import numpy as np

import sgd_oracle as so

F32 = np.float32


def _round_f32(v):
  """The float32 nearest to the Fraction v, ties to the even significand: chosen among float32(float(v)) and its two
  neighbours by exact comparison, so no rounding of v is trusted."""
  r = F32(float(v))
  best = None
  for c in (np.nextafter(r, F32(-np.inf)), r, np.nextafter(r, F32(np.inf))):
    if not np.isfinite(c):
      continue
    dist = abs(Fraction(float(c)) - v)
    even = int(np.array(c, F32).view(np.uint32)) & 1 == 0
    key = (dist, not even)
    if best is None or key < best[0]:
      best = (key, c)
  return best[1]


def _exact(a, b, c):
  return np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                   for x, y, z in zip(a, b, c)], F32)


def _bits(x):
  return np.asarray(x, F32).view(np.uint32)


def _halfway_cases():
  """(a, b, c) whose exact a * b + c lies 2^-70 (relative) beside a float32 halfway point, so that the float64 sum
  is the halfway point itself: a * b = +-(2^-24 - 2^-70) * 2^k with a = 1 + 2^-23, b = +-(1 - 2^-23) 2^(k-24), and
  c = (1 + j 2^-23) 2^k, on either side of every significand parity, both signs, at binades from 2^-100 to
  2^100; plus exact ties (a = 1, b = 2^(k-24)), which round to even."""
  a, b, c = [], [], []
  for k in (-100, -60, -1, 0, 1, 20, 100):
    for j in range(8):
      for sb in (1.0, -1.0):
        for sc in (1.0, -1.0):
          a.append(1.0 + 2.0 ** -23)
          b.append(sb * (1.0 - 2.0 ** -23) * 2.0 ** (k - 24))
          c.append(sc * (1.0 + j * 2.0 ** -23) * 2.0 ** k)
          a.append(1.0)
          b.append(sb * 2.0 ** (k - 24))
          c.append(sc * (1.0 + j * 2.0 ** -23) * 2.0 ** k)
  return tuple(np.array(t, F32) for t in (a, b, c))


def test_fma32_on_constructed_halfway_cases():
  a, b, c = _halfway_cases()
  assert np.all(np.isfinite(b)) and np.all(b != 0)          # the constructed operands are float32 values
  got, want = so.fma32(a, b, c), _exact(a, b, c)
  assert np.array_equal(_bits(got), _bits(want))
  # control: rounding the float64 sum once more (ties to even) gets many of them wrong
  naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
  wrong = int((_bits(naive) != _bits(want)).sum())
  assert wrong >= len(a) // 8, wrong


def test_fma32_on_random_operands():
  """Random signs and exponents over the whole float32 range the step meets (subnormals, cancellation, products
  far below the addend), and the operand classes of the step itself (lr, momentum, weight decay)."""
  rng = np.random.RandomState(0)
  n = 4000
  mant = lambda: rng.uniform(1.0, 2.0, n) * rng.choice([-1.0, 1.0], n)
  a = (mant() * 2.0 ** rng.randint(-75, 60, n)).astype(F32)
  b = (mant() * 2.0 ** rng.randint(-75, 60, n)).astype(F32)
  c = (mant() * 2.0 ** rng.randint(-149, 100, n)).astype(F32)
  c[::7] = (-(a[::7].astype(np.float64) * b[::7].astype(np.float64))).astype(F32)     # near-total cancellation
  c[::11] = 0.0
  c[5::13] = -0.0
  step = (rng.choice([0.1, 0.9, 1e-4, 1e-2], n).astype(F32), rng.standard_normal(n).astype(F32),
          (1e-3 * rng.standard_normal(n)).astype(F32))
  for x, y, z in ((a, b, c), step):
    got, want = so.fma32(x, y, z), _exact(x, y, z)
    # the exact rational has no sign: an exact zero sum of a nonzero product and its negation is +0 under round
    # to nearest (IEEE 754 6.3), which _round_f32 also returns
    assert np.array_equal(_bits(got), _bits(want))


def test_sgd_step_signed_zero_and_masked_out_gradient():
  """A masked-out element never reads its gradient (a NaN there stays out), and with weight decay 0 and an empty
  momentum buffer it does not move: fma(0, p, +0) is +0 whatever the sign of p."""
  p = np.array([-1.5, 2.0, -0.0, 3.0], F32)
  m = np.zeros(4, F32)
  g = np.array([np.nan, np.nan, 1.0, 1.0], F32)
  on = np.array([False, False, True, True])
  p1, m1 = so.sgd_step(p, m, g, on, 0.5, 0.0, 0.1, 0.9, True)
  assert np.array_equal(_bits(p1[:2]), _bits(p[:2])) and np.array_equal(_bits(m1[:2]), np.zeros(2, np.uint32))
  assert np.all(np.isfinite(p1))
  # on elements: g_eff = 0.5, m = 0.5, p -= 0.1 * (0.9 * 0.5 + 0.5), each step rounded once
  want = so.fma32(-F32(0.1), so.fma32(F32(0.9), F32(0.5), F32(0.5)), p[2:])
  assert np.array_equal(_bits(p1[2:]), _bits(want))


def test_oracle_distinguishes_the_update_forms():
  """The bit-exact test of the fused step tells its forms apart: on the same inputs the Nesterov and plain updates
  differ (the plain one is the Nesterov one with its inner fma(momentum, m, ge) replaced by m), and so do momentum
  0 and 0.9; at momentum 0 the two forms coincide."""
  rng = np.random.RandomState(3)
  p, m, g = (rng.standard_normal(4096).astype(F32) for _ in range(3))
  out = {(nest, mom): so.sgd_step(p, m, g, None, 0.5, 1e-4, 0.1, mom, nest)[0]
         for nest in (True, False) for mom in (0.0, 0.9)}
  keys = list(out)
  for i in range(len(keys)):
    for j in range(i + 1, len(keys)):
      if keys[i][1] == 0.0 and keys[j][1] == 0.0:
        # momentum 0: fma(0, m, ge) = ge either way, so the two forms coincide
        assert _bits(out[keys[i]]).tobytes() == _bits(out[keys[j]]).tobytes()
        continue
      assert _bits(out[keys[i]]).tobytes() != _bits(out[keys[j]]).tobytes(), (keys[i], keys[j])
