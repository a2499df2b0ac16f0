"""NumPy restatement of gradual magnitude pruning (contrib model_pruning, TF 1.14/1.15 semantics, DESIGN.md 5):
the sparsity schedule, the update decision and the per-layer threshold / mask update, written independently of
rigl_b200.pruning and ranking by a full np.sort.  No CUDA."""
import re

import numpy as np

f32 = np.float32


def sparsity(gs, initial, target, begin, end, exponent):
  p = f32(gs - begin) / f32(end - begin)
  p = f32(min(1.0, max(0.0, float(p))))
  decay = f32(float(f32(1) - p) ** exponent)
  return f32(f32(initial - target) * decay + f32(target))


def layer_sparsity(s, weight_name, weight_sparsity_map, target):
  hits = [float(e.rpartition(':')[2]) for e in weight_sparsity_map
          if e and re.search(e.rpartition(':')[0], weight_name)]
  if len(hits) > 1:
    raise ValueError('multiple matches for %s' % weight_name)
  return s if not hits else f32(s * f32(hits[0] / target))


def update_steps(steps, begin, end, frequency):
  """Global steps (as read after the increment) on which an update runs."""
  last, out = 0, []
  for gs in steps:
    if gs >= begin and (gs <= end or end < 0) and last + frequency <= gs:
      out.append(gs)
      last = gs
  return out


def keep(n, s):
  k = int(np.rint(f32(f32(n) * f32(f32(1) - f32(s)))))
  return min(max(k, 1), n)


def prune_layer(w, s, old_thr, decay):
  """-> (mask bool[n], thr float32) for flat float32 weights w at layer sparsity s."""
  a = np.abs(np.asarray(w, np.float32).reshape(-1))
  a = np.where(a == 0, f32(0), a)                  # -0.0 counts as 0
  k = keep(a.size, s)
  cur = np.sort(a)[::-1][k - 1]
  thr = f32(f32(cur * f32(f32(1) - f32(decay))) + f32(f32(old_thr) * f32(decay)))
  return a >= thr, thr
