"""Times one gradual-magnitude-pruning update (rigl_mask_prune_run: every layer's threshold and mask) of the
ResNet-50 (54 masked tensors, 25.5 M weights) and WRN-22-2 layer sets, dense masks, target sparsity 0.8, against a
per-layer torch baseline in the same process (torch.kthvalue of |w| and a compare per layer).

  python tools/bench_prune.py [--iters 50] [--warmup 5]

Timing: CUDA events around each update, median over --iters after --warmup, the two paths alternated.  Two
figures per path: `call` starts on an idle device, so it includes the host work of the call (plan lookup, argument
building, launches); `device` enqueues the update behind a 20 ms device sleep, so the events see the kernels only.
Bytes/s: the algorithmic bytes (read every weight once, write the bitmap: 4.125 bytes per weight) over the median
device time."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rigl_b200 import _cabi, pruning  # noqa: E402
from rigl_b200.masks import MaskUpdateEngine, MaskVariable  # noqa: E402

DEV = 'cuda:0'


def shapes(tag):
  with open(os.path.join(os.path.dirname(__file__), '..', 'tests', 'golden', 'sparse_utils_golden.json')) as f:
    return [tuple(sh) for _, sh in [c for c in json.load(f)['cases'] if c['tag'] == tag][0]['layers']]


def gpu_info():
  try:
    return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                                    '--format=csv,noheader'], text=True).strip().splitlines()[0]
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name(0) + ', power limit unknown'


def timed(fn, device_only):
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  if device_only:
    torch.cuda._sleep(40 * 10 ** 6)        # ~20 ms: the host has enqueued everything before `a` is reached
  a.record()
  fn()
  b.record()
  b.synchronize()
  return a.elapsed_time(b)


def bench(tag, sparsity, iters, warmup):
  g = torch.Generator(device=DEV).manual_seed(0)
  specs = []
  for i, sh in enumerate(shapes(tag)):
    n = int(np.prod(sh))
    w = torch.randn(n, device=DEV, generator=g) * 0.05
    specs.append(dict(mask=MaskVariable('l%d' % i, sh, DEV), weights=w, score_grow=w,
                      flags=_cabi.LAYER_DROP_ONLY | _cabi.LAYER_ALL_ACTIVE))
  sizes = [s['mask'].size for s in specs]
  keep = [pruning.keep_count(n, np.float32(sparsity)) for n in sizes]
  thr = torch.zeros(len(specs), device=DEV)
  eng = MaskUpdateEngine()
  ref_masks = [torch.empty(n, dtype=torch.bool, device=DEV) for n in sizes]
  ref_thr = torch.zeros(len(specs), device=DEV)

  def batched():
    eng.prune(specs, keep, thr, 0.0)

  def per_layer():
    for i, (s, k) in enumerate(zip(specs, keep)):
      a = s['weights'].abs()
      cur = torch.kthvalue(a, a.numel() - k + 1).values
      ref_thr[i] = cur
      torch.ge(a, cur, out=ref_masks[i])

  t = {k: [] for k in ('batched_call', 'batched_device', 'torch_call', 'torch_device')}
  for it in range(warmup + iters):
    got = dict(batched_call=timed(batched, False), torch_call=timed(per_layer, False),
               batched_device=timed(batched, True), torch_device=timed(per_layer, True))
    if it >= warmup:
      for k, v in got.items():
        t[k].append(v)
  # same thresholds and masks on both paths
  assert torch.equal(thr, ref_thr)
  for s, m in zip(specs, ref_masks):
    assert torch.equal(s['mask'].to_dense().view(-1) > 0, m)
  total = sum(sizes)
  algo_bytes = 4 * total + total / 8.0
  med = {k: float(np.median(v)) for k, v in t.items()}
  return dict(workload=tag.split('_')[0], layers=len(sizes), weights=total, sparsity=sparsity,
              batched_call_ms=round(med['batched_call'], 4), batched_device_ms=round(med['batched_device'], 4),
              per_layer_torch_call_ms=round(med['torch_call'], 4),
              per_layer_torch_device_ms=round(med['torch_device'], 4),
              speedup_device=round(med['torch_device'] / med['batched_device'], 2),
              batched_device_GBps=round(algo_bytes / (med['batched_device'] * 1e-3) / 1e9, 1),
              algorithmic_bytes=int(algo_bytes), iters=iters)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--sparsity', type=float, default=0.8)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_prune.py needs a GPU')
  print('gpu: %s' % gpu_info())
  for tag in ('r50_erk80', 'wrn22_2_erk95'):
    print(json.dumps(bench(tag, args.sparsity, args.iters, args.warmup)))


if __name__ == '__main__':
  main()
