"""The inner optimizer step on the ResNet-50 parameter set (54 masked tensors at ERK 0.8, 25.5 M weights, plus the
batch-norm and bias parameters), on the same gradients:

  fused_adam      optim.FusedAdam.step -- one launch, mask * dense_grad formed in-kernel, + the powers update
  torch_adam      torch.optim.Adam(fused=True) after one rigl_apply_mask_f32 per masked layer (the non-fused path)
  fused_momentum  optim.FusedMomentumSGD.step -- the default inner optimizer, for scale

  python tools/bench_inner_optimizer.py [--iters 50] [--warmup 10]

Timing: CUDA events around each step, median over --iters after --warmup steps.  Bytes are the least each path
must move (float32 reads and writes, 1 bit per masked weight for the bitmap), divided by the median time and set
beside the H100 SXM data-sheet HBM3 bandwidth.  The card's name and power limit are printed with the result."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rigl_b200 import workloads  # noqa: E402
from rigl_b200.optim import FusedAdam, FusedMomentumSGD  # noqa: E402

HBM_TBS = 3.35


def power_limit():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    return out or 'unknown'
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def time_steps(fn, iters, warmup):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  times = []
  for _ in range(iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    times.append(start.elapsed_time(stop))
  return float(np.median(times)), float(np.min(times)), float(np.max(times))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=10)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_inner_optimizer: needs a CUDA device')
  dev = 'cuda:0'
  torch.manual_seed(0)
  model = workloads.ResNet50(device=dev)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
  layers = model.registry.layers()
  masked_ids = {id(l.weight) for l in layers}
  others = [p for p in model.parameters() if id(p) not in masked_ids]
  gen = torch.Generator(device=dev).manual_seed(1)
  for l in layers:
    l.masked_weights.dense_grad.copy_(torch.randn(l.weight.numel(), device=dev, generator=gen) * 1e-3)
  for p in others:
    p.grad = torch.randn(p.shape, device=dev, generator=gen) * 1e-3
  n_masked = sum(l.weight.numel() for l in layers)
  n_other = sum(p.numel() for p in others)

  fused_adam = FusedAdam(model.parameters(), lr=1e-4, weight_decay=1e-4).attach_masked_layers(layers)
  fused_sgd = FusedMomentumSGD(model.parameters(), lr=1e-4, momentum=0.9, weight_decay=1e-4).attach_masked_layers(layers)
  for l in layers:
    l.weight.grad = torch.empty_like(l.weight)
  torch_adam = torch.optim.Adam(model.parameters(), lr=1e-4, eps=1e-8, weight_decay=1e-4, fused=True)

  def torch_adam_step():
    for l in layers:
      l.mask.apply_to(l.masked_weights.dense_grad, out=l.weight.grad.view(-1))
    torch_adam.step()

  bits = n_masked / 8.0
  rows = [
      # (name, step, bytes): w, m, v, g read + w, m, v written = 28 B per element
      ('fused_adam', fused_adam.step, 28.0 * (n_masked + n_other) + bits),
      # apply-mask: dense grad read + masked grad written (8 B) + bitmap; then the 28 B of Adam
      ('torch_adam', torch_adam_step, 36.0 * n_masked + bits + 28.0 * n_other),
      # w, accum, g read + w, accum written = 20 B per element
      ('fused_momentum', fused_sgd.step, 20.0 * (n_masked + n_other) + bits),
  ]
  gpu = torch.cuda.get_device_name(0)
  result = dict(gpu=gpu, power_limit=power_limit(), masked_weights=n_masked, other_params=n_other,
                hbm_peak_tbs=HBM_TBS, iters=args.iters, warmup=args.warmup, rows=[])
  print('%s, power limit %s; %d masked weights + %d other parameters' % (gpu, result['power_limit'], n_masked,
                                                                        n_other))
  print('%-16s %10s %10s %10s %10s %10s %8s' % ('path', 'ms median', 'ms min', 'ms max', 'GB/step', 'TB/s',
                                                 'of peak'))
  for name, fn, nbytes in rows:
    med, lo, hi = time_steps(fn, args.iters, args.warmup)
    tbs = nbytes / (med * 1e-3) / 1e12
    result['rows'].append(dict(path=name, ms_median=med, ms_min=lo, ms_max=hi, bytes=nbytes, tbs=tbs))
    print('%-16s %10.4f %10.4f %10.4f %10.3f %10.3f %7.1f%%' % (name, med, lo, hi, nbytes / 1e9, tbs,
                                                                100 * tbs / HBM_TBS))
  print(json.dumps(result))


if __name__ == '__main__':
  main()
