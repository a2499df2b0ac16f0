"""Cost of the per-step training summaries (TrainHarness(summaries=True)) on ResNet-50, ERK 0.8, batch 256, 224²,
CUDA-graph replay.

  python tools/bench_summaries.py [--windows 6] [--steps 21] [--frequency 20] [--kernel-iters 50]

One harness, one model and one captured graph are timed in alternating windows in one process: without summaries,
and with the summaries computed and read back every step.  A window is --steps steps; with RigL every
--frequency global steps a step is a mask update (and does not advance the global step), so a window of
frequency + 1 steps holds exactly one mask update.  Step time: host clock around a window that ends in a device
synchronisation, divided by the steps.  Kernel time: CUDA events around --kernel-iters runs of the two summary
launches (rigl_summary_plan_run), set against the bytes they must read (weights and gradients in float32, one bit
per masked weight, the partial rows).  The card's name and power limit are printed with the result."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rigl_b200 import _cabi, workloads  # noqa: E402

HBM_TBS = 3.35


def power_limit():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    return out or 'unknown'
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def build(frequency, images, labels):
  torch.manual_seed(0)
  model = workloads.ResNet50(device='cuda:0')
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
  model.train()
  h = workloads.TrainHarness(model, lr=0.1, weight_decay=1e-4, frequency=frequency, end_step=10 ** 6,
                             summaries=True)
  h.step(images, labels)          # eager: the first step is the initial mask update
  h.step(images, labels)
  if not h.enable_cuda_graph(images, labels):
    raise SystemExit('bench_summaries: CUDA-graph capture failed')
  return h


def window(h, summ, images, labels, steps, on):
  """ms per step over `steps` steps with the summaries computed and read back every step (on) or not at all."""
  h._summaries = summ if on else None      # one model and one captured graph for both legs
  updates = 0
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(steps):
    h.step(images, labels)
    updates += h.opt.last_update_was_mask_update
    if on:
      h.summaries()
  torch.cuda.synchronize()
  ms = (time.perf_counter() - t0) * 1e3 / steps
  h._summaries = summ
  return ms, updates


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--windows', type=int, default=6)
  ap.add_argument('--steps', type=int, default=21)
  ap.add_argument('--frequency', type=int, default=20)
  ap.add_argument('--kernel-iters', type=int, default=50)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_summaries: needs a CUDA device')
  g = torch.Generator(device='cuda:0').manual_seed(1)
  images = torch.randn(256, 3, 224, 224, device='cuda:0', generator=g).to(torch.bfloat16) \
      .contiguous(memory_format=torch.channels_last)
  labels = torch.randint(0, 1000, (256,), device='cuda:0', generator=g)
  h = build(args.frequency, images, labels)
  ts = h._summaries
  for on in (False, True):        # warm-up, one whole update period each
    window(h, ts, images, labels, args.steps, on)
  times = {'off': [], 'on': []}
  updates = {'off': [], 'on': []}
  for _ in range(args.windows):
    for name in ('off', 'on'):
      ms, up = window(h, ts, images, labels, args.steps, name == 'on')
      times[name].append(ms)
      updates[name].append(int(up))

  # the two summary launches alone, on the last step's gradients
  ents = h.inner.plan_params()
  n_all = sum(p.numel() for p, _, _, _ in ents)
  n_masked = sum(p.numel() for p, _, b, _ in ents if b is not None)
  n_tasks = sum((p.numel() + 8191) // 8192 for p, _, _, _ in ents)
  nbytes = 8.0 * n_all + n_masked / 8.0 + 2 * 40.0 * n_tasks
  ts.run()                        # the plan for these buffers exists; the loop below is the two launches alone
  lib, stream = _cabi.lib(), _cabi.stream_ptr()
  run = lambda: _cabi.check(lib.rigl_summary_plan_run(ts._plan, ts.out.data_ptr(), stream), 'rigl_summary_plan_run')
  for _ in range(5):
    run()
  torch.cuda.synchronize()
  start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(args.kernel_iters):
    run()
  stop.record()
  stop.synchronize()
  kernel_ms = start.elapsed_time(stop) / args.kernel_iters

  off, on = float(np.median(times['off'])), float(np.median(times['on']))
  result = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), batch=256, image=224,
                steps_per_window=args.steps, windows=args.windows, mask_updates_per_window=updates,
                ms_per_step_off=times['off'], ms_per_step_on=times['on'], median_ms_off=off, median_ms_on=on,
                overhead_ms=on - off, overhead_pct=100.0 * (on - off) / off,
                summary_params=len(ents), summary_elements=n_all, summary_bytes=nbytes,
                summary_kernels_us=kernel_ms * 1e3, summary_tbs=nbytes / (kernel_ms * 1e-3) / 1e12,
                hbm_peak_tbs=HBM_TBS, data_sheet_floor_us=nbytes / (HBM_TBS * 1e12) * 1e6)
  print('%s, power limit %s' % (result['gpu'], result['power_limit']))
  print('ms/step  off %.3f  on %.3f  (+%.3f ms, %+.2f %%)' % (off, on, on - off, result['overhead_pct']))
  print('summary kernels %.1f us for %.3f GB: %.2f TB/s (data-sheet floor %.1f us)' % (
      result['summary_kernels_us'], nbytes / 1e9, result['summary_tbs'], result['data_sheet_floor_us']))
  print(json.dumps(result))


if __name__ == '__main__':
  main()
