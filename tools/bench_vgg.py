"""VGG-16 (rigl/imagenet_resnet/vgg.py) on the CUDA path: RigL ERK-0.8 train steps with the ReLU in the conv
epilogues against the standalone-gate composition (RIGL_FUSE_RELU=0's route: plain conv + rigl_relu_gate), timed
alternately in one process.  Prints one JSON line per measurement; needs a CUDA GPU.

  python tools/bench_vgg.py [--vgg-type vgg_16] [--batch 256] [--image 224] [--steps 24] [--rounds 4] [--warmup 3]

  * card: name and power limit (nvidia-smi), read in the same run as the numbers;
  * shapes: algorithmic FLOPs of a step (fwd + dgrad + dense wgrad of every masked layer at full density) and the
    bytes the fused ReLU route does not move, computed from the shapes (not measured);
  * train: per route, img/s and ms per step over `rounds` alternated blocks of steps/rounds CUDA-graph replays
    (momentum SGD, label smoothing 0.1), ONE mask update inside each route's timed window.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tools')]

from bench_mobilenet_v2 import card  # noqa: E402


def _emit(d):
  print(json.dumps(d), flush=True)


def shapes(vgg_type, batch, image):
  from rigl_b200 import workloads
  plan = workloads.vgg_plan(vgg_type)
  hw, macs, relu_fwd, gate_conv, gate_pool = image, 0, 0, 0, 0
  for i, (_, cin, cout, pool) in enumerate(plan):
    elems = batch * hw * hw * cout
    macs += 9 * cin * cout * hw * hw * batch
    relu_fwd += 4 * elems                       # the ReLU pass: read + write bf16
    if pool:
      gate_pool += 6 * elems                    # gate pass after the pool backward: read g and x, write (2+2+2 B)
      hw //= 2
    elif i + 1 < len(plan):
      gate_conv += 4 * elems                    # the gate reads x in the next dgrad's epilogue instead
  macs += plan[-1][2] * 1000 * batch
  _emit({'what': 'shapes', 'model': vgg_type, 'batch': batch, 'image': image, 'measured': False,
         'algorithmic_tflop_per_step': round(6 * macs / 1e12, 3),
         'bytes_not_moved_gb': {'relu_fwd': round(relu_fwd / 1e9, 2), 'gate_conv_edges': round(gate_conv / 1e9, 2),
                                'gate_pool_edges': round(gate_pool / 1e9, 2),
                                'total': round((relu_fwd + gate_conv + gate_pool) / 1e9, 2)}})
  return 6 * macs


def _harness(vgg_type, fuse, batch, image, update_at, dev):
  from rigl_b200 import layers, workloads
  layers.FUSE_RELU = fuse                      # the route is fixed into the captured graph
  torch.manual_seed(0)
  model = workloads.VGG(vgg_type, device=dev)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
  h = workloads.TrainHarness(model, lr=0.01, frequency=10 ** 6, begin_step=update_at, end_step=10 ** 7)
  return h


def train(vgg_type, batch, image, steps, rounds, warmup, flop):
  from rigl_b200 import layers
  dev = 'cuda:0'
  g = torch.Generator(device=dev).manual_seed(1)
  x = torch.randn(batch, 3, image, image, device=dev, generator=g).to(torch.bfloat16) \
      .contiguous(memory_format=torch.channels_last)
  y = torch.randint(0, 1000, (batch,), device=dev, generator=g)
  per_round = steps // rounds
  update_at = warmup + 1 + steps // 2          # global step of the mask update: inside the timed window
  hs = {}
  for route, fuse in (('fused_epilogues', True), ('standalone_gate', False)):
    h = _harness(vgg_type, fuse, batch, image, update_at, dev)
    for _ in range(warmup):
      h.step(x, y)
    assert h.enable_cuda_graph(x, y), 'CUDA-graph capture failed'
    h.step(x, y)
    hs[route] = h
  layers.FUSE_RELU = True
  torch.cuda.synchronize()
  times = {r: [] for r in hs}
  updates = {r: [] for r in hs}
  for i in range(rounds):
    order = list(hs) if i % 2 == 0 else list(hs)[::-1]
    for r in order:
      h = hs[r]
      ev = [torch.cuda.Event(enable_timing=True) for _ in range(per_round + 1)]
      ev[0].record()
      for k in range(per_round):
        h.step(x, y)
        updates[r].append(h.opt.last_update_was_mask_update)
        ev[k + 1].record()
      torch.cuda.synchronize()
      times[r] += [ev[k].elapsed_time(ev[k + 1]) for k in range(per_round)]
  for r in hs:
    t = np.array(times[r])
    normal = t[~np.array(updates[r])]
    _emit({'what': 'train', 'model': vgg_type, 'route': r, 'sparsity': 'erk0.8', 'batch': batch, 'image': image,
           'cuda_graph': True, 'steps': len(t), 'mask_updates_in_window': int(sum(updates[r])),
           'img_per_s': round(batch * len(t) / (t.sum() / 1e3), 1), 'median_step_ms': round(float(np.median(normal)), 3),
           'min_step_ms': round(float(normal.min()), 3), 'max_step_ms': round(float(normal.max()), 3),
           'algorithmic_tflops': round(flop / (float(np.median(normal)) / 1e3) / 1e12, 1)})


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--vgg-type', default='vgg_16')
  ap.add_argument('--batch', type=int, default=256)
  ap.add_argument('--image', type=int, default=224)
  ap.add_argument('--steps', type=int, default=24)
  ap.add_argument('--rounds', type=int, default=4)
  ap.add_argument('--warmup', type=int, default=3)
  args = ap.parse_args()
  flop = shapes(args.vgg_type, args.batch, args.image)
  if not torch.cuda.is_available():
    sys.exit('bench_vgg: needs a CUDA GPU (nothing is measured without one)')
  _emit(card())
  train(args.vgg_type, args.batch, args.image, args.steps, args.rounds, args.warmup, flop)


if __name__ == '__main__':
  main()
