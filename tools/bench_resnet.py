"""ResNet-18 ... 200 at any width (workloads.ResNet) on the CUDA path: RigL ERK-0.8 train steps under CUDA-graph
replay, and, for width > 1, the space-to-depth stem against the patch-matrix stem (RIGL_STEM_S2D=0's route) for the
stem alone.  Prints one JSON line per measurement; needs a CUDA GPU.

  python tools/bench_resnet.py [--depth 18] [--width 1] [--batch 256] [--image 224] [--steps 24] [--rounds 4]
                               [--warmup 3]

  * card: name and power limit (nvidia-smi), read in the same run as the numbers;
  * shapes: algorithmic FLOPs of a step (fwd + dgrad + dense wgrad of every masked layer at full density) and the
    stem's bytes: the folded input its halo tiles read once per 64-channel group against the output it writes,
    computed from the shapes (not measured);
  * stem (width > 1): fprop and wgrad of the stem alone, space-to-depth and patch-matrix routes alternated over
    `rounds` blocks in one process, with the 64-channel space-to-depth stem of width 1 as a yardstick for the
    grouped grid;
  * train: img/s and ms per step over `steps` CUDA-graph replays (momentum SGD, label smoothing 0.1), ONE mask update
    inside the timed window.  A configuration that does not fit in memory is reported as such.
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


def shapes(depth, width, batch, image):
  from rigl_b200 import workloads
  kind, c0, plan, fc_in = workloads.resnet_plan(depth, width)
  hw = image // 2
  macs = 49 * 3 * c0 * hw * hw
  hw = -(-hw // 2)                                       # the 3x3/2 'SAME' max pool
  mult = 4 if kind == 'bottleneck' else 1
  for _, cin, f, stride, proj in plan:
    out = -(-hw // stride)
    if proj:
      macs += cin * mult * f * out * out
    if kind == 'bottleneck':
      macs += cin * f * hw * hw + 9 * f * f * out * out + f * 4 * f * out * out
    else:
      macs += 9 * cin * f * out * out + 9 * f * f * out * out
    hw = out
  macs = (macs + fc_in * 1000) * batch
  # stem_s2d.cuh: R = 8 output rows per fprop strip, a halo tile of R + 3 folded rows x 128 positions x 32 B
  oh = image // 2
  r = min(8, oh)
  strips = -(-oh // r) * batch
  groups = -(-c0 // 64)
  halo = strips * (r + 3) * 128 * 32
  _emit({'what': 'shapes', 'model': 'resnet%d' % depth, 'width': width, 'batch': batch, 'image': image,
         'measured': False, 'algorithmic_tflop_per_step': round(6 * macs / 1e12, 3),
         'stem': {'cout': c0, 'groups': groups, 's2d_route': c0 <= 256 and c0 % 8 == 0,
                  'folded_input_gb': round(batch * ((image + 6) // 2) ** 2 * 32 / 1e9, 3),
                  'halo_reads_gb_per_group': round(halo / 1e9, 3), 'halo_reads_gb': round(groups * halo / 1e9, 3),
                  'output_gb': round(batch * oh * oh * c0 * 2 / 1e9, 3)}})
  return 6 * macs


def _stem_layer(cout, s2d, dev):
  from rigl_b200 import layers, pruning
  old = layers.STEM_S2D_PATH
  layers.STEM_S2D_PATH = s2d                  # read when the layer is built
  try:
    layer = layers.SparseConv2d(3, cout, 7, strides=2, padding='FIXED', device=dev,
                                registry=pruning.MaskedLayerRegistry())
  finally:
    layers.STEM_S2D_PATH = old
  rng = np.random.RandomState(0)
  layer.mask.assign((rng.rand(7, 7, 3, cout) < 0.5).astype(np.float32))
  layer.pack()
  return layer


def stem(width, batch, image, steps, rounds):
  """fprop (fold or im2col + conv) and wgrad (dense, + reduce) of the stem alone, routes alternated."""
  dev = 'cuda:0'
  c0 = int(64 * width)
  g = torch.Generator(device=dev).manual_seed(2)
  x = torch.randn(batch, 3, image, image, device=dev, generator=g).to(torch.bfloat16) \
      .contiguous(memory_format=torch.channels_last)
  routes = {'s2d': _stem_layer(c0, True, dev), 'patch_matrix': _stem_layer(c0, False, dev),
            's2d_width1_64ch': _stem_layer(64, True, dev)}
  dys = {}
  for r, l in routes.items():
    dys[r] = torch.randn(batch, l.out_channels, image // 2, image // 2, device=dev, generator=g) \
        .to(torch.bfloat16).contiguous(memory_format=torch.channels_last)

  def once(r):
    l = routes[r]
    l.masked_weights.fresh = False
    l.weight.grad = None
    e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    e[0].record()
    y = l(x)
    e[1].record()
    y.backward(dys[r])
    e[2].record()
    return e

  for r in routes:
    for _ in range(3):
      once(r)
  assert routes['s2d']._use_s2d and routes['s2d_width1_64ch']._use_s2d and not routes['patch_matrix']._use_s2d
  torch.cuda.synchronize()
  fw, wg = {r: [] for r in routes}, {r: [] for r in routes}
  per_round = max(1, steps // rounds)
  for i in range(rounds):
    for r in (list(routes) if i % 2 == 0 else list(routes)[::-1]):
      evs = [once(r) for _ in range(per_round)]
      torch.cuda.synchronize()
      fw[r] += [e[0].elapsed_time(e[1]) for e in evs]
      wg[r] += [e[1].elapsed_time(e[2]) for e in evs]
  for r in routes:
    _emit({'what': 'stem', 'route': r, 'cout': routes[r].out_channels, 'batch': batch, 'image': image,
           'calls': len(fw[r]), 'fprop_median_ms': round(float(np.median(fw[r])), 4),
           'wgrad_median_ms': round(float(np.median(wg[r])), 4),
           'note': 'fprop includes the fold / im2col, wgrad the backward through the layer (dense wgrad + reduce)'})
  del routes, dys
  torch.cuda.empty_cache()


def train(depth, width, batch, image, steps, warmup, flop):
  from rigl_b200 import workloads
  dev = 'cuda:0'
  g = torch.Generator(device=dev).manual_seed(1)
  what = {'what': 'train', 'model': 'resnet%d' % depth, 'width': width, 'sparsity': 'erk0.8', 'batch': batch,
          'image': image, 'cuda_graph': True}
  try:
    x = torch.randn(batch, 3, image, image, device=dev, generator=g).to(torch.bfloat16) \
        .contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (batch,), device=dev, generator=g)
    update_at = warmup + 1 + steps // 2          # global step of the mask update: inside the timed window
    torch.manual_seed(0)
    model = workloads.ResNet(depth, width=width, device=dev)
    workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
    h = workloads.TrainHarness(model, lr=0.1, frequency=10 ** 6, begin_step=update_at, end_step=10 ** 7)
    for _ in range(warmup):
      h.step(x, y)
    assert h.enable_cuda_graph(x, y), 'CUDA-graph capture failed'
    h.step(x, y)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
    updates = []
    ev[0].record()
    for k in range(steps):
      h.step(x, y)
      updates.append(h.opt.last_update_was_mask_update)
      ev[k + 1].record()
    torch.cuda.synchronize()
  except torch.cuda.OutOfMemoryError as e:
    _emit(dict(what, error='out of memory', detail=str(e).splitlines()[0]))
    return
  t = np.array([ev[k].elapsed_time(ev[k + 1]) for k in range(steps)])
  normal = t[~np.array(updates)]
  _emit(dict(what, steps=len(t), mask_updates_in_window=int(sum(updates)),
             img_per_s=round(batch * len(t) / (t.sum() / 1e3), 1), median_step_ms=round(float(np.median(normal)), 3),
             min_step_ms=round(float(normal.min()), 3), max_step_ms=round(float(normal.max()), 3),
             algorithmic_tflops=round(flop / (float(np.median(normal)) / 1e3) / 1e12, 1),
             peak_memory_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--depth', type=int, default=18)
  ap.add_argument('--width', type=float, default=1.0)
  ap.add_argument('--batch', type=int, default=256)
  ap.add_argument('--image', type=int, default=224)
  ap.add_argument('--steps', type=int, default=24)
  ap.add_argument('--rounds', type=int, default=4)
  ap.add_argument('--warmup', type=int, default=3)
  args = ap.parse_args()
  flop = shapes(args.depth, args.width, args.batch, args.image)
  if not torch.cuda.is_available():
    sys.exit('bench_resnet: needs a CUDA GPU (nothing is measured without one)')
  _emit(card())
  if args.width > 1:
    stem(args.width, args.batch, args.image, args.steps, args.rounds)
  train(args.depth, args.width, args.batch, args.image, args.steps, args.warmup, flop)


if __name__ == '__main__':
  main()
