"""MobileNet-v2 (rigl/imagenet_resnet/mobilenetv2_model.py) on the CUDA path: RigL ERK-0.8 train steps and the
linear-bottleneck batch-norm backward.  Prints one JSON line per measurement; needs a CUDA GPU.

  python tools/bench_mobilenet_v2.py [--batch 256] [--image 224] [--steps 40] [--warmup 5] [--bn-iters 30]

  * card: name and power limit (nvidia-smi), read in the same run as the numbers;
  * train: img/s over `steps` CUDA-graph-replayed steps (momentum SGD, label smoothing 0.1) with ONE mask update
    inside the timed window, the update step's time and what it costs over a normal step;
  * flops: masked-FLOP accounting of bench.masked_flops_per_image at the model's ERK densities;
  * bn_bwd: the backward of a no-ReLU BN whose output has two consumers, at the shapes MobileNet-v2 forks at batch
    `batch`: the in-kernel gradient sum (rigl_bn_backward with da2) against a torch add followed by the kernel on
    the sum, timed alternately with CUDA events.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _emit(d):
  print(json.dumps(d), flush=True)


def card():
  name = torch.cuda.get_device_name(0)
  try:
    q = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                       stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=60).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    q = 'unavailable'
  return {'what': 'card', 'name': name, 'power_limit_and_max_sm_clock': q}


def train(batch, image, steps, warmup):
  import numpy as np
  import bench
  from rigl_b200 import workloads
  dev = 'cuda:0'
  torch.manual_seed(0)
  model = workloads.MobileNetV2(device=dev)
  workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
  # one mask update, in the middle of the timed window (RigL: no global-step increment on the update iteration)
  update_at = warmup + steps // 2
  h = workloads.TrainHarness(model, lr=0.1, frequency=10 ** 6, begin_step=update_at, end_step=10 ** 7)
  g = torch.Generator(device=dev).manual_seed(1)
  x = torch.randn(batch, 3, image, image, device=dev, generator=g).to(torch.bfloat16) \
      .contiguous(memory_format=torch.channels_last)
  y = torch.randint(0, 1000, (batch,), device=dev, generator=g)
  for _ in range(warmup):
    h.step(x, y)
  graphed = h.enable_cuda_graph(x, y)
  h.step(x, y)                               # first replay (warm)
  torch.cuda.synchronize()
  ev = [torch.cuda.Event(enable_timing=True) for _ in range(steps + 1)]
  updates = []
  ev[0].record()
  for i in range(steps):
    h.step(x, y)
    updates.append(h.opt.last_update_was_mask_update)
    ev[i + 1].record()
  torch.cuda.synchronize()
  per = [ev[i].elapsed_time(ev[i + 1]) for i in range(steps)]
  total_s = ev[0].elapsed_time(ev[-1]) / 1e3
  normal = [t for t, u in zip(per, updates) if not u]
  upd = [t for t, u in zip(per, updates) if u]
  _emit({'what': 'train', 'model': 'mobilenet_v2', 'sparsity': 'erk0.8', 'batch': batch, 'image': image,
         'cuda_graph': graphed, 'steps': steps, 'mask_updates_in_window': len(upd),
         'img_per_s': round(batch * steps / total_s, 1), 'median_step_ms': round(float(np.median(normal)), 3),
         'update_step_ms': [round(t, 3) for t in upd],
         'mask_update_extra_ms': [round(t - float(np.median(normal)), 3) for t in upd]})
  fl = bench.masked_flops_per_image(model, image, dev)
  _emit(dict({'what': 'flops', 'image': image, 'per_image': True}, **{k: round(v, 4) for k, v in fl.items()}))
  step_s = float(np.median(normal)) / 1e3
  _emit({'what': 'flops_rate', 'algorithmic_tflops': round(fl['algorithmic_gflop'] * batch / step_s / 1e3, 2),
         'dense_executed_tflops': round(fl['dense_executed_gflop'] * batch / step_s / 1e3, 2)})
  del h, model
  torch.cuda.empty_cache()


def bn_backward(batch, iters):
  from rigl_b200 import _cabi
  lib = _cabi.lib()
  dev = 'cuda:0'
  # (spatial, channels) of every MobileNet-v2 block output that is handed to two consumers
  shapes = [(56, 24), (28, 32), (14, 64), (14, 96), (7, 160)]
  for hw, c in shapes:
    rows = batch * hw * hw
    nbytes = rows * c * 2
    copies = max(2, int(120e6 // nbytes) + 1)                 # rotate the inputs through more than 2x L2
    mk = lambda: [torch.randn(rows, c, device=dev).to(torch.bfloat16) for _ in range(copies)]
    ys, das, da2s = mk(), mk(), mk()
    dy = torch.empty(rows, c, dtype=torch.bfloat16, device=dev)
    scratch = torch.empty(rows, c, dtype=torch.bfloat16, device=dev)
    save = torch.stack([torch.zeros(c), torch.ones(c), torch.ones(c), torch.zeros(c)]).to(dev)
    dgb = torch.empty(2, c, device=dev)
    ws = torch.empty(int(lib.rigl_bn_workspace_bytes(rows, c)) + 8 * c + 256, dtype=torch.uint8, device=dev)

    def call(k, da, da2, g_out):
      _cabi.check(lib.rigl_bn_backward(
          da.data_ptr(), None if da2 is None else da2.data_ptr(), ys[k].data_ptr(), save[0].data_ptr(),
          save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(), rows, c, 0, dy.data_ptr(),
          None if g_out is None else g_out.data_ptr(), dgb[0].data_ptr(), dgb[1].data_ptr(), ws.data_ptr(),
          ws.numel(), None, _cabi.stream_ptr()), 'rigl_bn_backward')

    def new(k):
      call(k, das[k], da2s[k], scratch)

    def old(k):
      call(k, das[k] + da2s[k], None, None)

    times = {'in_kernel_sum': [], 'torch_add_then_kernel': []}
    for k in range(copies):          # warm-up (and the same result both ways)
      new(k)
      a = dy.clone()
      old(k)
      assert torch.equal(a, dy), (hw, c)
    for i in range(iters):
      for name, fn in (('in_kernel_sum', new), ('torch_add_then_kernel', old)) if i % 2 == 0 else \
          (('torch_add_then_kernel', old), ('in_kernel_sum', new)):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for k in range(copies):
          fn(k)
        b.record()
        b.synchronize()
        times[name].append(a.elapsed_time(b) * 1e3 / copies)
    med = {n: sorted(t)[len(t) // 2] for n, t in times.items()}
    _emit({'what': 'bn_bwd_two_grads_no_relu', 'batch': batch, 'hw': hw, 'c': c, 'tensor_mb': round(nbytes / 1e6, 1),
           'us_in_kernel_sum': round(med['in_kernel_sum'], 2), 'us_torch_add_then_kernel':
           round(med['torch_add_then_kernel'], 2), 'speedup': round(med['torch_add_then_kernel'] / med['in_kernel_sum'], 3),
           'passes': {'in_kernel_sum': 7, 'torch_add_then_kernel': 8}})


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--batch', type=int, default=256)
  ap.add_argument('--image', type=int, default=224)
  ap.add_argument('--steps', type=int, default=40)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--bn-iters', type=int, default=30)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit('bench_mobilenet_v2: needs a CUDA GPU (nothing is measured without one)')
  _emit(card())
  train(args.batch, args.image, args.steps, args.warmup)
  bn_backward(args.batch, args.bn_iters)


if __name__ == '__main__':
  main()
