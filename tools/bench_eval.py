"""Eval-forward throughput (images/s) with the batch norm in the conv epilogue vs conv + rigl_bn_apply.

  python tools/bench_eval.py [--models resnet50,mobilenet_v1,mobilenet_v2] [--batches 256,1000] [--iters 20]

Each (model, batch) captures one CUDA graph of the evaluation step (forward + metric update) per setting of
layers.FUSE_BN_INFER and times the replays with device events, alternating the two settings round by round in
one process.  Also prints the GPU name and power limit read in the same run and, from the layer shapes, the bytes
the fusion removes per image (the conv output written and re-read: 4 bytes per element of every fused layer).
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from rigl_b200 import layers, workloads  # noqa: E402
from rigl_b200.evaluate import Evaluator  # noqa: E402

MODELS = {'resnet50': workloads.ResNet50, 'mobilenet_v1': workloads.MobileNetV1,
          'mobilenet_v2': workloads.MobileNetV2}


def gpu_info():
  try:
    out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
    return out.strip().splitlines()[0]
  except Exception as e:     # still report the device torch sees
    return '%s (power limit unavailable: %s)' % (torch.cuda.get_device_name(0), e)


def fused_bytes_per_image(model, size):
  """4 bytes per conv-output element of every layer that ran the fused variant (probed with one image)."""
  sizes = []
  hooks = [m.register_forward_hook(lambda m, i, o: sizes.append(o.numel()))
           for m in model.modules() if isinstance(m, layers.SparseConv2d)]
  ran = []
  orig = layers.SparseConv2d._fprop_bn

  def probe(self, x, bn, residual):
    out = orig(self, x, bn, residual)
    ran.append(out is not None)
    return out
  layers.SparseConv2d._fprop_bn = probe
  try:
    model.eval()
    with torch.no_grad():
      model(torch.zeros(1, 3, size, size, device='cuda', dtype=torch.bfloat16).contiguous(
          memory_format=torch.channels_last))
  finally:
    layers.SparseConv2d._fprop_bn = orig
    for h in hooks:
      h.remove()
  return 4 * sum(n for n, r in zip(sizes, ran) if r), sum(ran), len(sizes)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--models', default='resnet50,mobilenet_v1,mobilenet_v2')
  ap.add_argument('--batches', default='256,1000')
  ap.add_argument('--size', type=int, default=224)
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_eval.py needs a GPU')
  print(json.dumps({'gpu': gpu_info()}), flush=True)
  for name in args.models.split(','):
    torch.manual_seed(0)
    model = MODELS[name](device='cuda')
    workloads.init_masks(model, 'erdos_renyi_kernel', 0.8, seed=0)
    saved, n_fused, n_convs = fused_bytes_per_image(model, args.size)
    for batch in (int(b) for b in args.batches.split(',')):
      x = torch.randn(batch, 3, args.size, args.size, device='cuda').to(torch.bfloat16).contiguous(
          memory_format=torch.channels_last)
      y = torch.randint(0, 1000, (batch,), device='cuda')
      evs = {}
      for fused in (True, False):
        layers.FUSE_BN_INFER = fused
        ev = Evaluator(model)
        ev.reset()
        if not ev.enable_cuda_graph(x, y):
          raise SystemExit('graph capture failed')
        evs[fused] = ev
      layers.FUSE_BN_INFER = True
      times = {True: [], False: []}
      for _ in range(args.rounds):
        for fused in (True, False):
          ev = evs[fused]
          ev.update(x, y)
          s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
          s.record()
          for _ in range(args.iters):
            ev.update(x, y)
          e.record()
          e.synchronize()
          times[fused].append(s.elapsed_time(e) / args.iters)
      best = {k: min(v) for k, v in times.items()}
      print(json.dumps({
          'model': name, 'batch': batch, 'image': args.size,
          'fused_ms': round(best[True], 3), 'unfused_ms': round(best[False], 3),
          'fused_img_s': round(batch / best[True] * 1e3, 1), 'unfused_img_s': round(batch / best[False] * 1e3, 1),
          'speedup': round(best[False] / best[True], 4),
          'spread_fused_ms': [round(t, 3) for t in times[True]], 'spread_unfused_ms': [round(t, 3) for t in times[False]],
          'fused_layers': '%d of %d masked convs' % (n_fused, n_convs),
          'bytes_removed_per_batch_MB': round(saved * batch / 1e6, 1)}), flush=True)
      del evs


if __name__ == '__main__':
  main()
