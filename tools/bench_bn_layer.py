"""Micro-benchmark of the fused batch-norm passes (forward train, backward) per ResNet-50 shape,
through the C ABI.  One JSON line per (shape, form): microseconds (CUDA events, median, inputs
rotated through more than 2x L2), algorithmic bytes and GB/s.

  python tools/bench_bn_layer.py [--iters 20] [--tag name]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rigl_b200 import _cabi  # noqa: E402

DEV = 'cuda:0'
# rows (= N*H*W at batch 256), channels, residual form
SHAPES = [
    (256 * 112 * 112, 64, False),
    (256 * 56 * 56, 64, False), (256 * 56 * 56, 256, True),
    (256 * 28 * 28, 128, False), (256 * 28 * 28, 512, True),
    (256 * 14 * 14, 256, False), (256 * 14 * 14, 1024, True),
    (256 * 7 * 7, 512, False), (256 * 7 * 7, 2048, True),
]
REPS = 5


def timed(fn, iters):
  ts = []
  for i in range(iters + 3):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda._sleep(1000000)
    a.record()
    for r in range(REPS):
      fn(i * REPS + r)
    b.record()
    b.synchronize()
    if i >= 3:
      ts.append(a.elapsed_time(b) * 1e3 / REPS)
  ts.sort()
  return ts[len(ts) // 2]


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--iters', type=int, default=20)
  ap.add_argument('--tag', default='')
  args = ap.parse_args()
  lib = _cabi.lib()
  for rows, c, res in SHAPES:
    nbytes = rows * c * 2
    copies = max(2, int(300e6 // nbytes) + 1)
    mk = lambda: [torch.randn(rows, c, device=DEV).to(torch.bfloat16) for _ in range(copies)]
    ys, das, outs = mk(), mk(), mk()
    rs = mk() if res else None
    da2s = mk() if res else None
    dys = [torch.empty(rows, c, dtype=torch.bfloat16, device=DEV) for _ in range(copies)]
    dres = [torch.empty(rows, c, dtype=torch.bfloat16, device=DEV) for _ in range(copies)] if res else None
    gamma = torch.ones(c, device=DEV); beta = torch.zeros(c, device=DEV)
    rm = torch.zeros(c, device=DEV); rv = torch.ones(c, device=DEV)
    save = torch.empty(4, c, device=DEV); dgb = torch.empty(2, c, device=DEV)
    ws = torch.empty(int(lib.rigl_bn_workspace_bytes(rows, c)) + 8 * c + 256, dtype=torch.uint8, device=DEV)
    p = lambda t: None if t is None else t.data_ptr()
    bits = [torch.empty(rows * c // 8, dtype=torch.uint8, device=DEV) for _ in range(copies)] if res else None

    def fwd(i):
      k = i % copies
      _cabi.check(lib.rigl_bn_forward_train(
          ys[k].data_ptr(), p(rs[k]) if res else None, gamma.data_ptr(), beta.data_ptr(), rows, c, 1e-5, 0.1, 1,
          rm.data_ptr(), rv.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(),
          save[3].data_ptr(), outs[k].data_ptr(), ws.data_ptr(), ws.numel(), bits[k].data_ptr() if res else None,
          _cabi.stream_ptr()), 'fwd')

    def bwd(i, two):
      k = i % copies
      _cabi.check(lib.rigl_bn_backward(
          das[k].data_ptr(), da2s[k].data_ptr() if (res and two) else None, ys[k].data_ptr(), save[0].data_ptr(),
          save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(), rows, c, 1, dys[k].data_ptr(),
          dres[k].data_ptr() if res else None, dgb[0].data_ptr(), dgb[1].data_ptr(), ws.data_ptr(), ws.numel(),
          bits[k].data_ptr() if res else None, _cabi.stream_ptr()), 'bwd')

    fwd(0)
    cases = [('fwd', fwd, (3 + (1 if res else 0)) * nbytes),
             ('bwd', lambda i: bwd(i, False), (8 if res else 5) * nbytes)]
    if res:
      cases.append(('bwd_2grads', lambda i: bwd(i, True), 9 * nbytes))
    for name, fn, alg in cases:
      us = timed(fn, args.iters)
      print(json.dumps({'tag': args.tag, 'rows': rows, 'c': c, 'residual': res, 'op': name, 'us': round(us, 2),
                        'tensor_mb': round(nbytes / 1e6, 1), 'passes_bytes_mb': round(alg / 1e6, 1),
                        'gbps': round(alg / us * 1e-3, 1)}), flush=True)


if __name__ == '__main__':
  main()
