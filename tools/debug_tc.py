"""On-device cross-check of the tensor-core (wgmma) implicit-GEMM kernels against the CUDA-core
kernels (same packed operands, same inputs), case by case, never stopping at a
failure.  Prints one line per (case, op) with max abs error / scale.

  python tools/debug_tc.py [--big]
"""
import argparse
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rigl_b200 import _cabi, pruning  # noqa: E402
from rigl_b200.layers import SparseConv2d, SparseLinear  # noqa: E402

DEV = 'cuda:0'

SMALL = [
    # n, h, w, cin, cout, k, stride, sparsity
    (2, 8, 8, 64, 64, 1, 1, 0.0),
    (4, 8, 8, 64, 128, 1, 1, 0.3),
    (2, 8, 8, 128, 64, 1, 1, 0.3),
    (2, 8, 8, 64, 256, 1, 1, 0.3),
    (3, 8, 8, 64, 64, 3, 1, 0.5),
    (2, 16, 16, 64, 64, 3, 1, 0.6),
    (2, 14, 14, 128, 128, 3, 1, 0.8),
    (2, 14, 14, 64, 128, 1, 2, 0.4),
    (2, 28, 28, 128, 128, 3, 2, 0.8),
    (8, 7, 7, 256, 256, 3, 1, 0.95),
    (2, 8, 8, 16, 32, 3, 1, 0.5),
    (2, 9, 7, 8, 16, 3, 2, 0.8),
    (2, 8, 8, 32, 72, 1, 1, 0.2),
    (4, 56, 56, 64, 64, 3, 1, 0.64),
    (4, 56, 56, 64, 256, 1, 1, 0.0),
    (4, 56, 56, 256, 64, 1, 1, 0.0),
    (2, 32, 32, 3, 64, 7, 2, 0.14),
    (2, 14, 14, 64, 64, 3, 1, 0.6),
    (2, 28, 28, 32, 128, 3, 1, 0.8),
    (2, 13, 27, 64, 24, 3, 1, 0.5),
    (5, 6, 14, 16, 64, 3, 1, 0.3),
]
BIG = [
    (32, 56, 56, 64, 64, 3, 1, 0.64),
    (32, 56, 56, 256, 128, 1, 1, 0.0),
    (32, 56, 56, 128, 128, 3, 2, 0.82),
    (32, 28, 28, 512, 128, 1, 1, 0.02),
    (32, 28, 28, 128, 512, 1, 1, 0.02),
    (32, 56, 56, 256, 512, 1, 2, 0.41),
    (32, 14, 14, 256, 256, 3, 1, 0.91),
    (32, 14, 14, 1024, 256, 1, 1, 0.51),
    (32, 7, 7, 512, 512, 3, 1, 0.957),
    (32, 7, 7, 2048, 512, 1, 1, 0.757),
    (32, 14, 14, 1024, 2048, 1, 2, 0.854),
    (16, 224, 224, 3, 64, 7, 2, 0.14),
]


def run_layer(layer, x, dy, force_simt):
  _cabi.lib().rigl_set_force_simt(1 if force_simt else 0)
  x = x.detach().clone().requires_grad_(True)
  layer.masked_weights.fresh = False
  layer.weight.grad = None
  y = layer(x)
  y.backward(dy)
  torch.cuda.synchronize()
  return y.detach().float(), x.grad.detach().float(), layer.masked_weights.dense_grad.clone()


def rel(a, b):
  scale = float(b.abs().max()) + 1e-30
  return float((a - b).abs().max()) / scale, scale


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--big', action='store_true')
  args = ap.parse_args()
  cases = SMALL + (BIG if args.big else [])
  bad = 0
  for case in cases:
    n, h, w, cin, cout, k, stride, sparsity = case
    torch.manual_seed(hash(case) % 100000)
    pruning.reset_default_registry()
    try:
      layer = SparseConv2d(cin, cout, k, strides=stride, padding='FIXED', name='t', device=DEV)
      layer.mask.assign((torch.rand(k, k, cin, cout, device=DEV) >= sparsity).float())
      x = torch.randn(n, cin, h, w, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
      ho = (h + 2 * layer.pad - k) // stride + 1
      wo = (w + 2 * layer.pad - k) // stride + 1
      dy = torch.randn(n, cout, ho, wo, device=DEV).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
      t0 = time.time()
      ref = run_layer(layer, x, dy, True)
      t1 = time.time()
      got = run_layer(layer, x, dy, False)
      t2 = time.time()
      line = []
      for name, a, b, tol in (('fprop', got[0], ref[0], 2e-2), ('dgrad', got[1], ref[1], 2e-2),
                              ('wgrad', got[2], ref[2], 1e-4)):
        r, sc = rel(a, b)
        ok = r <= tol and bool(torch.isfinite(a).all())
        bad += 0 if ok else 1
        line.append('%s %s rel=%.2e' % (name, 'ok ' if ok else 'BAD', r))
      print('%-40s %s   (simt %.3fs tc %.3fs)' % (case, ' | '.join(line), t1 - t0, t2 - t1), flush=True)
    except Exception as e:  # keep going: one line per failure
      bad += 1
      print('%-40s EXC %s' % (case, str(e)[:300]), flush=True)
      if 'CUDA error' in str(e) or 'unspecified launch failure' in str(e) or 'illegal' in str(e):
        print('fatal CUDA error; context is dead, stopping', flush=True)
        break
  # dense layers
  for m_rows, n_in, n_out in ((256, 2048, 1000), (100, 784, 300), (37, 64, 64)):
    try:
      pruning.reset_default_registry()
      layer = SparseLinear(n_in, n_out, name='fc', device=DEV, out_dtype=torch.float32)
      layer.mask.assign((torch.rand(n_in, n_out, device=DEV) >= 0.8).float())
      with torch.no_grad():
        layer.bias.normal_()
      x = torch.randn(m_rows, n_in, device=DEV).to(torch.bfloat16)
      dy = torch.randn(m_rows, n_out, device=DEV)
      ref = run_layer(layer, x, dy, True)
      got = run_layer(layer, x, dy, False)
      line = []
      for name, a, b, tol in (('fprop', got[0], ref[0], 1e-4), ('dgrad', got[1], ref[1], 2e-2),
                              ('wgrad', got[2], ref[2], 1e-4)):
        r, sc = rel(a, b)
        ok = r <= tol
        bad += 0 if ok else 1
        line.append('%s %s rel=%.2e' % (name, 'ok ' if ok else 'BAD', r))
      print('linear %-33s %s' % ((m_rows, n_in, n_out), ' | '.join(line)), flush=True)
    except Exception as e:
      bad += 1
      print('linear %s EXC %s' % ((m_rows, n_in, n_out), str(e)[:300]), flush=True)
  _cabi.lib().rigl_set_force_simt(0)
  print('DEBUG_TC bad=%d' % bad)


if __name__ == '__main__':
  main()
