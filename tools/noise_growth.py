"""How far apart are the reference's fp32 train step and the SAME step with bf16 activation storage (BASELINE's
bf16 configuration)?  Both run on the CPU oracle (oracle/cpu_train_step.py; `bf16_act` rounds every stored
activation tensor and its gradient to bf16, arithmetic inside an op stays fp32), so no kernel is involved: the
table is a property of the networks at initialisation, and it is why the whole-step parity tests compare the CUDA
step with the bf16-storage oracle, not with the fp32 one.

  python tools/noise_growth.py > noise_growth.md
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import cpu_train_step as cpu  # noqa: E402


def run(cls, shape, classes, seed, **kw):
  torch.manual_seed(seed)
  nets = [cls(seed=seed, bf16_weights=True, **kw) for _ in range(2)]
  nets[1].bf16_act = True
  x = torch.randn(*shape).to(torch.bfloat16).float()
  y = torch.randint(0, classes, (shape[0],))
  out = []
  for n in nets:
    n.trace = []
    out.append(n.forward_backward(x, y))
  return nets, out


def main():
  print('# r02: fp32 step vs bf16-activation-storage step on the CPU oracle (no kernels involved)')
  print()
  print('`python tools/noise_growth.py`.  Same weights (bf16-representable), masks, inputs; the only difference is '
        'that the second run rounds every stored activation tensor and its gradient to bf16.  `rel L2` = '
        '||a_bf16 - a_fp32|| / ||a_fp32|| of each batch-norm output in execution order (forward), and of the dense '
        'weight gradients (backward).')
  for title, cls, shape, classes, kw in (
      ('ResNet-50, 80 % ERK, batch 8, 64x64', cpu.CpuResNet50, (8, 3, 64, 64), 1000, dict(sparsity=0.8)),
      ('MobileNet-v1, 90 % uniform, batch 8, 64x64', cpu.CpuMobileNetV1, (8, 3, 64, 64), 1000, dict(sparsity=0.9)),
      ('WideResNet-22-2, 95 % ERK, batch 16, 32x32', cpu.CpuWideResNet, (16, 3, 32, 32), 10, dict(sparsity=0.95))):
    nets, ((l32, d32), (l16, d16)) = run(cls, shape, classes, 11, **kw)
    print()
    print('## ' + title)
    print()
    print('loss fp32 %.5f, bf16 storage %.5f' % (l32, l16))
    print()
    rows = [(k, float((b - a).norm() / (a.norm() + 1e-30))) for (k, a), (_, b) in zip(nets[0].trace, nets[1].trace)
            if not (cls is cpu.CpuResNet50 and k.endswith('3'))]          # (pre-add BN outputs are not stored)
    idx = sorted(set(list(range(0, len(rows), max(1, len(rows) // 12))) + [len(rows) - 1]))
    print('| BN output # | key | rel L2 (forward) |')
    print('|---|---|---|')
    for i in idx:
      print('| %d | %s | %.4f |' % (i, rows[i][0], rows[i][1]))
    growth = (rows[-1][1] / rows[0][1]) ** (1.0 / max(len(rows) - 1, 1))
    print()
    print('geometric growth per stored BN output: x%.3f' % growth)
    rel = [(k, float((d16[k] - d32[k]).norm() / (d32[k].norm() + 1e-30))) for k in d32]
    print()
    print('dense weight gradients: first layer %.3f, median %.3f, last layer %.3f' % (
        rel[0][1], float(np.median([r for _, r in rel])), rel[-1][1]))
  print()
  print('## Reading')
  print()
  print('* One bf16 rounding perturbs a tensor by ~1e-3 (2^-9 / sqrt(3) per element, two to three roundings per '
        'layer).  A batch-normalised ReLU network at initialisation amplifies a perturbation geometrically with '
        'depth (the known gradient-explosion / chaotic regime of BN networks at init, Yang et al. 2019): x1.1-1.2 '
        'per layer here, i.e. O(1) relative differences after ~50 layers and in every back-propagated gradient.')
  print('* The CUDA step agrees with the bf16-storage oracle to the bounds in tests/test_whole_step_parity_gpu.py, '
        'so its deviation from the fp32 oracle is of the size printed above.  The '
        'north-star 1e-5 is a per-op bound on fp32 accumulators (tests/test_conv_gpu.py); a whole-network bound '
        'against fp32 does not exist for bf16 storage at initialisation.')


if __name__ == '__main__':
  main()
