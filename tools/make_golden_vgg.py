"""Generates tests/golden/vgg_sparsities_golden.json from the REFERENCE ITSELF.

Like tools/make_golden_mobilenet_v2.py: imports the reference's own, unmodified `rigl/sparse_utils.py` (with its
TensorFlow and micronet-counting imports stubbed) and calls `get_sparsities` on fake mask objects carrying the mask
names and shapes of the reference's vgg_a, vgg_16 and vgg_19 at width 1.0 and 1000 classes (tests/vgg_oracle.py),
with and without the masked fc8.  Needs a checkout of google-research/rigl; the tests only read the JSON.

  python tools/make_golden_vgg.py [path to the rigl checkout]
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.dirname(os.path.abspath(__file__))]

import make_golden as mg  # noqa: E402  (stubs, fake mask objects)


def main():
  ref_root = sys.argv[1] if len(sys.argv) > 1 else mg.REF
  mg._install_stubs()
  sys.path.insert(0, ref_root)
  from rigl import sparse_utils as ref  # the reference, unmodified
  import vgg_oracle as vo

  out = {'generator': 'tools/make_golden_vgg.py', 'reference': 'google-research/rigl d39fc7d', 'cases': []}
  for vgg_type in sorted(vo.CFG):
    for method, s in (('erdos_renyi_kernel', 0.8), ('erdos_renyi_kernel', 0.9), ('random', 0.9)):
      for prune_last in (True, False):
        layers = [(n, sh) for n, sh, _ in vo.masked_layers(vgg_type, 1000, prune_last)]
        masks = [mg.RefMask(n, sh) for n, sh in layers]
        sp = ref.get_sparsities(masks, method, s, {})
        nnz = {}
        for n, sh in layers:
          size = int(np.prod(sh))
          nnz[n + '/mask:0'] = size - ref.get_n_zeros(size, sp[n + '/mask:0'])
        out['cases'].append({'tag': '%s_%s%g_%s' % (vgg_type, method, s, 'prune_last' if prune_last else 'dense_last'),
                             'vgg_type': vgg_type, 'prune_last_layer': prune_last,
                             'layers': [[n, list(sh)] for n, sh in layers], 'method': method,
                             'default_sparsity': s, 'custom': {}, 'erk_power_scale': 1.0,
                             'sparsities_hex': mg._hex(sp), 'nnz': nnz})
  path = os.path.join(ROOT, 'tests', 'golden', 'vgg_sparsities_golden.json')
  with open(path, 'w') as f:
    json.dump(out, f, indent=1, sort_keys=True)
  print('wrote', path, len(out['cases']), 'cases')


if __name__ == '__main__':
  main()
