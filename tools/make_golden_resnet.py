"""Generates tests/golden/resnet_sparsities_golden.json from the REFERENCE ITSELF.

Like tools/make_golden_vgg.py: imports the reference's own, unmodified `rigl/sparse_utils.py` (with its TensorFlow
and micronet-counting imports stubbed) and calls `get_sparsities` on fake mask objects carrying the mask names and
shapes of the reference's resnet_v1_ (tests/resnet_oracle.py) at 1000 classes: depths 18, 34, 101, 152 and 200 at
widths 0.5, 1 and 2 with both layers pruned, and at width 1 with prune_first_layer / prune_last_layer off, under
ERK 0.8, ERK 0.9 and random 0.9.  Per case the sparsities (float.hex) and surviving-weight counts are stored in the
layer order of the table.  Needs a checkout of google-research/rigl; the tests only read the JSON.

  python tools/make_golden_resnet.py [path to the rigl checkout]
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests'), os.path.dirname(os.path.abspath(__file__))]

import make_golden as mg  # noqa: E402  (stubs, fake mask objects)

DEPTHS = (18, 34, 101, 152, 200)
WIDTHS = (0.5, 1.0, 2.0)
METHODS = (('erdos_renyi_kernel', 0.8), ('erdos_renyi_kernel', 0.9), ('random', 0.9))
FLAGS = ((True, True), (False, True), (True, False), (False, False))


def cases():
  """(depth, width, prune_first_layer, prune_last_layer, method, sparsity) of every case."""
  for depth in DEPTHS:
    for width in WIDTHS:
      for first, last in FLAGS:
        if width != 1.0 and not (first and last):
          continue
        for method, s in METHODS:
          yield depth, width, first, last, method, s


def main():
  ref_root = sys.argv[1] if len(sys.argv) > 1 else mg.REF
  mg._install_stubs()
  sys.path.insert(0, ref_root)
  from rigl import sparse_utils as ref  # the reference, unmodified
  import resnet_oracle as ro

  out = {'generator': 'tools/make_golden_resnet.py', 'reference': 'google-research/rigl d39fc7d', 'cases': []}
  for depth, width, first, last, method, s in cases():
    layers = ro.masked_layers(depth, width, 1000, first, last)
    masks = [mg.RefMask(n, sh) for n, sh in layers]
    sp = ref.get_sparsities(masks, method, s, {})
    names = [n + '/mask:0' for n, _ in layers]
    nnz = [int(np.prod(sh)) - ref.get_n_zeros(int(np.prod(sh)), sp[n]) for n, (_, sh) in zip(names, layers)]
    assert set(sp) == set(names)
    out['cases'].append({'depth': depth, 'width': width, 'prune_first_layer': first, 'prune_last_layer': last,
                         'method': method, 'default_sparsity': s, 'n_layers': len(layers),
                         'sparsities_hex': [float(sp[n]).hex() for n in names], 'nnz': nnz})
  path = os.path.join(ROOT, 'tests', 'golden', 'resnet_sparsities_golden.json')
  with open(path, 'w') as f:
    json.dump(out, f, separators=(',', ':'), sort_keys=True)
  print('wrote', path, len(out['cases']), 'cases')


if __name__ == '__main__':
  main()
