"""rigl_b200: H100-native RigL dynamic-sparse training hot path.

Host mirror of the reference API (google-research/rigl):
  rigl_b200.sparse_utils        <- rigl/sparse_utils.py
  rigl_b200.sparse_optimizers   <- rigl/sparse_optimizers.py (+ _base)
  rigl_b200.layers              <- rigl/imagenet_resnet/pruning_layers.py
  rigl_b200.pruning             <- tf.contrib.model_pruning getters
backed by hand-written sm_90a CUDA kernels behind the C ABI of include/rigl_b200.h.
"""
__version__ = '0.1.0'
