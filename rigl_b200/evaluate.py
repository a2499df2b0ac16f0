"""Evaluation of a sparse model with the reference's eval metrics.

Mirror of `metric_fn` in resnet_model_fn_w_pruning (rigl/imagenet_resnet/imagenet_train_eval.py:594-621), the
metrics of `--mode=train_and_eval` / `--mode=eval_once`:
  eval_accuracy        tf.metrics.accuracy(labels, tf.argmax(logits, 1))     (ties: the lowest class index)
  top_5_eval_accuracy  tf.metrics.mean(tf.nn.in_top_k(logits, labels, 5))
  cross_loss           tf.metrics.mean of the batch's label-smoothed softmax cross-entropy broadcast to the batch,
                       i.e. the batch means weighted by batch size
  reg_loss             tf.losses.get_regularization_loss(): weight_decay * sum 1/2 ||W||^2 over the kernels that
                       carry an l2 kernel_regularizer
  pruning/<scope>/mask/sparsity   (eval_once only: utils.mask_summaries, tf.nn.zero_fraction of every mask)
`use_batch_statistics` is the reference's --use_batch_statistics (:545-546): batch norm normalises with the
statistics of the evaluated batch instead of the moving averages (which it leaves untouched).

The operands of the masked layers are packed once per pass (reset()): the weights do not change during an
evaluation.  Metrics accumulate on the device; result() synchronises once.  DESIGN.md 5 pins the semantics.
"""
import torch
import torch.nn.functional as F
from torch import nn

from . import _cabi
from . import layers
from .norm import FusedBatchNormReLU


def regularized_kernels(model):
  """The weights that carry an l2 kernel_regularizer in the reference model files: every conv and dense kernel
  (conv2d_fixed_padding, the masked layers, tf.layers.dense) except the depthwise ones, which are built with
  weights_regularizer=None (mobilenetv1_model.py:89, mobilenetv2_model.py:89), and modules marked
  `l2_regularized = False` (VGG's dense fc8, a contrib layers.conv2d without weights_regularizer, vgg.py:196).  Biases
  are not regularized."""
  from .workloads import DenseConv2d
  return [m.weight for m in model.modules() if isinstance(m, (layers._MaskedLayer, DenseConv2d, nn.Linear))
          and getattr(m, 'l2_regularized', True)]


def reg_loss(model, weight_decay):
  """weight_decay * sum 1/2 ||W||^2 over regularized_kernels(model) (tf.contrib.layers.l2_regularizer) as a 0-d
  fp32 tensor on the weights' device."""
  ws = regularized_kernels(model)
  total = torch.zeros((), dtype=torch.float32, device=ws[0].device) if ws else torch.zeros(())
  for w in ws:
    total = total + 0.5 * w.detach().float().pow(2).sum()
  return weight_decay * total


def batch_metrics(logits, labels, label_smoothing, k=5):
  """Sums of one batch as a float64 [3] tensor on the logits' device, no host synchronisation:
  (top-1 hits, in_top_k hits, batch size * mean label-smoothed cross-entropy).
    top-1     argmax picks the lowest index among equal maxima (tf.argmax).
    in_top_k  the target is in when fewer than k classes score strictly higher, so a tie straddling the k-th place
              counts as in; a row with any non-finite logit is a miss, and so is a label outside [0, classes).
    cross     tf.losses.softmax_cross_entropy(one_hot(labels), logits, label_smoothing): the target distribution is
              one_hot * (1 - label_smoothing) + label_smoothing / classes (an out-of-range label: one_hot = 0)."""
  logits = logits.float()
  n, classes = logits.shape
  labels = labels.to(device=logits.device, dtype=torch.long)
  valid = (labels >= 0) & (labels < classes)
  idx = labels.clamp(0, classes - 1).unsqueeze(1)
  top1 = (torch.argmax(logits, 1) == labels) & valid
  target = logits.gather(1, idx)
  in_k = ((logits > target).sum(1) < k) & torch.isfinite(logits).all(1) & valid
  onehot = torch.zeros_like(logits).scatter_(1, idx, valid.unsqueeze(1).float())
  soft = onehot * (1.0 - label_smoothing) + label_smoothing / classes
  cross = -(soft * torch.log_softmax(logits, 1)).sum(1).mean() * n
  return torch.stack([top1.sum().double(), in_k.sum().double(), cross.double()])


class Evaluator(object):
  """Accumulates the reference's eval metrics of `model` over batches:

    ev = Evaluator(model, weight_decay=1e-4)
    ev.reset()                       # packs the masked operands and the BN coefficients for this pass
    for images, labels in data:
      ev.update(images, labels)
    metrics = ev.result()            # dict of floats; one synchronisation

  An evaluation changes nothing a training step reads: weights, masks, dense gradients, BN running statistics,
  optimizer slots, the global step, the `fresh` flags, the pack-ahead set and the modules' training flags are as
  they were.  Call reset() again after the weights change."""

  def __init__(self, model, label_smoothing=0.1, weight_decay=1e-4, use_batch_statistics=False,
               mask_summaries=False):
    self.model = model
    self.label_smoothing = float(label_smoothing)
    self.weight_decay = float(weight_decay)
    self.use_batch_statistics = bool(use_batch_statistics)
    self.mask_summaries = bool(mask_summaries)
    registry = getattr(model, 'registry', None)
    self._masked = registry.layers() if registry is not None else \
        [m for m in model.modules() if isinstance(m, layers._MaskedLayer)]
    self._bns = [m for m in model.modules() if isinstance(m, FusedBatchNormReLU)]
    self._device = next(model.parameters()).device
    self._acc = torch.zeros(3, dtype=torch.float64, device=self._device)
    self._coef = {}
    self._count = 0
    self._ready = False
    self.graphed = False

  def reset(self):
    """Starts a pass: zero metrics; ONE launch packs the operands of every masked layer (pack_all, leaving the
    training step's pack-ahead set as it was); the BN inference coefficients, the regularization loss and the mask
    counts are computed from the current weights."""
    self._count = 0
    self._acc.zero_()
    ahead = set(layers._PACKED_AHEAD)
    layers.pack_all(self._masked)
    layers._PACKED_AHEAD.clear()
    layers._PACKED_AHEAD.update(ahead)
    with torch.no_grad():
      for bn in self._bns:
        bn.frozen_coefficients = None
        scale, shift = bn.inference_coefficients()
        if bn in self._coef:              # in place: a captured graph keeps reading the same buffers
          self._coef[bn][0].copy_(scale)
          self._coef[bn][1].copy_(shift)
        else:
          self._coef[bn] = (scale.clone(), shift.clone())
      self._reg = reg_loss(self.model, self.weight_decay)
    self._ones = None
    if self.mask_summaries:
      self._ones = torch.zeros(len(self._masked), dtype=torch.int32, device=self._device)
      for i, l in enumerate(self._masked):
        _cabi.check(_cabi.lib().rigl_mask_popcount(l.mask.bits.data_ptr(), l.mask.size,
                                                   self._ones[i:].data_ptr(), _cabi.stream_ptr()),
                    'rigl_mask_popcount')
    self._ready = True

  class _Scope(object):
    """Eval mode, no autograd, packed operands and BN coefficients frozen; everything restored on exit."""

    def __init__(self, ev):
      self.ev = ev

    def __enter__(self):
      ev = self.ev
      self.was_training = ev.model.training
      ev.model.eval()
      for bn in ev._bns:
        bn.frozen_coefficients = ev._coef[bn]
        bn.batch_statistics = ev.use_batch_statistics
      self.frozen = layers.frozen_operands(ev._masked).__enter__()
      self.no_grad = torch.no_grad()
      self.no_grad.__enter__()
      return self

    def __exit__(self, *exc):
      ev = self.ev
      self.no_grad.__exit__(*exc)
      self.frozen.__exit__(*exc)
      for bn in ev._bns:
        bn.frozen_coefficients = None
        bn.batch_statistics = False
      ev.model.train(self.was_training)
      return False

  def _step(self, images, labels):
    logits = self.model(images)
    self._acc += batch_metrics(logits, labels, self.label_smoothing)
    return logits

  def update(self, images, labels):
    """Inference forward of one batch and device-side accumulation of its metrics.  Returns the logits (with a
    captured graph: its static output buffer, overwritten by the next update)."""
    if not self._ready:
      raise RuntimeError('Evaluator.update before reset()')
    n = int(images.shape[0])
    if self.graphed:
      if tuple(images.shape) != tuple(self._sx.shape) or tuple(labels.shape) != tuple(self._sy.shape):
        raise ValueError('captured for images %s / labels %s, got %s / %s' % (
            tuple(self._sx.shape), tuple(self._sy.shape), tuple(images.shape), tuple(labels.shape)))
      self._sx.copy_(images, non_blocking=True)
      self._sy.copy_(labels, non_blocking=True)
      self._graph.replay()
      self._count += n
      return self._slogits
    with Evaluator._Scope(self):
      logits = self._step(images, labels)
    self._count += n
    return logits

  def enable_cuda_graph(self, images, labels=None, warmup=2):
    """Captures the forward and the metric update for the batch shape of `images` (in the manner of
    TrainHarness.enable_cuda_graph); update() then replays it.  Needs reset() first; the metrics of the warm-up
    and capture runs are discarded.  Returns False (and stays eager) if the capture fails."""
    if not self._ready:
      raise RuntimeError('Evaluator.enable_cuda_graph before reset()')
    if labels is None:
      labels = torch.zeros(images.shape[0], dtype=torch.long, device=images.device)
    self._sx, self._sy = images.clone(), labels.clone()
    try:
      with Evaluator._Scope(self):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
          for _ in range(warmup):
            self._step(self._sx, self._sy)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph, capture_error_mode='thread_local'):
          self._slogits = self._step(self._sx, self._sy)
      self.graphed = True
    except Exception as e:      # stay eager, but say why
      import warnings
      warnings.warn('CUDA-graph capture of the evaluation failed, running eagerly: %r' % (e,))
      torch.cuda.synchronize()
      self.graphed = False
    self._acc.zero_()
    return self.graphed

  def result(self):
    """The metrics accumulated since reset() as a dict of floats (one device synchronisation)."""
    if not self._ready:
      raise RuntimeError('Evaluator.result before reset()')
    parts = [self._acc, self._reg.double().reshape(1).to(self._acc.device)]
    if self._ones is not None:
      parts.append(self._ones.double())
    vals = torch.cat(parts).cpu().tolist()
    n = float(self._count)
    top1, top5, cross, reg = vals[:4]
    out = {
        'eval_accuracy': top1 / n if n else float('nan'),
        'top_5_eval_accuracy': top5 / n if n else float('nan'),
        'cross_loss': cross / n if n else float('nan'),
        'reg_loss': reg,
    }
    if self._ones is not None:
      for l, ones in zip(self._masked, vals[4:]):
        out['pruning/%s/mask/sparsity' % l.mask.scope] = 1.0 - ones / float(l.mask.size)
    return out
