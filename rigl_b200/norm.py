"""Fused batch-norm + ReLU (+ residual add) on NHWC bf16 activations.

Host mirror of `batch_norm_relu(inputs, is_training, relu, init_zero)`
(rigl/imagenet_resnet/resnet_model.py:41-80; BATCH_NORM_DECAY 0.9, EPSILON 1e-5) and of the
`relu(inputs + shortcut)` tail of the bottleneck block (:501), backed by csrc/bn.cu.
Not a masked op in the reference -- it is the HBM-bound glue between the masked convs
(SURVEY 8f row 1), so it gets streaming kernels instead of tensor cores.
"""
import torch
from torch import nn

from . import _cabi
from .layers import _timed, _workspace, relu_gate


def _p(t):
  return None if t is None else t.data_ptr()


class _BNFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, y, gamma, beta, residual, mod, partial, fork=False):
    n, c, h, w = y.shape
    rows = n * h * w
    dev = y.device
    out = torch.empty_like(y, memory_format=torch.channels_last)
    save = torch.empty((4, c), dtype=torch.float32, device=dev)      # mean, rstd, scale, shift
    ws = _workspace(dev, _cabi.lib().rigl_bn_workspace_bytes(rows, c) + 8 * c + 256)
    # residual form with a ReLU: the backward needs only the SIGN of the block output -> one bit per element,
    # written by the apply pass.  Without a ReLU (MobileNet-v2's linear bottleneck) the backward needs nothing of it.
    bits = torch.empty(rows * c // 8, dtype=torch.uint8, device=dev) if (residual is not None and mod.relu) else None

    # batch statistics outside training (evaluation): the running statistics are not updated (NULL pointers)
    rmean, rvar = (mod.running_mean, mod.running_var) if mod.training else (None, None)

    def run():
      if partial is not None:       # statistics already reduced by the producing conv's epilogue
        _cabi.check(_cabi.lib().rigl_bn_forward_train_partials(
            y.data_ptr(), _p(residual), gamma.data_ptr(), beta.data_ptr(), partial[0].data_ptr(), partial[1],
            rows, c, mod.eps, mod.momentum, int(mod.relu), _p(rmean),
            _p(rvar), save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(),
            save[3].data_ptr(), out.data_ptr(), _p(bits), _cabi.stream_ptr()), 'rigl_bn_forward_train_partials')
        return
      _cabi.check(_cabi.lib().rigl_bn_forward_train(
          y.data_ptr(), _p(residual), gamma.data_ptr(), beta.data_ptr(), rows, c, mod.eps, mod.momentum,
          int(mod.relu), _p(rmean), _p(rvar), save[0].data_ptr(),
          save[1].data_ptr(), save[2].data_ptr(), save[3].data_ptr(), out.data_ptr(), ws.data_ptr(),
          ws.numel(), _p(bits), _cabi.stream_ptr()), 'rigl_bn_forward_train')
    _timed('bn_fwd', mod, run)
    ctx.mod, ctx.has_res, ctx.fork = mod, residual is not None, bool(fork)
    ctx.save_for_backward(y, bits, save)
    if fork:
      # Two handles on the same activation for its two consumers (next block's first conv and its
      # shortcut): backward then receives their gradients SEPARATELY and the sum is folded into
      # the column-sum pass (rigl_bn_backward) instead of autograd's elementwise add.
      ctx.set_materialize_grads(False)
      return out, out.detach()
    return out

  @staticmethod
  def backward(ctx, da, da_b=None):
    y, bits, save = ctx.saved_tensors
    mod = ctx.mod
    n, c, h, w = y.shape
    rows = n * h * w

    def as_grad(t):
      t = t.contiguous(memory_format=torch.channels_last)
      return t if t.dtype == torch.bfloat16 else t.to(torch.bfloat16)
    if ctx.fork:
      if da is None and da_b is None:
        return None, None, None, None, None, None, None
      if da is None:
        da, da_b = da_b, None
    da = as_grad(da)
    if da_b is not None:
      da_b = as_grad(da_b)
      if not ctx.has_res and mod.relu:       # a forked plain BN+ReLU: the sum is a separate elementwise add
        da, da_b = da + da_b, None
    dy = torch.empty_like(y, memory_format=torch.channels_last)
    # What the kernel writes besides dy (`g_out`, its residual-form output) and what this returns as the
    # gradient of the shortcut:
    #   residual, ReLU              g = da [+ da_b] masked by the bitmap -> a new tensor, returned
    #   residual, no ReLU, 1 grad   g = da itself: the plain form runs and `da` is handed back, no copy
    #   residual, no ReLU, 2 grads  g = bf16(da + da_b)                  -> a new tensor, returned
    #   plain, no ReLU, 2 grads     g = bf16(da + da_b)                  -> scratch that the dy pass reads (one
    #                               pass fewer than the elementwise add + plain backward: 7 vs 8 tensor passes)
    g_out, dres = None, None
    if ctx.has_res and (mod.relu or da_b is not None):
      g_out = dres = torch.empty_like(y, memory_format=torch.channels_last)
    elif ctx.has_res:
      dres = da
    elif da_b is not None:
      g_out = torch.empty_like(y, memory_format=torch.channels_last)
    dgb = torch.empty((2, c), dtype=torch.float32, device=y.device)
    ws = _workspace(y.device, _cabi.lib().rigl_bn_workspace_bytes(rows, c) + 8 * c + 256)

    def run():
      _cabi.check(_cabi.lib().rigl_bn_backward(
          da.data_ptr(), _p(da_b), y.data_ptr(), save[0].data_ptr(), save[1].data_ptr(), save[2].data_ptr(),
          save[3].data_ptr(), rows, c, int(mod.relu), dy.data_ptr(), _p(g_out), dgb[0].data_ptr(), dgb[1].data_ptr(),
          ws.data_ptr(), ws.numel(), _p(bits), _cabi.stream_ptr()), 'rigl_bn_backward')
    _timed('bn_bwd', mod, run)
    return dy, dgb[0], dgb[1], dres, None, None, None


class FusedBatchNormReLU(nn.Module):
  """y -> [relu](BN(y) [+ residual]); training mode uses batch statistics."""

  def __init__(self, channels, relu=True, init_zero=False, eps=1e-5, decay=0.9, device='cuda', name=None):
    super(FusedBatchNormReLU, self).__init__()
    if channels % 8:
      raise ValueError('FusedBatchNormReLU needs channels % 8 == 0')
    self.channels, self.relu, self.eps, self.momentum = channels, bool(relu), float(eps), 1.0 - float(decay)
    self.scope = name or 'batch_normalization'
    self.weight = nn.Parameter(torch.zeros(channels, device=device) if init_zero
                               else torch.ones(channels, device=device))
    self.bias = nn.Parameter(torch.zeros(channels, device=device))
    self.register_buffer('running_mean', torch.zeros(channels, device=device))
    self.register_buffer('running_var', torch.ones(channels, device=device))
    # Evaluation with batch statistics (the reference's --use_batch_statistics): in eval mode the training-form
    # forward runs, without updating the running statistics.
    self.batch_statistics = False
    self.frozen_coefficients = None     # (scale, shift) precomputed for an evaluation pass (workloads.Evaluator)

  def inference_coefficients(self):
    """(scale, shift) fp32 [C] of the inference form out = y * scale + shift: scale = gamma * rsqrt(var + eps),
    shift = beta - mean * scale.  The unfused eval forward and the conv-epilogue form (SparseConv2d.forward with
    `bn`) both take them from here, so both apply the same bits."""
    if self.frozen_coefficients is not None:
      return self.frozen_coefficients
    scale = self.weight.detach() * torch.rsqrt(self.running_var + self.eps)
    shift = self.bias.detach() - self.running_mean * scale
    return scale, shift

  def uses_inference_form(self):
    return not self.training and not self.batch_statistics

  def forward(self, y, residual=None, producer=None, fork=False, applied=False):
    """`producer`: the SparseConv2d whose output `y` is; if its epilogue emitted the batch statistics
    of exactly this tensor (layer.bn_partial), the stats pass is skipped.
    `fork`: return the activation TWICE (same storage) for its two consumers; their gradients are
    then summed inside the backward kernel instead of by a separate elementwise add (residual form, and
    the plain form without ReLU).
    `applied`: `y` is already this module's output (the producing conv applied the inference form in its
    epilogue); it is passed through."""
    if y.dim() != 4 or y.shape[1] != self.channels:
      raise ValueError('expected [N,%d,H,W]' % self.channels)
    if applied:
      return (y, y) if fork else y
    partial = None
    if producer is not None and getattr(producer, 'bn_partial', None) is not None:
      part, nrows, ptr = producer.bn_partial
      if ptr == y.data_ptr() and y.dtype == torch.bfloat16 and y.is_contiguous(memory_format=torch.channels_last):
        partial = (part, nrows)
      producer.bn_partial = None
    y = y.contiguous(memory_format=torch.channels_last)
    if y.dtype != torch.bfloat16:
      y = y.to(torch.bfloat16)
    if residual is not None:
      residual = residual.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    if self.training:
      return _BNFn.apply(y, self.weight, self.bias, residual, self, partial, fork)
    if self.batch_statistics:
      with torch.no_grad():
        out = _BNFn.apply(y, self.weight, self.bias, residual, self, partial, False)
      return (out, out) if fork else out
    scale, shift = self.inference_coefficients()
    out = torch.empty_like(y, memory_format=torch.channels_last)
    n, c, h, w = y.shape
    _cabi.check(_cabi.lib().rigl_bn_apply(y.data_ptr(), _p(residual), scale.data_ptr(), shift.data_ptr(),
                                          n * h * w, c, int(self.relu), out.data_ptr(), _cabi.stream_ptr()),
                'rigl_bn_apply')
    return (out, out) if fork else out


class _MaxPoolFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, ksize, stride):
    n, c, h, w = x.shape
    oh, ow = (h + stride - 1) // stride, (w + stride - 1) // stride
    y = torch.empty((n, c, oh, ow), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    arg = torch.empty((n, oh, ow, c), dtype=torch.uint8, device=x.device)
    _cabi.check(_cabi.lib().rigl_maxpool_same_forward(x.data_ptr(), n, h, w, c, ksize, stride, y.data_ptr(),
                                                      arg.data_ptr(), _cabi.stream_ptr()),
                'rigl_maxpool_same_forward')
    ctx.save_for_backward(arg)
    ctx.geom = (n, h, w, c, ksize, stride)
    return y

  @staticmethod
  def backward(ctx, dy):
    arg, = ctx.saved_tensors
    n, h, w, c, ksize, stride = ctx.geom
    dy = dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dx = torch.empty((n, c, h, w), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
    _cabi.check(_cabi.lib().rigl_maxpool_same_backward(dy.data_ptr(), arg.data_ptr(), n, h, w, c, ksize, stride,
                                                       dx.data_ptr(), _cabi.stream_ptr()),
                'rigl_maxpool_same_backward')
    return dx, None, None


def max_pool_same(x, ksize=3, stride=2):
  """tf.layers.max_pooling2d(pool_size, strides, padding='SAME') on NHWC bf16
  (resnet_model.py:636-642); x is [N,C,H,W] channels_last."""
  x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  return _MaxPoolFn.apply(x, int(ksize), int(stride))


class _MaxPool2x2ReluFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x):
    n, c, h, w = x.shape
    y = torch.empty((n, c, h // 2, w // 2), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
    arg = torch.empty((n, h // 2, w // 2, c), dtype=torch.uint8, device=x.device)
    _cabi.check(_cabi.lib().rigl_maxpool2x2_relu_forward(x.data_ptr(), n, h, w, c, y.data_ptr(), arg.data_ptr(),
                                                         _cabi.stream_ptr()), 'rigl_maxpool2x2_relu_forward')
    ctx.save_for_backward(arg)
    ctx.geom = (n, h, w, c)
    return y

  @staticmethod
  def backward(ctx, dy):
    arg, = ctx.saved_tensors
    n, h, w, c = ctx.geom
    dy = dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dx = torch.empty((n, c, h, w), dtype=torch.bfloat16, device=dy.device, memory_format=torch.channels_last)
    _cabi.check(_cabi.lib().rigl_maxpool2x2_relu_backward(dy.data_ptr(), arg.data_ptr(), n, h, w, c, dx.data_ptr(),
                                                          _cabi.stream_ptr()), 'rigl_maxpool2x2_relu_backward')
    return dx


def max_pool2x2_relu(x):
  """layers.max_pool2d([2, 2]) (stride 2, 'VALID') of VGG (vgg.py) over a ReLU output `x` ([N,C,H,W] channels_last
  bf16).  Its gradient goes only to each window's first maximum and only where that maximum is > 0, so it is already
  the gradient of the ReLU's input: the producing conv (SparseConv2d.relu_out) takes it as is."""
  x = x.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
  return _MaxPool2x2ReluFn.apply(x)


class _ReluGradGateFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, y):
    ctx.save_for_backward(y)
    return y.view_as(y)

  @staticmethod
  def backward(ctx, dy):
    y, = ctx.saved_tensors
    dy = dy.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    return relu_gate(y, dy, torch.empty_like(y, memory_format=torch.channels_last))


def relu_grad_gate(y):
  """Identity on a ReLU output `y` (SparseConv2d.relu_out) whose consumer does not gate (VGG's last conv feeds the
  global mean); the backward applies the ReLU's derivative, dy * (y > 0), with the standalone gate."""
  return _ReluGradGateFn.apply(y.contiguous(memory_format=torch.channels_last))
