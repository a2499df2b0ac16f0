"""world_size-2 gloo test of the data-parallel host logic (no GPU): flat gradient
layout, SUM of dense grads, AVERAGE of optimizer grads, replica-identical digests."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp


class _FakeMask(object):

  def __init__(self, dense):
    self.dense = dense
    self.bits = (dense.view(-1) > 0).to(torch.int32)

  def apply_to(self, src, out=None, scale=1.0):
    out.copy_(src * self.dense.view(-1) * scale)
    return out


class _FakeMW(object):

  def __init__(self, n):
    self.dense_grad = torch.zeros(n)


class _FakeLayer(object):

  def __init__(self, shape, seed):
    g = torch.Generator().manual_seed(seed)
    self.weight = torch.nn.Parameter(torch.randn(shape, generator=g))
    self.mask = _FakeMask((torch.rand(shape, generator=g) > 0.5).float())
    self.masked_weights = _FakeMW(self.weight.numel())


class _FakeRegistry(object):

  def __init__(self, layers):
    self._l = layers

  def layers(self):
    return self._l


class _FakeModel(torch.nn.Module):

  def __init__(self, rank):
    super(_FakeModel, self).__init__()
    layers = [_FakeLayer((5, 7), 10 + rank), _FakeLayer((130,), 20 + rank)]
    self.registry = _FakeRegistry(layers)
    self.w0, self.w1 = layers[0].weight, layers[1].weight
    self.bias = torch.nn.Parameter(torch.full((3,), float(rank)))


def _worker(rank, world, port):
  os.environ['MASTER_ADDR'] = '127.0.0.1'
  os.environ['MASTER_PORT'] = str(port)
  dist.init_process_group('gloo', rank=rank, world_size=world)
  from rigl_b200.data_parallel import DataParallel
  model = _FakeModel(rank)
  dp = DataParallel().attach(model)
  # replicas identical after attach (rank 0 wins)
  ref = _FakeModel(0)
  assert torch.equal(model.w0.data, ref.w0.data) and torch.equal(model.bias.data, ref.bias.data)
  assert torch.equal(model.registry.layers()[0].mask.bits, ref.registry.layers()[0].mask.bits)
  assert dp.masks_identical(model)
  for l in model.registry.layers():          # the fake keeps a dense copy: refresh it from the bits
    l.mask.dense = l.mask.bits.float().view(l.weight.shape)
  # dense grads are views of one flat, 128-element-aligned buffer
  l0, l1 = model.registry.layers()
  assert l0.masked_weights.dense_grad.data_ptr() == dp.flat_dense.data_ptr()
  assert l1.masked_weights.dense_grad.data_ptr() == dp.flat_dense.data_ptr() + 128 * 4
  l0.masked_weights.dense_grad.fill_(rank + 1.0)
  l1.masked_weights.dense_grad.fill_(10.0 * (rank + 1))
  model.bias.grad.fill_(rank + 1.0)
  dp.reduce_gradients(model)
  assert torch.all(l0.masked_weights.dense_grad == 3.0)           # SUM over 2 ranks
  assert torch.all(l1.masked_weights.dense_grad == 30.0)
  assert torch.all(model.bias.grad == 1.5)                         # AVERAGE
  want = 3.0 * ref.registry.layers()[0].mask.dense / 2.0           # mask * dense / world
  assert torch.equal(l0.weight.grad, want)
  assert getattr(l0.masked_weights.dense_grad, 'rigl_reduced', False)
  # scaling folded into the fused optimizer: the exchange leaves SUMS and does not form the masked gradient
  dp.masked_grads_in_optimizer = dp.other_scale_in_optimizer = True
  l0.masked_weights.dense_grad.fill_(rank + 1.0)
  l1.masked_weights.dense_grad.fill_(10.0 * (rank + 1))
  model.bias.grad.fill_(rank + 1.0)
  l0.masked_weights.dense_grad.rigl_reduced = False
  w_grad_before = l0.weight.grad.clone()
  dp.reduce_gradients(model)
  assert torch.all(l0.masked_weights.dense_grad == 3.0) and torch.all(l1.masked_weights.dense_grad == 30.0)
  assert torch.all(model.bias.grad == 3.0)                         # SUM: 1/world is the optimizer's
  assert torch.equal(l0.weight.grad, w_grad_before)               # masked gradient left to the fused optimizer
  assert getattr(l0.masked_weights.dense_grad, 'rigl_reduced', False)
  # diverging masks are detected
  if rank == 1:
    l1.mask.bits[0] ^= 1
  assert not dp.masks_identical(model)
  dist.destroy_process_group()


def test_data_parallel_one_all_reduce_two_ranks_gloo():
  with socket.socket() as s:
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
  mp.spawn(_worker, args=(2, port), nprocs=2, join=True)
