"""Synchronous data parallelism for the sparse train step: one process per GPU,
torch.distributed (NCCL over NVLink on the box, gloo in the CPU tests).

Reference semantics (SURVEY 2b / 8e): weights, masks and optimizer slots are
replicated; the batch is split; per step
  * the DENSE masked-weight gradients are SUMMED across replicas
    (tpu_ops.cross_replica_sum, sparse_optimizers_base.py:471-476) -- they are the
    grow scores, so every replica ranks identical numbers and the masks stay
    replica-identical with no mask communication at all;
  * the gradients that feed the weight update are AVERAGED (CrossShardOptimizer,
    imagenet_train_eval.py:363-365);
  * batch-norm statistics stay per replica.

Layout: ONE flat fp32 buffer  [ other gradients (BN, biases) | layer 0 | layer 1 | ... ]  (128-element aligned
slices).  The masked weight gradient is re-derived locally as mask * dense / world (inside the fused optimizer
kernel), so it is never communicated.

Exchange: after backward, ONE SUM all-reduce of the whole flat buffer (`reduce_gradients`); under CUDA graphs it
runs eagerly between the backward replay and the optimizer replay.
"""
import torch
import torch.distributed as dist


def _align(n, a=128):
  return (n + a - 1) // a * a


class DataParallel(object):

  def __init__(self, process_group=None):
    if not (dist.is_available() and dist.is_initialized()):
      raise RuntimeError('torch.distributed must be initialised before DataParallel')
    self.group = process_group
    self.world = dist.get_world_size(process_group)
    self.rank = dist.get_rank(process_group)
    self.flat = None
    self.flat_dense = None
    self.flat_other = None
    self._others = []
    self.masked_grads_in_optimizer = False   # the fused optimizer forms mask * dense / world itself
    self.other_scale_in_optimizer = False    # ... and scales the other gradients by 1 / world

  # -- setup ------------------------------------------------------------------
  def attach(self, model):
    """Makes replicas identical (rank 0 wins) and lays the gradient buffers out flat."""
    layers = model.registry.layers()
    for p in model.parameters():
      dist.broadcast(p.data, 0, group=self.group)
    for b in model.buffers():
      dist.broadcast(b.data, 0, group=self.group)
    for l in layers:
      dist.broadcast(l.mask.bits, 0, group=self.group)
    dev = layers[0].weight.device
    masked = {id(l.weight) for l in layers}
    self._others = [p for p in model.parameters() if id(p) not in masked and p.requires_grad]
    n_other = _align(max(sum(_align(p.numel(), 4) for p in self._others), 1))
    total = n_other + sum(_align(l.weight.numel()) for l in layers)
    self.flat = torch.zeros(total, dtype=torch.float32, device=dev)
    self.flat_other = self.flat[:n_other]
    self.flat_dense = self.flat[n_other:]
    off = 0
    for p in self._others:
      n = p.numel()
      p.grad = self.flat_other[off:off + n].view_as(p)
      off += _align(n, 4)
    off = n_other
    for l in layers:
      n = l.weight.numel()
      l.masked_weights.dense_grad = self.flat[off:off + n]
      off += _align(n)
    return self

  # -- exchange -------------------------------------------------------------------
  def reduce_gradients(self, model):
    """SUM the dense grads, AVERAGE everything the inner optimizer consumes (one all-reduce of the flat buffer)."""
    if self.world > 1:
      dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group)
    self._post_reduce(model)

  def _post_reduce(self, model):
    if self.world > 1 and not self.other_scale_in_optimizer:
      self.flat_other.mul_(1.0 / self.world)
    scale = 1.0 / self.world
    for l in model.registry.layers():
      g = l.masked_weights.dense_grad
      g.rigl_reduced = True
      if self.masked_grads_in_optimizer:
        continue
      if l.weight.grad is None:
        l.weight.grad = torch.empty_like(l.weight)
      l.mask.apply_to(g, out=l.weight.grad.view(-1), scale=scale)

  def masks_identical(self, model):
    """Debug check: a 64-bit digest of every bitmap agrees on all ranks."""
    digest = torch.zeros(1, dtype=torch.int64, device=model.registry.layers()[0].weight.device)
    for i, l in enumerate(model.registry.layers()):
      digest += (l.mask.bits.to(torch.int64) * (2 * i + 1)).sum()
    lo, hi = digest.clone(), digest.clone()
    dist.all_reduce(lo, op=dist.ReduceOp.MIN, group=self.group)
    dist.all_reduce(hi, op=dist.ReduceOp.MAX, group=self.group)
    return bool((lo == hi).item())
