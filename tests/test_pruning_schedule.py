"""Host side of gradual magnitude pruning (rigl_b200.pruning) against the NumPy restatement in
tests/pruning_oracle.py: hyperparameters, the float32 sparsity schedule, the update steps, weight_sparsity_map
scaling and the per-layer keep count."""
import numpy as np
import pytest

import pruning_oracle as oracle
from rigl_b200 import pruning

DEFAULTS = dict(name='model_pruning', begin_pruning_step=0, end_pruning_step=-1, weight_sparsity_map=[''],
                threshold_decay=0.0, pruning_frequency=10, nbins=256, block_height=1, block_width=1,
                block_pooling_function='AVG', initial_sparsity=0.0, target_sparsity=0.5,
                sparsity_function_begin_step=0, sparsity_function_end_step=100, sparsity_function_exponent=3,
                use_tpu=False)

# (begin = sparsity_function_begin_step, end = sparsity_function_end_step, frequency, target) of the drivers'
# default flags: cifar_resnet/resnet_train_eval.py and mnist/mnist_train_eval.py
CIFAR = (20000, 75000, 1000, 0.9)
MNIST = (2000, 30000, 500, 0.98)


def _spec(begin, end, frequency, target, decay=0.0):
  s = ('begin_pruning_step={0},sparsity_function_begin_step={0},end_pruning_step={1},'
       'sparsity_function_end_step={1},target_sparsity={2},pruning_frequency={3},threshold_decay={4},'
       'use_tpu=False'.format(begin, end, target, frequency, decay))
  return pruning.get_pruning_hparams().parse(s)


def _pruning(spec):
  return pruning.Pruning(spec, global_step=None, registry=pruning.MaskedLayerRegistry())


def test_hparams_defaults():
  assert pruning.get_pruning_hparams().values() == DEFAULTS


def test_hparams_parse_and_set():
  hp = _spec(*CIFAR)
  assert hp.begin_pruning_step == 20000 and hp.end_pruning_step == 75000
  assert hp.sparsity_function_begin_step == 20000 and hp.sparsity_function_end_step == 75000
  assert hp.target_sparsity == 0.9 and hp.pruning_frequency == 1000 and hp.threshold_decay == 0.0
  assert hp.use_tpu is False and isinstance(hp.pruning_frequency, int)
  hp.set_hparam('weight_sparsity_map', ['layer2:0.81', 'layer3:0.0'])
  assert hp.weight_sparsity_map == ['layer2:0.81', 'layer3:0.0']
  assert pruning.get_pruning_hparams().parse('weight_sparsity_map=[a:0.1,b:0.2]').weight_sparsity_map == \
      ['a:0.1', 'b:0.2']
  assert pruning.get_pruning_hparams().parse('nbins=512,use_tpu=True').nbins == 512


def test_hparams_reject():
  with pytest.raises(ValueError):
    pruning.get_pruning_hparams().parse('no_such_hparam=1')
  with pytest.raises(ValueError):
    pruning.get_pruning_hparams().set_hparam('no_such_hparam', 1)
  with pytest.raises(ValueError):
    pruning.get_pruning_hparams().parse('pruning_frequency=1.5')
  for dims in ('block_height=2', 'block_width=4'):
    with pytest.raises(ValueError):
      _pruning(pruning.get_pruning_hparams().parse(dims))
  with pytest.raises(ValueError):
    _pruning(pruning.get_pruning_hparams().parse('sparsity_function_begin_step=100,sparsity_function_end_step=100'))


@pytest.mark.parametrize('flags', [CIFAR, MNIST], ids=['cifar', 'mnist'])
def test_sparsity_sweep(flags):
  begin, end, frequency, target = flags
  p = _pruning(_spec(*flags))
  steps = list(range(0, end + 3 * frequency, 37)) + [begin - 1, begin, begin + 1, end - 1, end, end + 1]
  for gs in steps:
    got = p.sparsity(gs)
    want = oracle.sparsity(gs, 0.0, target, begin, end, 3)
    assert got.dtype == np.float32 and got.tobytes() == want.tobytes(), gs
  assert p.sparsity(0) == 0 and p.sparsity(end + 5) == np.float32(target)


def test_sparsity_initial_and_exponent():
  hp = pruning.get_pruning_hparams().parse('initial_sparsity=0.2,target_sparsity=0.95,sparsity_function_exponent=2,'
                                           'sparsity_function_begin_step=7,sparsity_function_end_step=1007')
  p = _pruning(hp)
  for gs in range(0, 1100, 13):
    assert p.sparsity(gs).tobytes() == oracle.sparsity(gs, 0.2, 0.95, 7, 1007, 2).tobytes()


@pytest.mark.parametrize('flags,end_pruning', [(CIFAR, None), (MNIST, None), (CIFAR, -1), ((2, 12, 2, 0.9), None),
                                               ((2, 12, 2, 0.9), -1)])
def test_update_steps(flags, end_pruning):
  begin, end, frequency, target = flags
  hp = _spec(*flags)
  if end_pruning is not None:
    hp.set_hparam('end_pruning_step', end_pruning)
  p = _pruning(hp)
  steps = range(1, end + 5 * frequency)
  got = []
  for gs in steps:
    if p.is_update_step(gs):
      got.append(gs)
      p.last_update_step = gs
  want = oracle.update_steps(steps, begin, hp.end_pruning_step, frequency)
  assert got == want
  assert got[0] == begin and (got[-1] == end if end_pruning is None else got[-1] > end)


def test_weight_sparsity_map_scaling():
  hp = _spec(*MNIST)
  hp.set_hparam('weight_sparsity_map', ['layer2:0.81', 'layer3:0.0'])
  p = _pruning(hp)
  for gs in (1999, 2000, 9000, 30000, 40000):
    s = p.sparsity(gs)
    for name in ('layer1/weights', 'layer2/weights', 'layer3/weights'):
      want = oracle.layer_sparsity(s, name, hp.weight_sparsity_map, hp.target_sparsity)
      ratio = p._ratio_for(name)
      got = s if ratio is None else np.float32(s * ratio)
      assert got.tobytes() == np.float32(want).tobytes(), (gs, name)
    assert np.float32(s * p._ratio_for('layer3/weights')) == 0
    assert pruning.keep_count(1000, np.float32(s * p._ratio_for('layer3/weights'))) == 1000


def test_weight_sparsity_map_multiple_match():
  hp = _spec(*MNIST)
  hp.set_hparam('weight_sparsity_map', ['layer:0.5', 'layer2:0.8'])
  p = _pruning(hp)
  with pytest.raises(ValueError):
    p._ratio_for('layer2/weights')
  with pytest.raises(ValueError):
    oracle.layer_sparsity(np.float32(0.5), 'layer2/weights', hp.weight_sparsity_map, hp.target_sparsity)
  hp.set_hparam('weight_sparsity_map', ['layer2:1.0'])
  with pytest.raises(ValueError):
    _pruning(hp)


@pytest.mark.parametrize('n,s,k', [(5, 0.5, 2), (7, 0.5, 4), (9, 0.5, 4), (11, 0.5, 6), (6, 0.75, 2),
                                   (10, 0.75, 2), (14, 0.75, 4), (2049, 0.5, 1024), (2051, 0.5, 1026)])
def test_keep_half_to_even(n, s, k):
  assert float(np.float32(n) * (np.float32(1) - np.float32(s))) % 1.0 == 0.5
  assert pruning.keep_count(n, np.float32(s)) == k == oracle.keep(n, np.float32(s))


@pytest.mark.parametrize('n,s', [(1, 0.9), (10, 0.99), (1000, 1.0), (129, 0.999)])
def test_keep_clamped_at_one(n, s):
  assert pruning.keep_count(n, np.float32(s)) == 1 == oracle.keep(n, np.float32(s))


def test_keep_matches_oracle_sweep():
  rng = np.random.RandomState(0)
  for n in list(rng.randint(1, 3 * 10 ** 6, size=200)) + [1, 2, 3, 128, 129]:
    for s in (np.float32(0), np.float32(0.5), np.float32(0.9), np.float32(0.99), np.float32(rng.rand())):
      k = pruning.keep_count(int(n), s)
      assert k == oracle.keep(int(n), s) and 1 <= k <= n


@pytest.mark.parametrize('bad', ['target_sparsity0.9', 'target_sparsity=0.9,stray', 'begin_pruning_step=1 2',
                                 'weight_sparsity_map=[a:0.1', '=3', 'threshold_decay=x'])
def test_hparams_parse_rejects_malformed(bad):
  with pytest.raises(ValueError):
    pruning.get_pruning_hparams().parse(bad)


def test_hparams_copy_and_pickle():
  import copy
  import pickle
  hp = _spec(*CIFAR)
  for other in (copy.deepcopy(hp), pickle.loads(pickle.dumps(hp))):
    assert other.values() == hp.values()
  assert not hasattr(hp, 'no_such_hparam')


@pytest.mark.parametrize('initial,target', [(0.1, 0.9), (0.3, 0.5), (0.45, 0.8), (0.15, 0.98)])
def test_sparsity_initial_minus_target_is_one_constant(initial, target):
  """(initial - target) is rounded to float32 once, after the subtraction (these pairs differ from
  f32(initial) - f32(target))."""
  assert np.float32(initial - target) != np.float32(initial) - np.float32(target)
  hp = pruning.get_pruning_hparams().parse('initial_sparsity=%r,target_sparsity=%r' % (initial, target))
  p = _pruning(hp)
  for gs in range(0, 101, 7):
    assert p.sparsity(gs).tobytes() == oracle.sparsity(gs, initial, target, 0, 100, 3).tobytes(), gs
  f = np.float32
  decay = f(np.float64(f(1)) ** 3)
  assert p.sparsity(0) == f(f(initial - target) * decay + f(target))
