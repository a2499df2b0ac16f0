"""The structured weight masks of the conv / linear GPU tests (tile_masks.py) really produce the dead 64 x 64 tiles
those tests exist for.  Runs without a GPU: it checks the masks and a numpy model of which K blocks the kernels
skip, so the GPU tests cannot silently turn into tests of uniformly live weights."""
import numpy as np
import pytest

from tile_masks import (PATTERNS, STRUCTURED_CONV_CASES, STRUCTURED_LINEAR_CASES, live_tiles, tile_counts,
                        tile_mask)

_LIVE_WORDS = 10        # igemm_tc.cu kLiveWords: liveness of at most 320 (tap, K block) pairs


def _block_live(counts, n_out, taps=None, dgrad=False, first_half_only=False, transposed=False):
  """Model of build_live_mask / weight_block_live (igemm_tc.cu): bool [N tile][tap][K block].  fprop reduces over
  ci tiles, dgrad over co tiles; an N tile is 128 wide when n_out > 64 and is live if either 64-wide half is; the
  first (tap, K block) is always live.  `first_half_only` / `transposed` model a broken lookup."""
  t = counts.transpose(0, 2, 1) if dgrad else counts            # -> [tap][N-direction tile][K-direction tile]
  if transposed:
    assert t.shape[1] == t.shape[2]
    t = t.transpose(0, 2, 1)
  taps = list(range(counts.shape[0])) if taps is None else list(taps)
  bn64 = 2 if n_out > 64 else 1
  n64 = -(-n_out // 64)
  live = np.zeros((-(-n64 // bn64), len(taps), t.shape[2]), bool)
  for n in range(live.shape[0]):
    nts = [n * bn64 + j for j in range(1 if first_half_only else bn64) if n * bn64 + j < n64]
    for i, tap in enumerate(taps):
      live[n, i] = t[tap, nts].sum(axis=0) > 0
  live[:, 0, 0] = True
  return live


def _mask(case, pattern, linear=False):
  shape = case[1:3] if linear else (case[5], case[5], case[3], case[4])
  return tile_mask(pattern, shape, np.random.RandomState(0), case[3] if linear else case[7])


def _halo(case):
  n, h, w, cin, cout, k, stride = case[:7]
  return k == 3 and stride == 1 and cin <= 64 and cout <= 64


def test_every_pattern_is_used():
  used = {p for _, p in STRUCTURED_CONV_CASES + STRUCTURED_LINEAR_CASES}
  assert used == set(PATTERNS)


@pytest.mark.parametrize('case,pattern', STRUCTURED_CONV_CASES + STRUCTURED_LINEAR_CASES)
def test_pattern_has_dead_and_live_tiles(case, pattern):
  linear = len(case) == 4
  m = _mask(case, pattern, linear)
  counts = tile_counts(m)
  if pattern == 'dead':
    assert not m.any()
    return
  assert (counts == 0).any() and (counts > 0).any(), (case, pattern)
  if pattern == 'corner':
    assert m.sum() == 1 and m.reshape(-1, *m.shape[-2:])[-1, -1, -1] == 1
    return
  want = live_tiles(pattern, counts.shape[0], counts.shape[2], counts.shape[1]).transpose(0, 2, 1)
  assert np.array_equal(counts > 0, want), 'a tile the pattern keeps has no survivor'


@pytest.mark.parametrize('case,pattern', [c for c in STRUCTURED_CONV_CASES if not _halo(c[0]) and
                                          c[1] not in ('half', 'block0_dead')] + STRUCTURED_LINEAR_CASES)
def test_kernels_skip_blocks_of_every_generic_case(case, pattern):
  """Every case that runs on the K-major kernels has K blocks the kernels skip, in fprop or dgrad.  ('half' keeps one
  live half in every 128-wide tile and 'block0_dead' only kills the always-live first block, so with a correct
  lookup neither skips anything.)"""
  linear = len(case) == 4
  m = _mask(case, pattern, linear)
  counts = tile_counts(m)
  cin, cout = m.shape[-2:]
  fwd, bwd = _block_live(counts, cout), _block_live(counts, cin, dgrad=True)
  assert not (fwd.all() and bwd.all()), (case, pattern)


def test_staircase_transposed_lookup_skips_a_live_block():
  """A dgrad that read the survivor table transposed would skip a live K block (equal tile counts, so the
  transposed index stays inside the table)."""
  case = [c for c, p in STRUCTURED_CONV_CASES if p == 'staircase' and c[3] == c[4]][0]
  counts = tile_counts(_mask(case, 'staircase'))
  for dgrad in (False, True):
    right = _block_live(counts, case[3], dgrad=dgrad)
    wrong = _block_live(counts, case[3], dgrad=dgrad, transposed=True)
    assert (right & ~wrong).any(), dgrad


@pytest.mark.parametrize('case', [c for c, p in STRUCTURED_CONV_CASES if p == 'half'])
def test_half_pattern_has_blocks_live_only_in_the_second_half(case):
  counts = tile_counts(_mask(case, 'half'))
  for n_out, dgrad in ((case[4], False), (case[3], True)):
    right = _block_live(counts, n_out, dgrad=dgrad)
    wrong = _block_live(counts, n_out, dgrad=dgrad, first_half_only=True)
    assert (right & ~wrong).any(), dgrad


@pytest.mark.parametrize('case', [c for c, p in STRUCTURED_CONV_CASES if p in ('dead_taps', 'one_tap') and c[6] == 2])
def test_stride2_dead_taps_leave_a_dgrad_parity_class_without_live_taps(case):
  """tc_dgrad runs one launch per input parity class over the taps that reach it: some class sees only dead
  taps (all its blocks skipped but the first), another sees live ones."""
  pattern = [p for c, p in STRUCTURED_CONV_CASES if c == case][0]
  n, h, w, cin, cout, k, stride = case[:7]
  padding = case[8] if len(case) > 8 else 'FIXED'
  pad = (max((-(-h // 2) - 1) * 2 + k - h, 0) // 2) if padding == 'SAME' else (k - 1) // 2
  counts = tile_counts(_mask(case, pattern))
  any_dead = any_live = False
  for ph in range(2):
    for pw in range(2):
      taps = [kh * k + kw for kh in range(k) for kw in range(k) if (ph + pad - kh) % 2 == 0 and (pw + pad - kw) % 2 == 0]
      live = _block_live(counts, cin, taps=taps, dgrad=True)
      any_dead |= live.sum() == live.shape[0]         # only the always-live first block of every N tile
      any_live |= live.sum() > live.shape[0]
  assert any_dead and any_live


def test_linear_cases_straddle_the_liveness_cap():
  """fprop K = n_in and dgrad K = units reach 320 blocks (skipping on) and 321 (skipping off)."""
  fwd = {c[1] // 64 for c, _ in STRUCTURED_LINEAR_CASES}
  bwd = {c[2] // 64 for c, _ in STRUCTURED_LINEAR_CASES}
  assert {32 * _LIVE_WORDS, 32 * _LIVE_WORDS + 1} <= fwd and {32 * _LIVE_WORDS, 32 * _LIVE_WORDS + 1} <= bwd
  for case, pattern in STRUCTURED_LINEAR_CASES:
    counts = tile_counts(_mask(case, pattern, linear=True))
    long_k_fprop = case[1] > case[2]
    live = _block_live(counts, case[2]) if long_k_fprop else _block_live(counts, case[1], dgrad=True)
    assert live.mean() < 0.1, (case, pattern)        # the long reduction is almost all dead blocks
