"""Weight masks that kill whole 64 x 64 (ci, co) tiles of a tap, in plain numpy.

The packed operands carry one survivor count per 64 x 64 tile of each tap (pack.cu); the K-major conv kernels
skip the load and the MMA of every K block whose tiles are all zero (igemm_tc.cu, `weight_block_live`).  Uniformly
random masks practically never produce an all-zero tile, so these patterns decide tile liveness explicitly and keep
a random mask inside the live tiles.  Tile (tap, kt, nt) covers input channels 64 kt .. 64 kt + 63 and output
channels 64 nt .. 64 nt + 63 of filter tap `tap` (row-major over kh, kw).
"""
import numpy as np


def tile_counts(mask):
  """Survivor count of every 64 x 64 tile, indexed [tap][co tile][ci tile] like the packed table.  `mask` is HWIO
  or [in, out]."""
  cin, cout = mask.shape[-2:]
  m = (np.asarray(mask) != 0).reshape(-1, cin, cout)
  kt, nt = -(-cin // 64), -(-cout // 64)
  pad = np.zeros((m.shape[0], kt * 64, nt * 64), np.int64)
  pad[:, :cin, :cout] = m
  return pad.reshape(m.shape[0], kt, 64, nt, 64).sum(axis=(2, 4)).transpose(0, 2, 1)


def live_tiles(pattern, taps, k_tiles, n_tiles):
  """bool [tap][kt][nt]: which tiles `pattern` keeps."""
  tap, kt, nt = np.meshgrid(np.arange(taps), np.arange(k_tiles), np.arange(n_tiles), indexing='ij')
  if pattern == 'staircase':         # different ci and co tile counts: a transposed table lookup skips live tiles
    return ~(kt > nt)
  if pattern == 'staircase_t':       # the transpose: long reductions over co (dgrad) with few live K blocks
    return ~(nt > kt)
  if pattern == 'block0':            # every K block but the first (tap 0, ci tile 0) dead
    return (tap == 0) & (kt == 0)
  if pattern == 'block0_dead':       # only the first K block dead
    return ~((tap == 0) & (kt == 0))
  if pattern == 'half':              # one half of every 128-wide N tile dead; which one alternates with the K block
    return (kt + nt) % 2 == 1
  if pattern == 'dead_taps':         # even taps (corners and centre of a 3x3) dead
    return tap % 2 == 1
  if pattern == 'one_tap':           # every tap but one dead (tap 5 = (kh 1, kw 2) of a 3x3)
    return tap == min(5, taps - 1)
  if pattern == 'dead':              # whole layer
    return np.zeros_like(tap, bool)
  raise ValueError(pattern)


PATTERNS = ('staircase', 'staircase_t', 'block0', 'block0_dead', 'half', 'dead_taps', 'one_tap', 'dead', 'corner')


def tile_mask(pattern, shape, rng, sparsity=0.5):
  """float32 mask of `shape` (HWIO or [in, out]): random at `sparsity` inside the tiles `pattern` keeps, zero in the
  others.  'corner' keeps exactly one weight: (last tap, cin - 1, cout - 1)."""
  cin, cout = shape[-2:]
  taps = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
  if pattern == 'corner':
    m = np.zeros((taps, cin, cout), np.float32)
    m[-1, -1, -1] = 1
    return m.reshape(shape)
  live = live_tiles(pattern, taps, -(-cin // 64), -(-cout // 64))
  keep = live.repeat(64, axis=1).repeat(64, axis=2)[:, :cin, :cout]
  rand = (rng.random_sample((taps, cin, cout)) >= sparsity)
  return (keep & rand).astype(np.float32).reshape(shape)


# (n, h, w, cin, cout, k, stride, sparsity inside live tiles[, padding]), pattern.  Channel counts > 64 (or a
# stride of 2) keep 3x3 layers off the halo kernels, which ignore the table -- except the last case, which is a
# halo layer on purpose.  n and the pixel grids give two or more 128-pixel M tiles.
STRUCTURED_CONV_CASES = [
    ((3, 8, 8, 192, 320, 3, 1, 0.5), 'staircase'),        # 3 vs 5 tile counts; the last 128-wide N tile is half past N
    ((3, 8, 8, 320, 192, 3, 1, 0.5), 'staircase'),
    ((3, 8, 8, 192, 192, 3, 1, 0.5), 'staircase'),
    ((3, 8, 8, 192, 256, 3, 1, 0.5), 'block0'),
    ((3, 8, 8, 256, 192, 3, 1, 0.5), 'block0_dead'),
    ((3, 8, 8, 256, 256, 3, 1, 0.5), 'half'),
    ((4, 9, 9, 256, 192, 1, 2, 0.5), 'half'),
    ((4, 16, 16, 128, 192, 3, 2, 0.5), 'dead_taps'),      # dgrad parity classes whose taps are all dead
    ((4, 16, 16, 192, 128, 3, 2, 0.5, 'SAME'), 'dead_taps'),
    ((4, 15, 15, 128, 128, 3, 2, 0.5), 'one_tap'),
    ((4, 16, 16, 128, 136, 3, 2, 0.5, 'SAME'), 'one_tap'),
    ((3, 8, 8, 128, 192, 3, 1, 0.5), 'dead'),
    ((3, 8, 8, 200, 136, 3, 1, 0.5), 'corner'),
    ((2, 14, 14, 64, 64, 3, 1, 0.5), 'dead_taps'),        # halo kernels
]

# (rows, n_in, units, sparsity), pattern: the liveness mask covers at most 320 (tap, K block) pairs
# (igemm_tc.cu, kLiveWords); a K of 20480 = 320 blocks still skips dead blocks, 20544 = 321 loads all of them.
# fprop reduces over n_in, dgrad over units.  192 rows = two M tiles.
STRUCTURED_LINEAR_CASES = [
    ((192, 20480, 128, 0.5), 'staircase'),
    ((192, 20544, 128, 0.5), 'staircase'),
    ((192, 128, 20480, 0.5), 'staircase_t'),
    ((192, 128, 20544, 0.5), 'staircase_t'),
]
