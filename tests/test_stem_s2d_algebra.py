"""Index algebra of the (experimental) space-to-depth stem kernels, checked on the CPU against the
oracle's direct convolution: the 2x2 input fold, the [16 taps][cout][16] weight operand, the tap ->
halo-row offsets and the partial -> HWIO scatter of the wgrad reduce are restated here in numpy
exactly as rigl_b200/csrc/stem_s2d.cuh indexes them (k_stem_s2d_fold / _pack / _fprop / _wgrad /
_reduce).  This pins the MATH of that path; the hardware layout (SWIZZLE_32B tiles, row-shifted ldmatrix
loads) is checked on the device by tests/test_conv_gpu.py::test_conv_stem_s2d_path."""
import numpy as np
import pytest

from oracle import rigl_oracle as orc

KS, STRIDE, PAD, WP = 7, 2, 3, 128


def fold(x):
  """x [N,H,W,cin<=3] -> xs [N,HS,WS,16]   (k_stem_s2d_fold)"""
  n, h, w, cin = x.shape
  hs, ws = (h + 2 * PAD) // 2, (w + 2 * PAD) // 2
  xs = np.zeros((n, hs, ws, 16), x.dtype)
  for hy in range(hs):
    for wx in range(ws):
      for dy in range(2):
        for dx in range(2):
          hi, wi = 2 * hy + dy - PAD, 2 * wx + dx - PAD
          if 0 <= hi < h and 0 <= wi < w:
            xs[:, hy, wx, (dy * 2 + dx) * 3:(dy * 2 + dx) * 3 + cin] = x[:, hi, wi, :]
  return xs


def pack(w, mask):
  """HWIO [7,7,cin,cout] (+mask) -> [16 taps][cout][16]   (k_stem_s2d_pack)"""
  cin, cout = w.shape[2], w.shape[3]
  out = np.zeros((16, cout, 16), w.dtype)
  for tap in range(16):
    th, tw = tap // 4, tap % 4
    for k16 in range(12):
      q, c = k16 // 3, k16 % 3
      kh, kw = 2 * th + (q >> 1), 2 * tw + (q & 1)
      if c < cin and kh < KS and kw < KS:
        out[tap, :, k16] = w[kh, kw, c, :] * mask[kh, kw, c, :]
  return out


def halo_rows(xs, n, h0, rows):
  """The halo tile of folded rows h0 .. h0+rows-1 as a flat [rows*WP, 16] matrix (TMA OOB zero fill)."""
  hs, ws = xs.shape[1], xs.shape[2]
  t = np.zeros((rows, WP, 16), xs.dtype)
  for r in range(rows):
    if h0 + r < hs:
      t[r, :min(ws, WP)] = xs[n, h0 + r, :min(ws, WP)]
  return t.reshape(rows * WP, 16)


@pytest.mark.parametrize('shape', [(2, 16, 12, 3, 8), (1, 8, 20, 3, 16), (2, 12, 12, 1, 8)])
def test_s2d_forward_and_wgrad_algebra(shape):
  n, h, w, cin, cout = shape
  rng = np.random.RandomState(h * 31 + w)
  x = rng.standard_normal((n, h, w, cin))
  wt = rng.standard_normal((KS, KS, cin, cout))
  mask = (rng.rand(KS, KS, cin, cout) > 0.3).astype(np.float64)
  ho, wo = h // 2, w // 2
  y_want = orc.conv2d_nhwc_general(x, wt * mask, STRIDE, PAD, (ho, wo))
  xs, bs = fold(x), pack(wt, mask)
  # ---- forward: M tile t = output row h0 + t, tap (th, tw) starts (t + th)*WP + tw rows into the halo tile
  R = 4
  y = np.zeros((n, ho, wo, cout))
  for img in range(n):
    for h0 in range(0, ho, R):
      tile = halo_rows(xs, img, h0, R + 3)
      tile = np.concatenate([tile, np.zeros((8, 16))])              # slack rows
      for t in range(min(R, ho - h0)):
        acc = np.zeros((WP, cout))
        for tap in range(16):
          row = (t + tap // 4) * WP + tap % 4
          acc += tile[row:row + WP] @ bs[tap].T
        y[img, h0 + t] = acc[:wo]                                    # columns >= W are clipped by the TMA store
  assert np.allclose(y, y_want, rtol=1e-10, atol=1e-10)
  # ---- wgrad: accumulator th holds D[atom*16 + k16][co] = sum_pos xs[pos + th*WP + atom][k16] * dy[pos][co]
  dy = rng.standard_normal((n, ho, wo, cout))
  _, dw_want = orc.conv2d_nhwc_general_bwd(x, wt * mask, dy, STRIDE, PAD)
  part = np.zeros((4, 128, cout))
  Rw = 2
  for img in range(n):
    for h0 in range(0, ho, Rw):
      tile = np.concatenate([halo_rows(xs, img, h0, Rw + 3), np.zeros((8, 16))])
      dyt = np.zeros((Rw, WP, cout))
      for r in range(min(Rw, ho - h0)):
        dyt[r, :wo] = dy[img, h0 + r]                                # padding columns / rows zero-filled
      dyt = dyt.reshape(Rw * WP, cout)
      for th in range(4):
        for atom in range(8):
          a = tile[th * WP + atom: th * WP + atom + Rw * WP]         # [positions, 16]
          part[th, atom * 16:(atom + 1) * 16] += a.T @ dyt
  dw = np.zeros_like(wt)
  for kh in range(KS):
    for kw in range(KS):
      for c in range(cin):
        row = (kw >> 1) * 16 + ((kh & 1) * 2 + (kw & 1)) * 3 + c     # k_stem_s2d_reduce
        dw[kh, kw, c] = part[kh >> 1, row]
  assert np.allclose(dw, dw_want, rtol=1e-10, atol=1e-9)
