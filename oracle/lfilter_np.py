"""NumPy restatement of ``scipy.signal.lfilter`` (direct form II transposed, float64) over a plane of
(signal, band) filters -- TEST INFRASTRUCTURE, see oracle/__init__.py.

scipy's inner loop (``_linear_filter`` / ``DOUBLE_filt``) per sample, after normalising b and a by a[0]:
    y       = z[0] + b[0] * x
    z[i]    = (z[i+1] + x * b[i+1]) - y * a[i+1]      i = 0 .. n - 3
    z[n-2]  = x * b[n-1] - y * a[n-1]
Each operation is one float64 ufunc here, in that order, so every product and sum is rounded on its own exactly
as in scipy's C loop (no fused multiply-add).  `csrc/filterbank.cu` evaluates the same sequence with
`__dmul_rn` / `__dadd_rn` / `__dsub_rn`, so its outputs are bit-identical to these.

`fma=True` gives the contracted recurrence (y = fma(b0, x, z0), z_i = fma(-y, a_{i+1}, fma(x, b_{i+1}, z_{i+1})))
that a compiler allowed to contract would produce: a wrong kernel for the tests to reject.
"""
import numpy as np


def _fma(a, b, c):
    """a * b + c with the product unrounded, as a fused multiply-add.  Dekker's TwoProduct gives p + e = a * b
    exactly, TwoSum gives s + t = p + c exactly, and s + (t + e) rounds the rest: the correctly rounded fma except in
    rare double-rounding corner cases, far fewer than the bit differences a contracted recurrence makes."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    p = a * b
    split = 134217729.0            # 2^27 + 1
    ah = a * split; ah = ah - (ah - a); al = a - ah
    bh = b * split; bh = bh - (bh - b); bl = b - bh
    e = ((ah * bh - p) + ah * bl + al * bh) + al * bl
    s = p + c
    bb = s - p
    t = (p - (s - bb)) + (c - bb)
    return s + (t + e)


def lfilter_plane(b, a, x, fma=False):
    """y[s, k, n] = lfilter(b[k], a[k], x[s]).  b, a [n_band, NC] float64; x [n_sig, L] (any float dtype; widened to
    float64 as scipy does) -> y [n_sig, n_band, L] float64."""
    b = np.asarray(b, np.float64)
    a = np.asarray(a, np.float64)
    x = np.asarray(x).astype(np.float64)
    n_band, nc = b.shape
    a0 = a[:, :1]
    bn, an = b / a0, a / a0                       # normalise by a[0], one division per coefficient
    n_sig, L = x.shape
    z = np.zeros((nc - 1, n_sig, n_band))
    y = np.empty((n_sig, n_band, L))
    for n in range(L):
        xn = x[:, n:n + 1]                        # [n_sig, 1] broadcast over bands
        if fma:
            yn = _fma(bn[:, 0], xn, z[0])
            for i in range(nc - 2):
                z[i] = _fma(-yn, an[:, i + 1], _fma(xn, bn[:, i + 1], z[i + 1]))
            z[nc - 2] = _fma(-yn, an[:, nc - 1], xn * bn[:, nc - 1])
        else:
            yn = z[0] + bn[:, 0] * xn
            for i in range(nc - 2):
                z[i] = (z[i + 1] + xn * bn[:, i + 1]) - yn * an[:, i + 1]
            z[nc - 2] = xn * bn[:, nc - 1] - yn * an[:, nc - 1]
        y[:, :, n] = yn
    return y


def band_stats(b, a, x, sel=None, fma=False):
    """The statistics `disco_band_stats` returns, restated: count, sequential sum and sum of squares of the outputs
    lfilter_plane(b, a, x) that are selected (sel != 0, or output != 0 without sel).  -> [n_sig, n_band, 3] float64;
    the sum is np.cumsum's left-to-right order, the squares are summed the same way (the kernel fuses them with
    fma, so they agree to 2 n 2^-53 relative, not bit for bit)."""
    y = lfilter_plane(b, a, x, fma=fma)
    take = (y != 0.0) if sel is None else np.broadcast_to((np.asarray(sel) != 0)[:, None, :], y.shape)
    v = np.where(take, y, 0.0)
    out = np.empty(y.shape[:2] + (3,))
    out[..., 0] = take.sum(-1)
    out[..., 1] = np.cumsum(v, axis=-1)[..., -1] if y.shape[-1] else 0.0
    out[..., 2] = np.cumsum(v * v, axis=-1)[..., -1] if y.shape[-1] else 0.0
    return out
