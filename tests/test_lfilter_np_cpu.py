"""oracle/lfilter_np.py (scipy's lfilter DF2T restated one ufunc per operation) against scipy.signal.lfilter on the
third-octave banks of post at filter orders 2, 4, 8 and 16: bit for bit, because the kernel that the GPU tests hold to
this restatement follows scipy's rounding sequence."""
import numpy as np
import pytest
from scipy.signal import lfilter

from disco_b200 import post
from oracle import lfilter_np


def bank(order, fs=16000, scale=1.0):
    F, _ = post.third_octave_bands(fs)
    b, a = post.third_octave_filterbank(F, fs, order=order // 2)
    return b * scale, a * scale


@pytest.mark.parametrize("order", [2, 4, 8, 16])
@pytest.mark.parametrize("scale", [1.0, 3.7])
def test_lfilter_plane_bit_equal_to_scipy(order, scale):
    rng = np.random.default_rng(order)
    x = rng.standard_normal((3, 700)).astype(np.float32)
    x[1, :50] = 0.0                               # an exactly zero prefix
    b, a = bank(order, scale=scale)
    got = lfilter_np.lfilter_plane(b, a, x)
    for s in range(x.shape[0]):
        for k in range(b.shape[0]):
            want = lfilter(b[k], a[k], x[s].astype(np.float64))
            np.testing.assert_array_equal(got[s, k], want, err_msg="signal %d band %d" % (s, k))


def test_contracted_recurrence_differs():
    """The fma variant is the negative control of the GPU tests: it must not coincide with scipy's sequence."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 400)).astype(np.float32)
    b, a = bank(8)                                # fw_snr's bank; bands 160 and 200 Hz
    exact = lfilter_np.lfilter_plane(b[:2], a[:2], x)
    fused = lfilter_np.lfilter_plane(b[:2], a[:2], x, fma=True)
    assert not np.array_equal(exact, fused)
    assert np.abs(exact - fused).max() <= 1e-3 * np.abs(exact).max()   # a rounding-level change, amplified


def test_fma_emulation_rounds_once():
    rng = np.random.default_rng(2)
    a, b, c = rng.standard_normal((3, 10000))
    got = lfilter_np._fma(a, b, c)
    from fractions import Fraction
    for i in range(0, 10000, 97):
        exact = Fraction(a[i]) * Fraction(b[i]) + Fraction(c[i])
        assert got[i] == float(exact), i
    # a case where separate rounding loses the low part of the product entirely
    x = 1.0 + 2.0 ** -30
    assert lfilter_np._fma(x, x, -(x * x)) == 2.0 ** -60


def test_band_stats_restatement():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((2, 300)).astype(np.float32)
    x[0, :40] = 0.0
    sel = (rng.uniform(size=x.shape) > 0.5).astype(np.float32)
    b, a = bank(4)
    y = lfilter_np.lfilter_plane(b, a, x)
    for s_ in (None, sel):
        st = lfilter_np.band_stats(b, a, x, s_)
        take = (y != 0) if s_ is None else np.broadcast_to(s_[:, None, :] != 0, y.shape)
        np.testing.assert_array_equal(st[..., 0], take.sum(-1))
        assert st[0, 0, 0] == (300 - 40 if s_ is None else take[0, 0].sum())
        for s in range(2):
            for k in range(b.shape[0]):
                acc = 0.0
                for v in y[s, k][take[s, k]]:
                    acc += v
                assert st[s, k, 1] == acc
