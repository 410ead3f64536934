"""STOI without a device: the float64 oracle (pystoi 0.3's algorithm, oracle/stoi_np.py) against its literal loop form
and STOI's defining properties, the resampler and band design of disco_b200/stoi.py against the oracle's, and the
argument checks of the compat layer and of the C ABI."""
import os
import re
from fractions import Fraction

import numpy as np
import pytest

from oracle import stoi_np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def speechlike(seed, L, period=4000, noise=0.0):
    """Gated low-passed noise (on 60 % of every period) plus optional white noise, float32-representable float64."""
    rng = np.random.default_rng(seed)
    x = np.convolve(rng.standard_normal(L + 31), np.hanning(32), mode="valid")[:L]
    x *= (np.arange(L) % period) < 0.6 * period
    x += noise * rng.standard_normal(L)
    return x.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize("L,period,noise", [(20000, 4000, 0.3), (30123, 2500, 1.0), (25600, 6000, 0.05)])
def test_loop_form_equals_vectorised(L, period, noise):
    x = speechlike(L, L, period)
    y = x + speechlike(L + 1, L, 1 << 30, noise)
    a = stoi_np.stoi_10k(x, y)
    b = stoi_np.stoi_loop(x, y)
    assert abs(a - b) <= 1e-12, (a, b)
    assert 0.0 < a < 1.0


def test_defining_properties():
    x = speechlike(1, 30000)
    y = x + speechlike(2, 30000, 1 << 30, 0.5)
    assert abs(stoi_np.stoi_10k(x, x) - 1.0) <= 1e-12
    d = stoi_np.stoi_10k(x, y)
    for cx, cy in ((2.0, 1.0), (1.0, 0.25), (8.0, 0.5)):    # powers of two: the scaled signals are exact
        assert abs(stoi_np.stoi_10k(cx * x, cy * y) - d) <= 1e-12
    assert stoi_np.stoi_10k(x, np.zeros_like(x)) == 0.0


def test_too_few_frames_and_too_short():
    x = speechlike(3, 128 * 30 + 256, 1 << 30)     # 31 frames, all loud: 30 STFT frames
    y = x + speechlike(4, len(x), 1 << 30, 0.5)
    assert len(stoi_np.selection(x)) == 31 and stoi_np.stoi_10k(x, y) != 1e-5
    x2, y2 = x[:-128], y[:-128]               # 29 STFT frames
    with pytest.warns(RuntimeWarning):
        assert stoi_np.stoi_10k(x2, y2) == 1e-5
    with pytest.raises(ValueError):
        stoi_np.stoi_10k(x[:255], y[:255])
    with pytest.raises(Exception):
        stoi_np.stoi(x, y[:-1], 10000)


@pytest.mark.parametrize("fs,taps", [(16000, 581), (8000, 365), (48000, 1741), (44100, 31947), (22050, 31947)])
def test_resampler_taps(fs, taps):
    from disco_b200 import stoi
    h = stoi_np.resample_window_oct(10000, fs)
    assert len(h) == taps
    np.testing.assert_array_equal(h, h[::-1])
    assert abs(np.sum(h / np.sum(h)) - 1.0) <= 1e-15
    got, up, down = stoi.resample_taps(fs)
    np.testing.assert_array_equal(got, h / np.sum(h))                    # bit for bit
    g = np.gcd(10000, fs)
    assert (up, down) == (10000 // g, fs // g)


def nearest_bin(f_hz):
    """First bin k (at k 10000 / 512 Hz) nearest to f_hz, in exact arithmetic on the decimal frequency."""
    pos = Fraction(f_hz) * 512 / 10000
    k = int(pos)
    return k if pos - k <= Fraction(1, 2) else k + 1


def test_band_table():
    want = [(7, 9), (9, 11), (11, 14), (14, 17), (17, 22), (22, 27), (27, 34), (34, 43), (43, 55), (55, 69), (69, 87),
            (87, 109), (109, 138), (138, 174), (174, 219)]
    indep = [(nearest_bin(150 * 2 ** ((2 * i - 1) / 6)), nearest_bin(150 * 2 ** ((2 * i + 1) / 6))) for i in range(15)]
    assert indep == want
    assert stoi_np.band_edges() == want
    from disco_b200 import stoi
    assert stoi.band_edges() == want
    src = open(os.path.join(ROOT, "disco_b200", "csrc", "stoi.cu")).read()
    edges = [int(v) for v in re.search(r"kStoiEdges\[[^\]]*\] = \{([^}]*)\}", src).group(1).split(",")]
    assert list(zip(edges[:-1], edges[1:])) == want


def test_compat_errors_without_device():
    from disco_b200.compat import stoi
    with pytest.raises(Exception, match="same length"):
        stoi.stoi(np.ones(1000), np.ones(999), 16000)
    with pytest.raises(NotImplementedError):
        stoi.stoi(np.ones(1000), np.ones(1000), 16000, extended=True)


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_abi_validation_and_workspace(lib):
    fake = 16
    assert lib.disco_stoi(fake, fake, fake, fake, fake, fake, 0, 1, 1, 1000, fake, 1 << 30, None) == -1   # no clean
    assert lib.disco_stoi(fake, fake, fake, fake, fake, fake, 1, 0, 1, 1000, fake, 1 << 30, None) == -1   # no degraded
    assert lib.disco_stoi(fake, fake, fake, fake, fake, fake, 1, 1, 0, 1000, fake, 1 << 30, None) == -1   # no pair
    assert lib.disco_stoi(fake, fake, fake, fake, fake, fake, 1, 1, 1, 255, fake, 1 << 30, None) == -1    # < 256
    assert b"256" in lib.disco_last_error()
    assert lib.disco_stoi(None, fake, fake, fake, fake, fake, 1, 1, 1, 1000, fake, 1 << 30, None) == -1
    assert lib.disco_stoi_workspace(1, 1, 255) == 0
    assert lib.disco_stoi_workspace(0, 1, 1000) == 0
    # energies + kept-frame lists per clean, band envelopes per clean and per pair
    C, P, L = 3, 7, 90000
    n_fr = (L - 256) // 128 + 1
    want = n_fr * (C * (8 + 4) + (C + P) * 15 * 8)
    assert lib.disco_stoi_workspace(C, P, L) == want
    assert lib.disco_stoi_workspace(1, 1, 256) == 1 * (12 + 2 * 120)
    # a device pointer is never touched before the size checks: a too-small workspace fails first
    assert lib.disco_stoi(fake, fake, fake, fake, fake, fake, C, 2, P, L, fake, want - 1, None) == -3
    assert lib.disco_resample_poly(fake, fake, fake, 0, 5, 8, 1, 100, None) == -1     # no taps
    assert lib.disco_resample_poly(fake, fake, fake, 5, 0, 8, 1, 100, None) == -1     # up = 0
    assert lib.disco_resample_poly(fake, fake, fake, 5, 10, 16, 1, 100, None) == -1   # not reduced
    assert lib.disco_resample_poly(fake, fake, fake, 5, 1, 1, 1, 100, None) == -1     # nothing to resample
    assert lib.disco_resample_poly(fake, fake, fake, 5, 5, 8, 1, 0, None) == -1       # empty signals
    assert lib.disco_resample_poly(None, fake, fake, 5, 5, 8, 1, 100, None) == -1
    assert lib.disco_resample_poly(fake, fake, fake, 5, 1 << 20, 1, 1, 1 << 12, None) == -1   # 2^32 outputs
