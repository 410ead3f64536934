"""CPU-side argument checks of disco_stft_filter_dual and of the optional spectrum of disco_stft_scm2: bad sizes,
shapes outside the kernel's coverage and null pointers are rejected before any CUDA work."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_stft_filter_dual_argument_validation(lib):
    p = ctypes.c_void_p(16)          # never dereferenced: every call below fails validation first
    f = lib.disco_stft_filter_dual
    #         x  W1 W2 z  zn yf ref lay G  C  L     n_fft
    assert f(p, p, p, p, p, p, 0, 0, 1, 4, 4000, 500, None) == -1        # n_fft
    assert b"n_fft" in lib.disco_last_error()
    assert f(p, p, p, p, p, p, 0, 0, 1, 4, 4000, 1024, None) == -2       # two-mask coverage: n_fft 256 / 512
    assert f(p, p, p, p, p, p, 0, 0, 1, 5, 4000, 512, None) == -2        # C <= 4
    assert f(p, p, p, p, p, p, 0, 0, 1, 0, 4000, 512, None) == -2
    assert f(p, p, p, p, p, p, 0, 0, 0, 4, 4000, 512, None) == -1        # no groups
    assert f(p, p, p, p, p, p, 0, 0, 1, 4, 200, 512, None) == -1         # too short for the reflect padding
    assert f(p, p, p, p, p, p, 4, 0, 1, 4, 4000, 512, None) == -1        # ref out of range
    assert b"ref" in lib.disco_last_error()
    assert f(p, p, p, p, p, p, -1, 0, 1, 4, 4000, 512, None) == -1
    assert f(p, p, p, p, p, p, 0, 2, 1, 4, 4000, 512, None) == -1        # neither TF nor FT
    assert b"out_layout" in lib.disco_last_error()
    for i in (0, 1, 2, 3, 5):                                          # x, W1, W2, z, yf; zn may be null
        args = [p] * 6
        args[i] = None
        assert f(*args, 0, 0, 1, 4, 4000, 512, None) == -1, i
        assert b"null" in lib.disco_last_error()


def test_spectrum_stays_required_outside_the_two_mask_pass(lib):
    # only disco_stft_scm2 may skip the spectrum (its GPU test covers Y = NULL); the plain and the single-mask
    # STFT still reject a missing output
    p = ctypes.c_void_p(16)
    assert lib.disco_stft(p, None, 4, 4000, 512, None) == -1
    assert b"null" in lib.disco_last_error()
    assert lib.disco_stft_scm(p, p, 0, None, None, None, 1, 4, 4000, 512, p, 1 << 30, None) == -1
    assert b"null" in lib.disco_last_error()
