"""CPU-side checks of the length-aware online (recursive) interface: disco_scm_recursive_lengths and
disco_filter_sum_blocks_lengths reject bad frame counts, null pointers and too-wide stacks before any CUDA work, and
online_tango validates `lengths` with the usual exception types before touching a tensor."""
import ctypes

import numpy as np
import pytest
import torch

DISCO_ERR_INVALID, DISCO_ERR_UNSUPPORTED = -1, -2
DUMMY = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def _host(vals):
    return (ctypes.c_int * len(vals))(*vals)


def _rec(lib, frames, frames_host, K=2, C=2, T=30, block=8, Y=DUMMY, Rss=DUMMY, n_utt=3):
    #                                      Y  Z      mask   R0s   R0n   Rss  Rnn    lambda block pow
    return lib.disco_scm_recursive_lengths(Y, DUMMY, DUMMY, None, None, Rss, DUMMY, 0.9, block, 2,
                                           n_utt, K, C, T, 512, None, 0, frames, frames_host, None)


def _filt(lib, frames, frames_host, K=2, C=2, T=30, W=DUMMY, out=DUMMY, n_utt=3):
    #                                          W  conj Y      Z      out  resid  ref block lag
    return lib.disco_filter_sum_blocks_lengths(W, 1, DUMMY, DUMMY, out, DUMMY, 0, 8, 1,
                                               n_utt, K, C, T, 512, None, 0, frames, frames_host, None)


@pytest.mark.parametrize("call", [_rec, _filt])
def test_frame_counts_checked_before_launch(lib, call):
    ok = _host([30, 1, 17])
    for bad in ([30, 0, 17], [31, 5, 5], [30, -1, 30]):          # T_b = 0, T_b > T, negative
        assert call(lib, DUMMY, _host(bad)) == DISCO_ERR_INVALID, bad
        assert b"length" in lib.disco_last_error()
    assert call(lib, DUMMY, None) == DISCO_ERR_INVALID            # no host copy
    assert b"null" in lib.disco_last_error()
    assert call(lib, None, ok) == DISCO_ERR_INVALID               # no device copy
    assert b"null" in lib.disco_last_error()


def test_null_outputs_and_inputs(lib):
    ok = _host([30, 1, 17])
    assert _rec(lib, DUMMY, ok, Y=None) == DISCO_ERR_INVALID
    assert _rec(lib, DUMMY, ok, Rss=None) == DISCO_ERR_INVALID
    assert _filt(lib, DUMMY, ok, W=None) == DISCO_ERR_INVALID
    assert _filt(lib, DUMMY, ok, out=None) == DISCO_ERR_INVALID


def test_stack_bounds_and_parameters(lib):
    ok = _host([30, 1, 17])
    assert _rec(lib, DUMMY, ok, K=1, C=17) == DISCO_ERR_UNSUPPORTED     # D = 17
    assert _rec(lib, DUMMY, ok, K=2, C=16) == DISCO_ERR_UNSUPPORTED
    assert _filt(lib, DUMMY, ok, K=9, C=9) == DISCO_ERR_UNSUPPORTED
    assert _rec(lib, DUMMY, ok, block=65) == DISCO_ERR_INVALID
    assert b"block" in lib.disco_last_error()
    assert _rec(lib, DUMMY, ok, T=0) == DISCO_ERR_INVALID


def test_online_tango_validates_lengths():
    from disco_b200 import online
    y = torch.zeros(2, 1, 2, 1000)
    m = torch.zeros(2, 1, 4, 257)
    for bad in ([1000, 256], [1001, 900], [1000]):                # <= n_fft / 2, > L, wrong count
        with pytest.raises(ValueError):
            online.online_tango(y, (m, m), lengths=bad)
    with pytest.raises(TypeError):
        online.online_tango(y, (m, m), lengths=[1000.0, 900.0])
    with pytest.raises(TypeError):
        online.online_tango(y, (m, m), lengths=torch.tensor([1000.0, 900.0]))

