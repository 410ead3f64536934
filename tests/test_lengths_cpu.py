"""CPU-side checks of the `lengths=` interface: the C ABI of the length-aware STFT / iSTFT rejects bad lengths, null
pointers and n_fft before any CUDA work, and the Python layer validates lengths with the usual exception types."""
import ctypes

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def _host(vals):
    arr = (ctypes.c_int * len(vals))(*vals)
    return arr


DUMMY = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first


def test_stft_lengths_abi_rejects(lib):
    L, n_fft = 4000, 512
    ok = _host([L, 257, 3000])
    assert lib.disco_stft_lengths(DUMMY, DUMMY, ok, DUMMY, 3, L, 500, None) == -1             # bad n_fft
    assert b"n_fft" in lib.disco_last_error()
    assert lib.disco_stft_lengths(DUMMY, DUMMY, ok, DUMMY, 0, L, n_fft, None) == -1           # no signals
    assert lib.disco_stft_lengths(DUMMY, DUMMY, ok, DUMMY, 3, 256, n_fft, None) == -1         # L_max = hop
    for bad in ([L, 256, 3000], [L, 0, 3000], [L + 1, 300, 300], [L, -5, 300]):                # <= hop, > L_max
        assert lib.disco_stft_lengths(DUMMY, DUMMY, _host(bad), DUMMY, 3, L, n_fft, None) == -1, bad
        assert b"length" in lib.disco_last_error()
    assert lib.disco_stft_lengths(DUMMY, DUMMY, None, DUMMY, 3, L, n_fft, None) == -1         # no host lengths
    assert lib.disco_stft_lengths(None, DUMMY, ok, DUMMY, 3, L, n_fft, None) == -1            # null x
    assert b"null" in lib.disco_last_error()
    assert lib.disco_stft_lengths(DUMMY, None, ok, DUMMY, 3, L, n_fft, None) == -1            # null device lengths
    assert lib.disco_stft_lengths(DUMMY, DUMMY, ok, None, 3, L, n_fft, None) == -1            # null Y


def test_istft_lengths_abi_rejects(lib):
    L, n_fft = 4000, 256
    ok = _host([L, 1, 3000])
    assert lib.disco_istft_lengths(DUMMY, DUMMY, ok, DUMMY, 3, 32, L, 300, None) == -1        # bad n_fft
    assert lib.disco_istft_lengths(DUMMY, DUMMY, ok, DUMMY, 3, 0, L, n_fft, None) == -1       # no frames
    assert lib.disco_istft_lengths(DUMMY, DUMMY, ok, DUMMY, 3, 32, 0, n_fft, None) == -1      # no samples
    for bad in ([L, 0, 3000], [L + 1, 1, 1]):
        assert lib.disco_istft_lengths(DUMMY, DUMMY, _host(bad), DUMMY, 3, 32, L, n_fft, None) == -1, bad
    assert lib.disco_istft_lengths(DUMMY, DUMMY, None, DUMMY, 3, 32, L, n_fft, None) == -1
    assert lib.disco_istft_lengths(None, DUMMY, ok, DUMMY, 3, 32, L, n_fft, None) == -1
    assert lib.disco_istft_lengths(DUMMY, None, ok, DUMMY, 3, 32, L, n_fft, None) == -1
    assert lib.disco_istft_lengths(DUMMY, DUMMY, ok, None, 3, 32, L, n_fft, None) == -1


def test_signal_lengths_expands_and_validates():
    from disco_b200.ops import signal_lengths
    out = signal_lengths([300, 400], (2, 3, 2), 500, lo=256)
    assert out.dtype == np.int32 and out.tolist() == [300] * 6 + [400] * 6
    assert signal_lengths(torch.tensor([[300, 301]]), (1, 2, 4), 500).tolist() == [300] * 4 + [301] * 4
    assert signal_lengths(np.array(450), (3,), 500).tolist() == [450] * 3
    with pytest.raises(ValueError):
        signal_lengths([300, 400, 500], (2, 3), 500)            # not a leading-axes shape
    with pytest.raises(ValueError):
        signal_lengths([256, 400], (2,), 500, lo=256)          # <= hop
    with pytest.raises(ValueError):
        signal_lengths([501, 400], (2,), 500)                  # > L_max
    with pytest.raises(TypeError):
        signal_lengths([300.0, 400.0], (2,), 500)              # not integers
    with pytest.raises(TypeError):
        signal_lengths(torch.tensor([300.0]), (1,), 500)


def test_python_entry_points_validate():
    from disco_b200 import ops
    from disco_b200.tango import _uneven_lengths, tango_batched
    x = torch.zeros(2, 1000)
    with pytest.raises(TypeError):                             # no CPU path
        ops.stft_lengths(x, [600, 700])
    with pytest.raises(TypeError):
        ops.istft_lengths(torch.zeros(2, 5, 257, dtype=torch.complex64), [600, 700], 1000)
    assert _uneven_lengths(None, 3, 1000, 512) is None
    assert _uneven_lengths([1000, 1000, 1000], 3, 1000, 512) is None           # the uniform batch
    assert _uneven_lengths([1000, 700, 1000], 3, 1000, 512).tolist() == [1000, 700, 1000]
    with pytest.raises(ValueError):
        _uneven_lengths([1000, 700], 3, 1000, 512)
    with pytest.raises(ValueError):
        _uneven_lengths([1000, 200, 1000], 3, 1000, 512)
    with pytest.raises(ValueError):
        tango_batched(torch.zeros(3, 1, 2, 1000), torch.zeros(3, 1, 2, 1000), torch.zeros(3, 1, 2, 1000),
                      lengths=[1000, 1001, 900])


def test_resample_and_stoi_lengths_abi_rejects(lib):
    ok = _host([4000, 300])
    for bad in ([4000, 0], [4001, 300]):
        assert lib.disco_resample_poly_lengths(DUMMY, DUMMY, DUMMY, 5, 5, 8, 2, 4000, DUMMY, _host(bad), None) == -1
        assert b"length" in lib.disco_last_error()
    assert lib.disco_resample_poly_lengths(DUMMY, DUMMY, DUMMY, 5, 5, 8, 2, 4000, None, ok, None) == -1
    assert lib.disco_resample_poly_lengths(DUMMY, DUMMY, DUMMY, 5, 5, 8, 2, 4000, DUMMY, None, None) == -1
    assert lib.disco_resample_poly_lengths(DUMMY, DUMMY, DUMMY, 5, 4, 8, 2, 4000, DUMMY, ok, None) == -1  # not coprime
    ws = lib.disco_stoi_workspace(2, 2, 4000)
    for bad in ([4000, 255], [4001, 300]):                      # STOI needs 256 samples at 10 kHz
        assert lib.disco_stoi_lengths(DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, 2, 2, 2, 4000, DUMMY, _host(bad),
                                      DUMMY, ws, None) == -1
    assert lib.disco_stoi_lengths(DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, 2, 2, 2, 4000, None, ok, DUMMY, ws,
                                  None) == -1
    assert lib.disco_stoi_lengths(DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, DUMMY, 2, 2, 2, 4000, DUMMY, ok, DUMMY, 0,
                                  None) == -3                  # workspace too small
