"""CPU checks of the online Tango stream (disco_b200/stream.py): the emission rule against the NumPy restatement of
librosa's stft / istft, and argument validation of the streaming entry points and of the session, before any CUDA
work."""
import ctypes

import numpy as np
import pytest

from oracle import librosa_np


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.mark.parametrize("n_fft", [256, 512])
def test_emission_rule_matches_whole_signal_librosa(n_fft):
    """At every prefix length l, the frames the rule declares out are those of the whole signal, and so are the time
    samples it declares final; after the end of the stream the frame count is librosa's."""
    from disco_b200.stream import emission
    H = n_fft // 2
    rng = np.random.default_rng(n_fft)
    y = rng.standard_normal(6 * H + 3).astype(np.float32)
    S_full = librosa_np.stft(y, n_fft, H)
    x_full = librosa_np.istft(S_full, H, n_fft, length=len(y))
    for l in range(H - 1, 4 * H + 2):
        T_out, S_out = emission(l, n_fft)
        if l <= H:
            assert (T_out, S_out) == (0, 0)
            with pytest.raises(ValueError):
                emission(l, n_fft, final=True)
            continue
        assert T_out == l // H and S_out == (T_out - 1) * H
        S_pre = librosa_np.stft(y[:l], n_fft, H)
        assert np.array_equal(S_pre[:, :T_out], S_full[:, :T_out]), l
        # one frame more would read a sample that has not arrived (or, at l = (t + 1) H - 1, a reflected one)
        assert not np.array_equal(S_pre[:, T_out], S_full[:, T_out]), l
        if S_out > 0:
            x_pre = librosa_np.istft(S_pre[:, :T_out], H, n_fft, length=S_out)
            assert np.array_equal(x_pre, x_full[:S_out]), l
        # end of the stream at l: every frame of the l-sample signal and all l samples
        T_fin, S_fin = emission(l, n_fft, final=True)
        assert T_fin == librosa_np.n_frames_of(l, n_fft, H) == S_pre.shape[1] and S_fin == l


def test_stream_entry_point_validation_without_gpu(lib):
    fake = ctypes.c_void_p(256)   # never dereferenced: every call below fails its argument check first
    st = lib.disco_stream_stft
    assert st(fake, None, None, fake, None, 2, 0, 1000, 0, 1, 0, 0, 0, 500, None) == -1          # bad n_fft
    assert b"n_fft" in lib.disco_last_error()
    assert st(fake, None, None, fake, None, 0, 0, 1000, 0, 1, 0, 0, 0, 512, None) == -1          # n_sig <= 0
    assert st(fake, None, None, fake, None, -3, 0, 1000, 0, 1, 0, 0, 0, 512, None) == -1
    assert st(None, None, None, fake, None, 2, 0, 1000, 0, 1, 0, 0, 0, 512, None) == -1          # no history
    assert b"null pointer" in lib.disco_last_error()
    assert st(fake, None, None, None, None, 2, 0, 1000, 0, 1, 0, 0, 0, 512, None) == -1          # no Y
    assert st(fake, None, None, fake, None, 2, 10, 1000, 0, 1, 0, 0, 0, 512, None) == -1         # chunk missing
    # frame 3 of 512 points needs 4 * 256 samples; frame 0 more than 256; the final call reflects frame L // 256
    assert st(fake, fake, None, fake, None, 2, 10, 1000, 3, 1, 0, 0, 0, 512, None) == -1
    assert b"not complete" in lib.disco_last_error()
    assert st(fake, fake, None, fake, None, 2, 10, 256, 0, 1, 0, 0, 0, 512, None) == -1
    assert st(fake, None, None, fake, None, 2, 0, 1000, 3, 2, 0, 0, 1, 512, None) == -1
    # frame 1 starts at sample 0, older than the history of the last 512 samples before sample 1000
    assert st(fake, fake, None, fake, None, 2, 10, 1010, 1, 1, 0, 0, 0, 512, None) == -1
    assert b"history" in lib.disco_last_error()
    assert st(fake, fake, None, fake, fake, 2, 300, 1000, 2, 1, 8, 8, 0, 512, None) == -1        # block slot
    assert b"block buffer" in lib.disco_last_error()
    si = lib.disco_stream_istft
    assert si(fake, fake, fake, 2, 0, 1, 1000, 0, 0, 100, 300, None) == -1                        # bad n_fft
    assert b"n_fft" in lib.disco_last_error()
    assert si(fake, fake, fake, 0, 0, 1, 1000, 0, 0, 100, 512, None) == -1                        # n_sig <= 0
    assert si(fake, None, fake, 2, 0, 1, 1000, 0, 0, 100, 512, None) == -1                        # no carry
    assert b"null pointer" in lib.disco_last_error()
    assert si(None, fake, fake, 2, 0, 1, 1000, 0, 0, 100, 512, None) == -1                        # no Y
    assert si(fake, fake, None, 2, 2, 3, 2000, 0, 0, 1000, 512, None) == -1                       # no x
    assert si(fake, fake, fake, 2, 2, 3, 2000, 0, 300, 1000, 512, None) == -1                     # x too late
    assert b"outside x" in lib.disco_last_error()
    assert si(fake, fake, fake, 2, 2, 3, 2000, 0, 256, 500, 512, None) == -1                      # x too short


def test_session_validation_without_gpu():
    import torch
    from disco_b200.stream import OnlineTangoStream
    for kw in (dict(n_fft=500), dict(n_fft=2048), dict(block=0), dict(block=65), dict(lambda_cor=1.0),
               dict(lambda_cor=-0.1), dict(ref_mic=4), dict(ref_mic=-1), dict(lag=-1)):
        with pytest.raises(ValueError):
            OnlineTangoStream(2, 1, 4, **kw)
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(2, 1, 4, lag=0)
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(1, 2, 8)          # D = 9
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(1, 8, 2)          # D = 9 (cfg 5)
    with pytest.raises(ValueError):
        OnlineTangoStream(0, 1, 4)
    with pytest.raises(TypeError):
        OnlineTangoStream(1, 1, 4, device="cpu")
    R = torch.zeros(1, 1, 257, 4, 4, dtype=torch.complex64)
    with pytest.raises(TypeError):
        OnlineTangoStream(1, 1, 4, R0=(R, R))
    with pytest.raises(ValueError):
        OnlineTangoStream(1, 1, 4, R0=R)
