"""CPU checks of the pool of online Tango streams (disco_b200/stream.py OnlineTangoPool): the round cutting against a
per-frame assignment, the pool's validation before any CUDA work, the ABI rejections of the per-slot stream entry
points, and the dispatch sets of their launchers against the GPU test's table."""
import ctypes
import re

import numpy as np
import pytest

import test_gpu_stream_pool as gpu
from test_kernel_instances_cpu import _function, _src


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_pool_rounds_against_per_frame_assignment():
    from disco_b200.stream import pool_rounds
    rng = np.random.default_rng(0)
    for _ in range(300):
        S, P = int(rng.integers(1, 9)), int(rng.integers(1, 12))
        T0 = rng.integers(0, 5 * P, S)
        T1 = T0 + rng.integers(0, 4 * P, S) * (rng.random(S) < 0.8)
        t0, n = pool_rounds(T0, T1, P)
        assert t0.shape == n.shape and (len(n) == 0 or n.max(axis=1).min() >= 1)   # every round has work
        for s in range(S):
            # brute force: frame t belongs to run r = (number of block boundaries in (T0, t])
            want = {}
            for t in range(T0[s], T1[s]):
                r = t // P - T0[s] // P
                want.setdefault(r, []).append(t)
            got = {r: list(range(t0[r, s], t0[r, s] + n[r, s])) for r in range(len(n)) if n[r, s]}
            assert got == want, (s, T0[s], T1[s], P)
            for r in range(len(n)):
                if n[r, s]:
                    assert t0[r, s] // P == (t0[r, s] + n[r, s] - 1) // P          # no run crosses a boundary
                else:
                    assert all(n[q, s] == 0 for q in range(r, len(n)))           # runs are consecutive rounds
        # slots are independent: each slot's runs are those of the slot cut alone
        for s in range(S):
            a, b = pool_rounds(T0[s:s + 1], T1[s:s + 1], P)
            k = len(b)
            assert np.array_equal(b[:, 0], n[:k, s]) and not n[k:, s].any()
            assert np.array_equal(a[b[:, 0] > 0, 0], t0[:k, s][n[:k, s] > 0])
    with pytest.raises(ValueError):
        pool_rounds([3], [2], 4)


def _pool(S=3, K=1, C=2, **kw):
    from disco_b200.stream import OnlineTangoPool
    return OnlineTangoPool(S, K, C, device="cuda:0", **kw)


def test_pool_validation_without_gpu():
    import torch
    from disco_b200.stream import OnlineTangoPool
    for kw in (dict(n_fft=500), dict(n_fft=2048), dict(block=0), dict(block=65), dict(lambda_cor=1.0),
               dict(lambda_cor=-0.1), dict(ref_mic=2), dict(ref_mic=-1), dict(lag=-1)):
        with pytest.raises(ValueError):
            _pool(**kw)
    with pytest.raises(NotImplementedError):
        _pool(lag=0)
    with pytest.raises(NotImplementedError):
        _pool(K=2, C=16)                               # D = 17
    _pool(K=8, C=2)                                    # D = 9 and
    _pool(K=1, C=16)                                   # D = 16 are covered
    with pytest.raises(ValueError):
        _pool(S=0)
    with pytest.raises(TypeError):
        OnlineTangoPool(2, 1, 4, device="cpu")
    ok = lambda *a: None
    p = _pool()
    with pytest.raises(ValueError):
        p.open([3])                                    # no such slot
    with pytest.raises(ValueError):
        p.open([1, 1])
    with pytest.raises(ValueError):
        p.close([0], ok)                               # free slot
    # host state of an open slot, set directly: the checks below read nothing else and launch nothing
    p._open[1], p._L[1] = True, 128
    with pytest.raises(ValueError):
        p.open([1])                                    # already open
    with pytest.raises(ValueError):
        p.close([1], ok)                               # 128 samples = n_fft / 2
    y = torch.zeros(3, 1, 2, 10)
    with pytest.raises(ValueError):
        p.push(y, [0, 5, 5], ok)                       # samples to free slot 2
    with pytest.raises(ValueError):
        p.push(y, [0, 11, 0], ok)                      # n > n_max
    with pytest.raises(ValueError):
        p.push(y, [0, -1, 0], ok)
    with pytest.raises(ValueError):
        p.push(y, [0, 1], ok)                          # one n per slot
    with pytest.raises(ValueError):
        p.push(torch.zeros(3, 2, 2, 10), [0, 1, 0], ok)
    with pytest.raises(TypeError):
        p.push(y, [0, 5, 0], ok)                       # a valid call on a CPU tensor
    assert p._L[1] == 128 and list(p._open) == [False, True, False]   # the pool is as it was
    R = torch.zeros(1, 1, 257, 2, 2, dtype=torch.complex64)
    with pytest.raises(TypeError):
        p.open([0], R0=(R, R))
    with pytest.raises(ValueError):
        p.open([0], R0=R)


def test_stream_slots_entry_point_validation_without_gpu(lib):
    fake = ctypes.c_void_p(256)   # never dereferenced: every call below fails its argument check first
    c_rec = lambda rows: (ctypes.c_int * (len(rows) * len(rows[0])))(*[v for r in rows for v in r])
    st = lib.disco_stream_stft_slots
    # record: length, n_new, t0, n_fr, blk_slot, final, hist_sel, hist_write
    good = [[770, 10, 2, 1, 0, 0, 0, 1], [0, 0, 0, 0, 0, 0, 0, 0]]
    args = lambda rows, n_fft=512, n_max=10, f_max=4, blk=8, Y=fake, chunk=fake, hist=fake: (
        hist, chunk, Y, fake, fake, c_rec(rows), len(rows), 3, n_max, f_max, blk, n_fft, None)
    assert st(*args(good, n_fft=500)) == -1
    assert b"n_fft" in lib.disco_last_error()
    assert st(*args(good, hist=None)) == -1
    assert b"null pointer" in lib.disco_last_error()
    assert st(*args(good, chunk=None)) == -1                                 # a slot has new samples
    assert st(*args(good, Y=None)) == -1                                     # a slot has frames
    assert st(*args([[1000, 11, 2, 1, 0, 0, 0, 1]])) == -1                   # n_new > n_max
    assert b"bad sizes" in lib.disco_last_error()
    assert st(*args([[1000, 10, 2, 5, 0, 0, 0, 1]])) == -1                   # n_fr > f_max
    assert st(*args([[1000, 10, 2, 1, 0, 0, 2, 1]])) == -1                   # hist_sel not 0 / 1
    assert st(*args([[1000, 10, 3, 1, 0, 0, 0, 1]])) == -1                   # frame 3 needs 1024 samples
    assert b"not complete" in lib.disco_last_error()
    assert st(*args([[1000, 0, 3, 2, 0, 1, 0, 0]])) == -1                    # final: frame 1000 // 256 is the last
    assert st(*args([[1000, 10, 2, 1, 0, 1, 0, 0]])) == -1                   # final with a chunk
    assert b"final" in lib.disco_last_error()
    assert st(*args([[1010, 10, 1, 1, 0, 0, 0, 1]])) == -1                   # older than the history
    assert b"history" in lib.disco_last_error()
    assert st(*args([[770, 10, 2, 1, 8, 0, 0, 1]])) == -1                     # block slot past the buffer
    assert b"block buffer" in lib.disco_last_error()
    assert st(fake, fake, fake, fake, fake, None, 1, 3, 10, 4, 8, 512, None) == -1
    assert st(*args([[0] * 8], n_max=-1)) == -1
    si = lib.disco_stream_istft_slots
    # record: t0, n_fr, length, final, x_first
    iargs = lambda rows, n_fft=512, s_max=1000, f_max=4, x=fake, Y=fake, carry=fake: (
        Y, carry, x, fake, c_rec(rows), len(rows), 3, f_max, s_max, n_fft, None)
    ig = [[2, 3, 2000, 0, 256], [0, 0, 5, 0, 0]]
    assert si(*iargs(ig, n_fft=300)) == -1
    assert b"n_fft" in lib.disco_last_error()
    assert si(*iargs(ig, carry=None)) == -1
    assert b"null pointer" in lib.disco_last_error()
    assert si(*iargs(ig, Y=None)) == -1
    assert si(*iargs(ig, x=None)) == -1
    assert si(*iargs([[2, 3, 2000, 0, 300]])) == -1                          # x starts after the first sample
    assert b"outside x" in lib.disco_last_error()
    assert si(*iargs([[2, 3, 2000, 0, 256]], s_max=500)) == -1               # x too short
    assert si(*iargs([[2, 3, 2000, 1, 256]], s_max=1000)) == -1              # final: up to sample 2000
    assert si(*iargs([[2, 5, 2000, 0, 256]])) == -1                          # n_fr > f_max
    assert b"bad sizes" in lib.disco_last_error()
    assert si(*iargs([[-1, 1, 2000, 0, 0]])) == -1
    assert si(fake, fake, fake, fake, None, 1, 3, 4, 100, 512, None) == -1


def test_slots_dispatch_sets_match_gpu_table():
    """Every n_fft the per-slot launchers instantiate has edge cases in tests/test_gpu_stream_pool.py, at the job and
    CTA sizes the kernels use."""
    src = _src("stream.cu")
    body = _function(src, "cudaError_t launch_stream_stft_slots(")
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_stft_slots_n<(\d+)>", body)
    assert found and all(a == b for a, b in found)
    assert {int(a) for a, _ in found} == set(gpu.SLOT_NFFTS)
    assert re.search(r"constexpr int kStreamWarps = (\d+);", src).group(1) == "4"
    for n in gpu.SLOT_NFFTS:
        assert gpu.JOB_FRAMES[n] == 32 // (n // 32) and gpu.CTA_FRAMES[n] == 4 * gpu.JOB_FRAMES[n]
    body = _function(_src("istft.cu"), "cudaError_t launch_stream_istft_slots(")
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_slots_n<(\d+)>", body)
    assert found and all(a == b for a, b in found)
    assert {int(a) for a, _ in found} == set(gpu.SLOT_NFFTS)
