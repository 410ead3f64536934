"""CPU checks of stream positions past C int (DESIGN §4.5, "Positions"): the records ops hands the library are
rebased to a hop-aligned origin, valid exactly when the absolute record is and inside the library's bound; nothing is
narrowed silently; reflect_index is exact up to the bound; and the ABI rejects every record or whole-signal length
past it, including records whose checks would wrap in 32-bit arithmetic."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "disco_b200", "csrc")
INT_MAX = 2 ** 31 - 1
NFFTS = (256, 512, 1024)


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def bound(n_fft):
    return INT_MAX - n_fft - 1024


# check_stft_record / check_istft_record (csrc/api.cu) restated on unbounded ints, every pointer given; lim = the
# library's position bound, or None for the absolute record
def stft_valid(r, n_fft, n_max, f_max, blk_frames, lim=None):
    length, n_new, t0, n_fr, blk_slot, final, sel, _ = r
    H = n_fft // 2
    if n_new < 0 or n_new > n_max or length < n_new or t0 < 0 or n_fr < 0 or n_fr > f_max or sel not in (0, 1):
        return False
    if lim is not None and (length > lim or (t0 + n_fr) * H > lim):
        return False
    if final and n_new > 0:
        return False
    if n_fr > 0:
        L0, t1 = length - n_new, t0 + n_fr - 1
        arrived = length > H and (t1 <= length // H if final else (t1 == 0 or (t1 + 1) * H <= length))
        if not arrived or (t0 >= 1 and (t0 - 1) * H < L0 - n_fft):
            return False
        if blk_slot < 0 or blk_slot + n_fr > blk_frames:
            return False
    return True


def istft_valid(r, n_fft, f_max, s_max, lim=None):
    t0, n_fr, length, final, x_first = r
    H = n_fft // 2
    if t0 < 0 or n_fr < 0 or n_fr > f_max or x_first < 0 or (length < 1 and (n_fr > 0 or final)):
        return False
    if lim is not None and (length > lim or x_first > lim or (t0 + n_fr) * H > lim):
        return False
    if n_fr <= 0 and not final:
        return True
    lo = max(t0 - 1, 0) * H
    hi = min(length if final else (t0 + n_fr - 1) * H, length)
    return hi <= lo or (lo >= x_first and hi <= x_first + s_max)


def _bases(n_fft):
    H = n_fft // 2
    out = [H * m for m in range(1, 5)] + [H * m + 1 for m in range(1, 5)]
    for big in (2 ** 30, 2 ** 31, 2 ** 32, 2 ** 62):
        for k in (0, 1, H - 1, H, H + 1, 2 * H - 1):
            out += [big + k, big - k]
    return sorted(set(v for v in out if v > 0))


def _stft_records(n_fft):
    """Records around every edge of the checks: frames just complete / not, just inside the history / not, final or
    not, chunks of 0 .. 3H + 1 samples, and no frames."""
    H = n_fft // 2
    for L in _bases(n_fft):
        for final in (0, 1):
            for n_new in ((0,) if final else (0, 1, H - 1, H, 3 * H + 1)):
                if n_new > L:
                    continue
                L0 = L - n_new
                T = L // H + 1 if final else L // H       # frames 0 .. T - 1 complete
                tmin = max(0, -((n_fft - L0) // H) + 1) if L0 > n_fft else 0   # first frame inside the history
                for t0 in {tmin - 1, tmin, tmin + 1, T - 1, T}:
                    for t1 in {t0, T - 2, T - 1, T}:
                        n_fr = t1 - t0 + 1
                        if t0 >= 0 and 0 <= n_fr <= 64:
                            yield [L, n_new, t0, n_fr, 3, final, 1, 1]
                yield [L, n_new, max(T - 1, 0), 0, 0, final, 0, 1]


def _istft_records(n_fft):
    """Records a stream can make: frames within a few of the last one (frame 0 only near the start; a record of
    positions far apart, such as frame 0 of a stream at 2^40 samples, fits no origin), around the edges of x."""
    H = n_fft // 2
    for L in _bases(n_fft):
        T = L // H
        for final in (0, 1):
            for t0 in {0, 1, max(T - 3, 0), T - 1, T, T + 1}:
                for n_fr in (0, 1, 2, 7):
                    if t0 < 0 or t0 < T - 8:
                        continue
                    lo = max(t0 - 1, 0) * H
                    for x_first in {lo - 1, lo, lo + 1, lo - H, 0 if lo <= 4 * n_fft else lo}:
                        if x_first >= 0:
                            yield [t0, n_fr, L, final, x_first]


@pytest.mark.parametrize("n_fft", NFFTS)
def test_rebase_stft_records(n_fft):
    from disco_b200 import ops
    H = n_fft // 2
    n_max, f_max, blk = 3 * H + 1, 64, 72
    n = 0
    for r in _stft_records(n_fft):
        ok = stft_valid(r, n_fft, n_max, f_max, blk)
        try:
            rel = [int(v) for v in ops._records(np.array([r], dtype=np.int64), 1, ops.STFT_SLOT_FIELDS, "s", n_fft)[0]]
        except ValueError:
            assert not ok, r                              # a valid record always fits after rebasing
            continue
        O = r[0] - rel[0]
        assert O % H == 0 and O >= 0, (r, rel)
        assert rel[2] == r[2] - O // H and rel[1:2] + rel[3:] == r[1:2] + r[3:], (r, rel)
        L0 = r[0] - r[1]
        if O > 0:
            assert O <= L0 - n_fft and O <= (r[2] - 1) * H, (r, O)   # not after the history or frame t0's start
        if r[2] == 0 or L0 < n_fft:
            assert O == 0, r                              # the start reflection or the zeros before sample 0
        assert stft_valid(rel, n_fft, n_max, f_max, blk, bound(n_fft)) == ok, (r, rel)
        if ok:
            assert rel[0] <= n_max + n_fft + H and rel[0] <= bound(n_fft), (r, rel)
        n += ok
    assert n > 300


@pytest.mark.parametrize("n_fft", NFFTS)
def test_rebase_istft_records(n_fft):
    from disco_b200 import ops
    H = n_fft // 2
    f_max, s_max = 7, 8 * H
    n = 0
    for r in _istft_records(n_fft):
        ok = istft_valid(r, n_fft, f_max, s_max)
        try:
            rel = [int(v) for v in ops._records(np.array([r], dtype=np.int64), 1, ops.ISTFT_SLOT_FIELDS, "s", n_fft)[0]]
        except ValueError:
            assert not ok, r
            continue
        O = r[2] - rel[2]
        assert O % H == 0 and O >= 0 and rel[4] == r[4] - O and rel[0] == r[0] - O // H, (r, rel)
        assert rel[1] == r[1] and rel[3] == r[3]
        if O > 0:
            assert O <= (r[0] - 1) * H and O <= r[4] and O <= r[2] - 1, (r, O)   # not after a sample written
        if r[0] == 0:
            assert O == 0, r
        assert istft_valid(rel, n_fft, f_max, s_max, bound(n_fft)) == ok, (r, rel)
        if ok:
            assert max(rel[2], rel[4], (rel[0] + rel[1]) * H) <= 4 * n_fft + s_max, (r, rel)
        n += ok
    assert n > 300


def test_rebase_is_per_slot_and_keeps_idle_slots():
    """A pool launch rebases every slot on its own: slots at 0, past 2^31 and past 2^62 in one record array."""
    from disco_b200 import ops
    n_fft, H = 512, 256
    recs = np.array([[700, 700, 0, 2, 0, 0, 0, 1], [2 ** 31 + 5 * H + 1, 300, (2 ** 31 + 5 * H) // H - 1, 1, 0, 0, 1, 1],
                     [2 ** 62 + 7, 0, (2 ** 62 + 7) // H, 1, 0, 1, 0, 0], [0] * 8], dtype=np.int64)
    rel = ops._records(recs, 4, ops.STFT_SLOT_FIELDS, "s", n_fft)
    assert rel.dtype == np.int32 and rel.flags.c_contiguous
    assert rel[0].tolist() == recs[0].tolist() and rel[3].tolist() == [0] * 8
    for s in (1, 2):
        O = int(recs[s, 0]) - int(rel[s, 0])
        assert O % H == 0 and int(recs[s, 2]) - int(rel[s, 2]) == O // H and 0 < rel[s, 0] < 4 * n_fft
        assert stft_valid([int(v) for v in rel[s]], n_fft, 300, 4, 8, bound(n_fft))


def test_narrowing_is_refused():
    from disco_b200 import ops
    S, I = ops.STFT_SLOT_FIELDS, ops.ISTFT_SLOT_FIELDS
    bad_stft = [
        [2 ** 31, 2 ** 31, 0, 0, 0, 0, 0, 1],          # a chunk of 2^31 samples: nothing to rebase
        [2 ** 31 + 5, 0, 0, 1, 0, 1, 0, 0],            # frame 0 of a 2^31-sample signal: the start reflection
        [2 ** 32 + 5, 5, 0, 1, 0, 0, 0, 0],            # would wrap to a small valid length
        [1000, 10, 2 ** 33, 1, 0, 0, 0, 0],            # frame far past the samples
        [1000, 10, 2, 2 ** 32 + 1, 0, 0, 0, 0],
        [1000, 10, 2, 1, -2 ** 31 - 1, 0, 0, 0],
    ]
    for r in bad_stft:
        with pytest.raises(ValueError):
            ops._records(np.array([r], dtype=np.int64), 1, S, "slots", 512)
    bad_istft = [[0, 1, 2 ** 31 + 1, 1, 0], [3, 1, 2 ** 32 + 1000, 0, 2 ** 32 + 9], [2 ** 40, 1, 1000, 0, 0],
                 [3, 2 ** 31, 4000, 0, 256]]
    for r in bad_istft:
        with pytest.raises(ValueError):
            ops._records(np.array([r], dtype=np.int64), 1, I, "slots", 512)
    with pytest.raises(ValueError):                    # past int64
        ops._records(np.array([[2 ** 70, 1, 0, 0, 0]], dtype=object), 1, I, "slots", 512)
    with pytest.raises(ValueError):
        ops._records(np.array([[2 ** 64 - 1, 1, 0, 0, 0]], dtype=np.uint64), 1, I, "slots", 512)
    with pytest.raises(TypeError):
        ops._records(np.zeros((1, 5)), 1, I, "slots", 512)


class _FakeLib:
    """Stands in for the library: records the scalar stream calls' int arguments and launches nothing."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, [a for a in args if isinstance(a, int)]))
            return 0
        return call


@pytest.fixture
def fake_ops(monkeypatch):
    import torch
    from disco_b200 import ops
    fake = _FakeLib()
    monkeypatch.setattr(ops, "_need", lambda t, dtype, name: t)
    monkeypatch.setattr(ops, "_stream", lambda: None)
    monkeypatch.setattr(ops._lib, "load", lambda: fake)
    return ops, fake, torch


def test_scalar_stream_ops_refuse_narrowing_before_device_work(fake_ops):
    ops, fake, torch = fake_ops
    hist, chunk = torch.zeros(2, 512), torch.zeros(2, 5)
    for length, t0, n_fr in ((2 ** 31 + 5, 0, 1), (2 ** 32 + 5, 0, 1), (2 ** 40, 2 ** 40, 1), (2 ** 64, 0, 0)):
        with pytest.raises(ValueError):
            ops.stream_stft(hist, chunk, length, t0, n_fr, 512)
    Y, carry = torch.zeros(2, 1, 257, dtype=torch.complex64), torch.zeros(2, 256)
    for t0, length, final, x_first in ((0, 2 ** 31 + 1, True, 0), (2 ** 33, 1000, False, 0),
                                       (5, 2 ** 32 + 2000, False, 2 ** 32 + 1024)):
        with pytest.raises(ValueError):
            ops.stream_istft(Y, carry, t0, length, 512, final=final, x=torch.zeros(2, 4096), x_first=x_first)
    assert fake.calls == []


def test_scalar_stream_ops_hand_the_library_rebased_positions(fake_ops):
    ops, fake, torch = fake_ops
    H = 256
    for base in (0, 2 ** 30, 2 ** 31, 2 ** 32, 2 ** 40, 2 ** 62):
        A = base + 9 * H + 7                                   # samples in; chunk of 300, frames 6 .. 7 complete
        hist, chunk = torch.zeros(3, 512), torch.zeros(3, 300)
        t0 = (A - 300 - 512) // H + 1 if base else 6
        n_fr = A // H - t0
        ops.stream_stft(hist, chunk, A, t0, n_fr, 512)
        name, ints = fake.calls.pop()
        assert name == "disco_stream_stft"
        n_sig, n_new, length, t0r, n_frr = ints[:5]
        O = A - length
        assert (n_sig, n_new, n_frr) == (3, 300, n_fr) and O % H == 0 and t0 - t0r == O // H
        assert 0 < length <= 300 + 512 + 2 * H
        Y, carry = torch.zeros(3, n_fr, 257, dtype=torch.complex64), torch.zeros(3, H)
        x = ops.stream_istft(Y, carry, t0, A, 512, final=True)
        name, ints = fake.calls.pop()
        n_sig, t0r, n_frr, length, final, x_first, s_max = ints[:7]
        O = A - length
        assert name == "disco_stream_istft" and final == 1 and O % H == 0 and t0 - t0r == O // H
        assert x_first == (t0 - 1) * H - O and s_max == x.shape[-1] == A - (t0 - 1) * H and 0 <= x_first < length


REFLECT_MAIN = r"""
#include <cstdio>
#include "stft_core.cuh"
int main() {
    long long s, L;
    while (scanf("%lld %lld", &s, &L) == 2) printf("%d\n", disco::reflect_index((int)s, (int)L));
    return 0;
}
"""

SHIM = r"""
#pragma once
#include <cmath>
struct float2 { float x, y; };
static inline float2 make_float2(float x, float y) { float2 v; v.x = x; v.y = y; return v; }
static inline float2 fadd2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
static inline float2 fmul2(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
static inline float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
static inline float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
static inline void __syncwarp() {}
#define DISCO_DEV static inline
"""


@pytest.mark.skipif(shutil.which("g++") is None, reason="needs a host C++ compiler")
def test_reflect_index_on_the_host_up_to_the_bound(tmp_path):
    """reflect_index (csrc/stft_core.cuh) compiled for the host with every signed overflow trapped (UBSan: an overflow
    is undefined behaviour the device compiler may build on), at both ends of signals longer than 2^30 samples and up
    to the bound, against the reflection on Python ints."""
    for fn in ("stft_core.cuh", "fft_reg.cuh", "tw32.cuh"):
        shutil.copy(os.path.join(CSRC, fn), tmp_path / fn)
    (tmp_path / "common.cuh").write_text(SHIM)
    (tmp_path / "main.cpp").write_text(REFLECT_MAIN)
    exe = tmp_path / "reflect"
    subprocess.run(["g++", "-std=c++17", "-O2", "-fsanitize=signed-integer-overflow", "-fno-sanitize-recover=all",
                    "-x", "c++", str(tmp_path / "main.cpp"), "-o", str(exe)], check=True, cwd=tmp_path)
    cases = []
    for n_fft in NFFTS:
        H = n_fft // 2
        for L in (2 ** 30 + 1, 2 ** 30 + 2, 2 ** 30 + 1000, bound(n_fft), INT_MAX - 1 - 1024 - H, 5 * H + 3):
            cases += [(s, L) for s in range(-H, 1)] + [(s, L) for s in range(L - 1, L + H)]
    out = subprocess.run([str(exe)], input="\n".join("%d %d" % c for c in cases), capture_output=True, text=True,
                         check=True).stdout.split()
    want = [(-s if s < 0 else s) if -s < L and s < L else (2 * (L - 1) - s) for s, L in cases]
    assert [int(v) for v in out] == want


def _fake():
    return ctypes.c_void_p(256)   # never dereferenced: every call below fails its argument check first


def _stft_both(lib, r, n_fft, n_sig=3, n_max=None, f_max=None, blk=None):
    """disco_stream_stft and disco_stream_stft_slots on one record, fake pointers throughout"""
    f = _fake()
    length, n_new, t0, n_fr, blk_slot, final, _, write = r
    n_max = n_new if n_max is None else n_max
    f_max = n_fr if f_max is None else f_max
    blk = blk_slot + n_fr if blk is None else blk
    one = lib.disco_stream_stft(f, f, f if write else None, f, f, n_sig, n_new, length, t0, n_fr, blk, blk_slot,
                                final, n_fft, None)
    rec = (ctypes.c_int * 8)(*r)
    pool = lib.disco_stream_stft_slots(f, f, f, f, f, rec, 1, n_sig, n_max, f_max, blk, n_fft, None)
    return one, pool


def _istft_both(lib, r, n_fft, s_max, n_sig=3):
    f = _fake()
    t0, n_fr, length, final, x_first = r
    one = lib.disco_stream_istft(f, f, f, n_sig, t0, n_fr, length, final, x_first, s_max, n_fft, None)
    rec = (ctypes.c_int * 5)(*r)
    pool = lib.disco_stream_istft_slots(f, f, f, f, rec, 1, n_sig, max(n_fr, 1), s_max, n_fft, None)
    return one, pool


def _wraps_in_32_bits(v):
    return not -2 ** 31 <= v <= INT_MAX


@pytest.mark.parametrize("n_fft", NFFTS)
def test_stream_entry_points_reject_positions_past_the_bound(lib, n_fft):
    H, B = n_fft // 2, bound(n_fft)
    stft = []
    # valid in every other respect, just above the bound: frames just complete, non-final and final
    for L in (B + 1, B + H, INT_MAX - 1, INT_MAX):
        stft.append([L, 300, L // H - 2, 1, 0, 0, 0, 1])
        stft.append([L, 0, L // H - 1, 2, 0, 1, 0, 0])
    # the record of a valid small call with t0 moved by 2^32 / H: the 32-bit checks saw the small call again
    small = [4 * H + 10, H + 20, 2, 2, 0, 0, 0, 1]
    assert stft_valid(small, n_fft, H + 20, 2, 2)
    stft.append(small[:2] + [2 + 2 ** 32 // H] + small[3:])
    assert _wraps_in_32_bits((stft[-1][2] + 2) * H)
    # a frame run whose end wraps: (t1 + 1) H past INT_MAX
    t0 = (INT_MAX - 2 * H) // H
    stft.append([INT_MAX, 10, t0, 4, 0, 0, 0, 1])
    stft.append(small[:3] + [2 ** 31 // H + 1] + small[4:])
    # blk_slot + n_fr past INT_MAX
    stft.append(small[:4] + [INT_MAX] + small[5:])
    for r in stft:
        kw = dict(blk=INT_MAX) if r[4] == INT_MAX else {}
        assert _stft_both(lib, r, n_fft, **kw) == (-1, -1), r
    istft = []
    for L in (B + 1, INT_MAX - 100, INT_MAX):
        T = L // H
        istft.append([T - 1, 2, L, 1, (T - 2) * H])       # final call: the tail runs up to L
        istft.append([T - 1, 1, L, 0, (T - 2) * H])
    istft.append([2 ** 32 // H + 2, 3, 2000, 0, 256])        # lo, hi wrap to [256, 1024)
    istft.append([2, 3, 2000, 0, B + 1])                    # x_first past the bound, nothing written
    istft.append([(INT_MAX - H) // H, 4, INT_MAX - 10, 0, INT_MAX - 2 * H])
    for r in istft:
        assert _istft_both(lib, r, n_fft, s_max=4 * n_fft) == (-1, -1), r


def test_whole_signal_entry_points_reject_lengths_past_the_bound(lib):
    f = _fake()
    lens = (ctypes.c_int * 4)(*([300] * 4))
    for n_fft in NFFTS:
        for L in (bound(n_fft) + 1, INT_MAX):
            T = L // (n_fft // 2) + 1
            assert lib.disco_stft(f, f, 4, L, n_fft, None) == -1
            assert b"length" in lib.disco_last_error()
            assert lib.disco_stft_scm(f, f, 0, f, f, f, 1, 2, L, n_fft, f, 2 ** 40, None) == -1
            assert lib.disco_stft_scm2(f, f, f, 0, f, 1, 2, L, n_fft, f, 2 ** 40, None) == -1
            if n_fft < 1024:
                assert lib.disco_stft_filter_dual(f, f, f, f, f, f, 0, 0, 1, 2, L, n_fft, None) == -1
            assert lib.disco_stft_lengths(f, f, lens, f, 4, L, n_fft, None) == -1
            assert lib.disco_istft(f, f, 4, T, L, n_fft, None) == -1
            assert b"length" in lib.disco_last_error()
            assert lib.disco_istft_lengths(f, f, lens, f, 4, T, L, n_fft, None) == -1


def test_bound_is_the_one_ops_states():
    from disco_b200 import ops
    src = open(os.path.join(CSRC, "api.cu")).read()
    assert "long long max_length(int n_fft) { return (long long)INT_MAX - n_fft - 1024; }" in src
    for n_fft in NFFTS:
        assert ops.max_stream_length(n_fft) == bound(n_fft)
