"""Online Tango streams at and past 2^31 samples (DESIGN §4.5, "Positions").  A frame's spectrum depends only on its
samples and its distance from the two reflections, never on its absolute position: every stream STFT / iSTFT call at
2^30, 2^31, 2^32 and 2^40 samples equals, bit for bit, its twin at a small position congruent mod the hop, and lies
within the float64 bound; a pool launch mixes such slots; a whole signal of 2^30 + r samples keeps its end reflection;
and streams pushed past 2^31 samples of zeros then give exactly what fresh streams give."""
import math
import time

import numpy as np
import pytest
import torch

from test_gpu_kernel_instances import SENTINEL, U, assert_bounded
from test_gpu_stft_instances import hann, pair_envelope, tol_fft
from test_gpu_stream_pool import _guarded, _guards_kept

pytestmark = pytest.mark.gpu

NFFTS = (256, 512, 1024)
BASES = (2 ** 30, 2 ** 31, 2 ** 32, 2 ** 40)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _residues(H):
    return (0, 1, H - 1)


def _twin(A, H):
    """The small position of the twin: congruent to A mod H, 20 hops from the start (no start reflection)."""
    return 20 * H + A % H


class _Signal:
    """Samples [first, first + n) of n_sig random signals, addressed by absolute position."""

    def __init__(self, rng, n_sig, first, n):
        self.first, self.x = first, rng.standard_normal((n_sig, n)).astype(np.float32)

    def at(self, s0, s1):
        return self.x[:, s0 - self.first:s1 - self.first]


def _ref_frames(sig, t0, n_fr, A, n_fft, final):
    """float64 rfft of the windowed frames [t0, t0 + n_fr) of a signal of A samples (end-reflected when final), and
    the per-frame sum_n w |x| of every signal."""
    H = n_fft // 2
    w = hann(n_fft)
    Y, E = [], []
    for t in range(t0, t0 + n_fr):
        s = np.abs(np.arange(t * H - H, t * H + H))           # the start reflection
        if final:
            s = np.where(s >= A, 2 * (A - 1) - s, s)
        seg = sig.x[:, s - sig.first].astype(np.float64)
        Y.append(np.fft.rfft(seg * w, axis=-1))
        E.append(np.abs(seg) @ w)
    return np.stack(Y, axis=1), np.stack(E, axis=1)


def _check_stft64(Y, sig, t0, n_fr, A, n_fft, final, what):
    Yr, Ar = _ref_frames(sig, t0, n_fr, A, n_fft, final)
    n_sig = Yr.shape[0]
    E = pair_envelope(Ar, n_sig, n_sig)
    assert_bounded(Y.cpu().numpy(), Yr, np.broadcast_to(E[:, :, None], Yr.shape), tol_fft(n_fft), what)


def _stft_call(dev, sig, A, n_new, t0, n_fr, n_fft, final, pos):
    """ops.stream_stft at sample count pos (the absolute A, or its twin), reading sig's samples around A."""
    from disco_b200 import ops
    N, H = n_fft, n_fft // 2
    L0 = A - n_new
    hist = torch.from_numpy(np.ascontiguousarray(sig.at(L0 - N, L0))).to(dev)
    chunk = torch.from_numpy(np.ascontiguousarray(sig.at(L0, A))).to(dev)
    n_sig, P = hist.shape[0], n_fr + 3
    ho = torch.full_like(hist, float("nan"))
    yb = torch.full((n_sig, P, H + 1), complex(float("nan"), 0), dtype=torch.complex64, device=dev)
    Y = ops.stream_stft(hist, chunk, pos, t0 - (A - pos) // H, n_fr, n_fft, hist_out=ho, Y_blk=yb, blk_slot=2,
                        final=final)
    return Y, ho, yb


def _stft_cases(n_fft):
    H, N = n_fft // 2, n_fft
    for base in BASES:
        for r in _residues(H):
            A = base + r
            n_new = 3 * H + 5
            t0 = -((N - (A - n_new)) // H) + 1              # the first frame inside the history
            yield "run", A, n_new, t0, A // H - t0, False
            t0 = -((N - A) // H) + 1
            yield "final", A, 0, t0, A // H - t0 + 1, True


@pytest.mark.parametrize("n_fft", NFFTS)
@pytest.mark.parametrize("n_sig", [1, 2, 3])
def test_stream_stft_at_large_positions(dev, n_fft, n_sig):
    H = n_fft // 2
    rng = np.random.default_rng(n_fft + n_sig)
    for kind, A, n_new, t0, n_fr, final in _stft_cases(n_fft):
        what = (kind, n_fft, n_sig, A)
        assert n_fr >= 1, what
        sig = _Signal(rng, n_sig, A - n_new - n_fft, n_new + n_fft)
        Y, ho, yb = _stft_call(dev, sig, A, n_new, t0, n_fr, n_fft, final, A)
        a = _twin(A, H)
        Yt, hot, ybt = _stft_call(dev, sig, A, n_new, t0, n_fr, n_fft, final, a)
        assert torch.equal(Y, Yt) and torch.equal(yb[:, 2:2 + n_fr], ybt[:, 2:2 + n_fr]), what
        assert torch.equal(ho, hot) and torch.equal(ho.cpu(), torch.from_numpy(sig.at(A - n_fft, A))), what
        assert torch.equal(yb[:, 2:2 + n_fr], Y), what
        _check_stft64(Y, sig, t0, n_fr, A, n_fft, final, what)


def _ref_ola(Yh, carry, t0, n_fft, final, n_out):
    """float64 overlap-add of frames [t0, t0 + n_fr) after a carried half frame: the samples the stream writes from
    (t0 - 1) hop on, and an entry-wise bound (4 log2 N + 8) U (w0 |frame| + |carry|) / wss with |frame| bounded by
    2 sum |Y| / N of the signal and its partner."""
    N, H = n_fft, n_fft // 2
    w = hann(N)
    n_fr = Yh.shape[1]
    fr = np.fft.irfft(Yh.astype(np.complex128), n=N, axis=-1)                 # [n_sig, n_fr, N]
    own = 2 * np.abs(Yh).sum(-1) / N                                            # [n_sig, n_fr]
    scale = own.copy()                   # plus the two-for-one partner's: signals 2p, 2p + 1 share a transform
    for s in range(0, Yh.shape[0] - 1, 2):
        scale[s] += own[s + 1]
        scale[s + 1] += own[s]
    prev, prev_env = carry.astype(np.float64), np.abs(carry.astype(np.float64))
    out, env = [], []
    tol = (4 * math.log2(N) + 8) * U
    for i in range(n_fr):
        j = t0 + i
        wss = w[:H] ** 2 + (w[H:] ** 2 if j >= 1 else 0)
        wss = np.where(wss > 1.17549435e-38, wss, 1.0)
        out.append((w[:H] * fr[:, i, :H] + prev) / wss)
        env.append((w[:H] * scale[:, i:i + 1] + prev_env) / wss)
        prev, prev_env = w[H:] * fr[:, i, H:], w[H:] * scale[:, i:i + 1]
    if final:
        wss = np.where(w[H:] ** 2 > 1.17549435e-38, w[H:] ** 2, 1.0)
        out.append(prev / wss)
        env.append(prev_env / wss)
    x, e = np.concatenate(out, axis=1), np.concatenate(env, axis=1)
    assert x.shape[1] >= n_out
    return x[:, :n_out], tol * e[:, :n_out]


@pytest.mark.parametrize("n_fft", NFFTS)
@pytest.mark.parametrize("n_sig", [1, 2, 3])
def test_stream_istft_at_large_positions(dev, n_fft, n_sig):
    from disco_b200 import ops
    H, F = n_fft // 2, n_fft // 2 + 1
    rng = np.random.default_rng(7 * n_fft + n_sig)
    for base in BASES:
        for r in _residues(H):
            A = base + r
            for final, t0, n_fr in ((False, A // H - 6, 5), (True, A // H - 1, 2)):
                what = (final, n_fft, n_sig, A)
                Yh = (rng.standard_normal((n_sig, n_fr, F)) + 1j * rng.standard_normal((n_sig, n_fr, F)))
                Yh = Yh.astype(np.complex64)
                Yh[..., 0].imag = 0
                Yh[..., -1].imag = 0
                c0 = rng.standard_normal((n_sig, H)).astype(np.float32)
                Y = torch.from_numpy(Yh).to(dev)
                outs = []
                for pos in (A, _twin(A, H)):
                    c = torch.from_numpy(c0).to(dev)
                    x = ops.stream_istft(Y, c, t0 - (A - pos) // H, pos, n_fft, final=final)
                    outs.append((x, c))
                (x, c), (xt, ct) = outs
                assert torch.equal(x, xt) and torch.equal(c, ct), what
                want = (A if final else (t0 + n_fr - 1) * H) - (t0 - 1) * H
                assert x.shape[-1] == want, what
                ref, bound = _ref_ola(Yh, c0, t0, n_fft, final, want)
                err = np.abs(x.cpu().numpy().astype(np.float64) - ref)
                assert (err <= bound).all(), (what, float(err.max()), float(bound[err > bound][0]))


@pytest.mark.parametrize("n_fft", NFFTS)
def test_pool_slots_at_mixed_magnitudes(dev, n_fft):
    """One stream_stft_slots and one stream_istft_slots launch: a slot at its start, a final slot at 2^30 + r, slots
    at 2^31 + r and 2^32 + r and an idle slot past 2^33; each equals its lone small-position twin bit for bit, inside
    NaN guard bands, rows past its frames untouched."""
    from disco_b200 import _lib, ops
    H, N, F, n_sig = n_fft // 2, n_fft, n_fft // 2 + 1, 3
    rng = np.random.default_rng(n_fft)
    r = H - 1
    # (A = samples after the chunk, n_new, t0, n_fr, final, hist_write)
    specs = [(3 * H + 5, 3 * H + 5, 0, 3, False, True)]
    A = 2 ** 30 + r
    t0 = -((N - A) // H) + 1
    specs.append((A, 0, t0, A // H - t0 + 1, True, False))
    for base in (2 ** 31, 2 ** 32):
        A, n_new = base + r, 2 * H + 7
        t0 = -((N - (A - n_new)) // H) + 1
        specs.append((A, n_new, t0, A // H - t0, False, True))
    specs.append((2 ** 33 + 5, 0, (2 ** 33 + 5) // H - 1, 0, False, False))
    S = len(specs)
    n_max, f_max, P = max(s[1] for s in specs) + 2, max(s[3] for s in specs), 8
    sigs = [_Signal(rng, n_sig, A - n_new - N, n_new + N) for (A, n_new, *_rest) in specs]
    for s, (A, n_new, *_rest) in enumerate(specs):
        if A - n_new - N < 0:                                   # before sample 0: the zeros a fresh stream holds
            sigs[s].x[:, :N - (A - n_new)] = 0
    hist = torch.full((2, S, n_sig, N), float("nan"), device=dev)
    chunk = torch.full((S, n_sig, n_max), float("nan"), device=dev)
    for s, (A, n_new, *_rest) in enumerate(specs):
        hist[0, s] = torch.from_numpy(sigs[s].at(A - n_new - N, A - n_new)).to(dev)
        chunk[s, :, :n_new] = torch.from_numpy(sigs[s].at(A - n_new, A)).to(dev)
    rec = np.array([[A, n_new, t0, n_fr, 1, int(fin), 0, int(w)] for (A, n_new, t0, n_fr, fin, w) in specs],
                   dtype=np.int64)
    host = ops._records(rec, S, ops.STFT_SLOT_FIELDS, "slots", n_fft)
    fy, Y = _guarded((S, n_sig, f_max, F), torch.complex64, dev)
    fb, Yb = _guarded((S, n_sig, P, F), torch.complex64, dev)
    lib = _lib.load()
    d = torch.from_numpy(host).to(dev)
    hist_before = hist.clone()
    _lib.check(lib.disco_stream_stft_slots(ops._ptr(hist), ops._ptr(chunk), ops._ptr(Y), ops._ptr(Yb), ops._ptr(d),
                                           host.ctypes.data_as(_lib.c_int_p), S, n_sig, n_max, f_max, P, n_fft, None))
    torch.cuda.synchronize()
    assert _guards_kept(fy) and _guards_kept(fb)
    yw, bw = fy[64:-64].view(S, n_sig, f_max, 2 * F), fb[64:-64].view(S, n_sig, P, 2 * F)
    for s, (A, n_new, t0, n_fr, fin, write) in enumerate(specs):
        a = A if A < 4 * N else _twin(A, H)
        ho = torch.zeros((n_sig, N), device=dev)
        want = ops.stream_stft(hist_before[0, s].contiguous(), chunk[s, :, :n_new].contiguous(), a, t0 - (A - a) // H,
                               n_fr, n_fft, hist_out=ho if write else None, final=fin)
        assert torch.equal(Y[s, :, :n_fr], want) and torch.equal(Yb[s, :, 1:1 + n_fr], want), s
        assert (yw[s, :, n_fr:] == SENTINEL).all() and (bw[s, :, :1] == SENTINEL).all(), s
        assert (bw[s, :, 1 + n_fr:] == SENTINEL).all(), s
        if write:
            assert torch.equal(hist[1, s], ho), s
        else:
            assert torch.isnan(hist[1, s]).all(), s
        if n_fr:
            _check_stft64(want, sigs[s], t0, n_fr, A, n_fft, fin, ("pool", n_fft, s))
    # the iSTFT of the same slots: frames t0 .. t0 + n_fr - 1 after a random carry, final slots up to their end
    Yv = torch.from_numpy((rng.standard_normal((S, n_sig, f_max, F)) +
                           1j * rng.standard_normal((S, n_sig, f_max, F))).astype(np.complex64)).to(dev)
    carry = torch.from_numpy(rng.standard_normal((S, n_sig, H)).astype(np.float32)).to(dev)
    carry_before = carry.clone()
    spans = []
    for (A, n_new, t0, n_fr, fin, _w) in specs:
        lo = max(t0 - 1, 0) * H
        hi = min(A, A if fin else (t0 + n_fr - 1) * H)
        spans.append((lo, hi))
    s_max = max(max(hi - lo, 0) for lo, hi in spans) + 5
    irec = np.array([[t0, n_fr, A, int(fin), lo] for (A, n_new, t0, n_fr, fin, _w), (lo, hi) in zip(specs, spans)],
                    dtype=np.int64)
    ihost = ops._records(irec, S, ops.ISTFT_SLOT_FIELDS, "slots", n_fft)
    fx, x = _guarded((S, n_sig, s_max), torch.float32, dev)
    di = torch.from_numpy(ihost).to(dev)
    _lib.check(lib.disco_stream_istft_slots(ops._ptr(Yv), ops._ptr(carry), ops._ptr(x), ops._ptr(di),
                                            ihost.ctypes.data_as(_lib.c_int_p), S, n_sig, f_max, s_max, n_fft, None))
    torch.cuda.synchronize()
    assert _guards_kept(fx)
    xw = fx[64:-64].view(S, n_sig, s_max)
    for s, ((A, n_new, t0, n_fr, fin, _w), (lo, hi)) in enumerate(zip(specs, spans)):
        if n_fr == 0 and not fin:
            assert (xw[s] == SENTINEL).all() and torch.equal(carry[s], carry_before[s]), s
            continue
        a = A if A < 4 * N else _twin(A, H)
        c = carry_before[s].clone()
        want = ops.stream_istft(Yv[s, :, :n_fr].contiguous(), c, t0 - (A - a) // H, a, n_fft, final=fin)
        assert torch.equal(x[s, :, :hi - lo], want) and torch.equal(carry[s], c), s
        assert (xw[s, :, hi - lo:] == SENTINEL).all(), s


def test_whole_signal_stft_past_2_30_samples(dev):
    """One row of 2^30 + r samples through ops.stft at n_fft 512 (about 13 GB): its first and last frames against
    float64, the last one reflected at the end."""
    from disco_b200 import ops
    n_fft, H = 512, 256
    L = 2 ** 30 + 3
    T = 1 + L // H
    need = L * 4 + T * (H + 1) * 8 + (2 << 30)
    free, _ = torch.cuda.mem_get_info(dev)
    if free < need:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free" % (need / 2 ** 30, free / 2 ** 30))
    g = torch.Generator(device=dev).manual_seed(5)
    x = torch.randn((1, L), generator=g, device=dev)
    Y = ops.stft(x, n_fft)
    assert Y.shape == (1, T, H + 1)
    for t_lo, t_hi in ((0, 3), (T - 4, T)):
        s0, s1 = max(t_lo * H - H, 0), min(t_hi * H + H, L)
        sig = _Signal(np.random.default_rng(0), 1, s0, 0)
        sig.x = x[:, s0:s1].cpu().numpy()
        if t_lo == 0:
            # the start reflection: frame t reads |s| for s < 0
            w = hann(n_fft)
            Yr, Er = [], []
            xs = sig.x[0].astype(np.float64)
            for t in range(t_lo, t_hi):
                idx = np.abs(np.arange(t * H - H, t * H + H))
                Yr.append(np.fft.rfft(xs[idx] * w))
                Er.append(np.abs(xs[idx]) @ w)
            Yr, Er = np.stack(Yr)[None], np.stack(Er)[None]
            assert_bounded(Y[:, t_lo:t_hi].cpu().numpy(), Yr, np.broadcast_to(Er[:, :, None], Yr.shape),
                           tol_fft(n_fft), "whole signal, first frames")
        else:
            _check_stft64(Y[:, t_lo:t_hi], sig, t_lo, t_hi - t_lo, L, n_fft, True, "whole signal, last frames")
    del x, Y
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- streams run past 2^31 samples
N_LONG, BLOCK, LAG, C_LONG = 1024, 64, 1, 4
PH = BLOCK * N_LONG // 2
Z_LONG = 2 ** 31 + 3 * PH             # samples of zeros before the signal
Z_TWIN = (LAG + 2) * PH               # the twin's zeros, Z_TWIN = Z_LONG mod PH
ZCHUNK = 2 ** 23


def _chunk_sizes(rng):
    """About five blocks of samples in uneven chunks"""
    H = N_LONG // 2
    sizes = [0, H - 1, H + 1, 3 * H + 7, 17 * H, PH + 5, 2 * PH - 3, 1]
    while sum(sizes) < 5 * PH:
        sizes.append(int(rng.integers(H, 3 * PH)))
    return sizes


def _signal_chunks(rng, shape, sizes):
    return [torch.from_numpy(rng.standard_normal(shape + (n,)).astype(np.float32)) for n in sizes]


def _mask_of(Y):
    p = (Y.real ** 2 + Y.imag ** 2)
    return p / (p + 0.37)


def test_stream_runs_past_2_31_samples(dev):
    """OnlineTangoStream (clean components, K = 1, C = 4, n_fft 1024, block 64, lag 1): 2^31 + 3 P H samples of zeros,
    then a random signal in uneven chunks and the flush, equal bit for bit to a fresh stream given 3 P H zeros and the
    same chunks, with the same Y and masks handed to mask_fn; t0 differs by exactly the extra frames."""
    from disco_b200.stream import OnlineTangoStream
    rng = np.random.default_rng(31)
    sizes = _chunk_sizes(rng)
    chunks, s_chunks, n_chunks = (_signal_chunks(rng, (1, 1, C_LONG), sizes) for _ in range(3))
    runs = []
    for zeros in (Z_LONG, Z_TWIN):
        t_start = time.time()
        seen, recording = [], [False]

        def mask_fn(t0, Y, z_y, zn, seen=seen, recording=recording):
            m = _mask_of(Y[:, :, 0])
            if recording[0]:
                seen.append((t0, Y.clone(), m))
            return m, None
        s = OnlineTangoStream(1, 1, C_LONG, n_fft=N_LONG, block=BLOCK, lag=LAG, device=dev, clean=True)
        zc = torch.zeros((1, 1, C_LONG, ZCHUNK), device=dev)
        left = zeros
        while left:
            n = min(left, ZCHUNK)
            z = zc[..., :n]
            s.push(z, mask_fn, s_chunk=z, n_chunk=z)
            left -= n
        assert s.samples_in == zeros
        recording[0] = True
        outs = []
        for y, sc, nc in zip(chunks, s_chunks, n_chunks):
            outs.append(s.push(y.to(dev), mask_fn, s_chunk=sc.to(dev), n_chunk=nc.to(dev)))
        outs.append(s.flush(mask_fn))
        runs.append((outs, list(seen)))
        print("stream after %d zeros: %.1f s" % (zeros, time.time() - t_start))
    (a, ma), (b, mb) = runs
    dt = (Z_LONG - Z_TWIN) // (N_LONG // 2)
    assert len(a) == len(b) and len(ma) == len(mb) and len(ma) > 5
    for oa, ob in zip(a, b):
        assert oa["t0"] - ob["t0"] == dt
        assert oa.keys() == ob.keys()
        for k in oa:
            if k != "t0":
                assert torch.equal(oa[k], ob[k]), k
    for (ta, Ya, Ma), (tb, Yb, Mb) in zip(ma, mb):
        assert ta - tb == dt and torch.equal(Ya, Yb) and torch.equal(Ma, Mb)


def test_pool_slot_runs_past_2_31_samples(dev):
    """OnlineTangoPool with two slots: slot 0 takes 2^31 + 3 P H zeros, then slot 1 opens and both take random chunks
    in the same launches and close.  Slot 0 equals a one-slot pool given 3 P H zeros and the same chunks, slot 1 a
    fresh one-slot pool, bit for bit, with the same Y and masks handed to mask_fn; t0 / s0 differ by exactly the
    extra frames and samples."""
    from disco_b200.stream import OnlineTangoPool
    K, C, H = 1, 2, N_LONG // 2
    rng = np.random.default_rng(41)
    ch = [_signal_chunks(rng, (K, C), _chunk_sizes(rng)), _signal_chunks(rng, (K, C), _chunk_sizes(rng))]
    n_call = max(len(ch[0]), len(ch[1]))

    def batch(slots, i):
        """the i-th chunk of every listed slot, stacked [S, K, C, n_max]; None past a slot's chunks"""
        cs = [ch[s][i] if i < len(ch[s]) else torch.zeros((K, C, 0)) for s in slots]
        n = [c.shape[-1] for c in cs]
        y = torch.zeros((len(slots), K, C, max(max(n), 1)))
        for j, c in enumerate(cs):
            y[j, :, :, :c.shape[-1]] = c
        return y.to(dev), n

    def make_mask_fn(seen, recording):
        def mask_fn(t0, n_fr, Y, z_y, zn):
            m = _mask_of(Y[:, :, 0])
            if recording[0]:
                seen.append((t0.copy(), n_fr.copy(), Y.clone(), m))
            return m, None
        return mask_fn

    def run(S, prefix_zeros, slot_of):
        """slot_of: which chunk sequence each slot of this pool plays (0 or 1)"""
        seen, recording = [], [False]
        mf = make_mask_fn(seen, recording)
        pool = OnlineTangoPool(S, K, C, n_fft=N_LONG, block=BLOCK, lag=LAG, device=dev)
        if 0 in slot_of:
            i0 = slot_of.index(0)
            pool.open([i0])
            zc = torch.zeros((S, K, C, ZCHUNK), device=dev)
            left = prefix_zeros
            while left:
                n = min(left, ZCHUNK)
                pool.push(zc[..., :n], [n if s == i0 else 0 for s in range(S)], mf)
                left -= n
        if 1 in slot_of:
            pool.open([slot_of.index(1)])
        recording[0] = True
        outs = []
        for i in range(n_call):
            y, n = batch(slot_of, i)
            outs.append(pool.push(y, n, mf))
        outs.append(pool.close(list(range(S)), mf))
        return outs, seen

    t_start = time.time()
    both, seen2 = run(2, Z_LONG, [0, 1])
    print("long pool: %.1f s for %d samples" % (time.time() - t_start, Z_LONG))
    lone0, seen0 = run(1, Z_TWIN, [0])
    lone1, seen1 = run(1, 0, [1])
    dt = (Z_LONG - Z_TWIN) // H
    for s, (lone, seen_l, shift) in enumerate(((lone0, seen0, dt), (lone1, seen1, 0))):
        assert len(lone) == len(both)
        for ob, ol in zip(both, lone):
            assert ob["t0"][s] - ol["t0"][0] == shift and ob["s0"][s] - ol["s0"][0] == shift * H
            assert ob["frames"][s] == ol["frames"][0] and ob["samples"][s] == ol["samples"][0]
            f, n = int(ob["frames"][s]), int(ob["samples"][s])
            for k in ("z_y", "zn", "yf"):
                assert torch.equal(ob[k][s, :, :f], ol[k][0, :, :f]), (s, k)
            assert torch.equal(ob["yf_time"][s, :, :n], ol["yf_time"][0, :, :n]), s
        # the Y and masks of each round, slot by slot (rows past a slot's frames are not defined)
        mine = [(t[s], nr[s], Y[s, :, :, :nr[s]], m[s, :, :nr[s]]) for t, nr, Y, m in seen2 if nr[s] > 0]
        theirs = [(t[0], nr[0], Y[0, :, :, :nr[0]], m[0, :, :nr[0]]) for t, nr, Y, m in seen_l if nr[0] > 0]
        assert len(mine) == len(theirs) > 5
        for (ta, na, Ya, Ma), (tb, nb, Yb, Mb) in zip(mine, theirs):
            assert ta - tb == shift and na == nb and torch.equal(Ya, Yb) and torch.equal(Ma, Mb)
