"""The kernels after the beamformer -- iSTFT, the metric filter bank, the oracle masks and the layout kernels -- at
every instantiation and launch-plan edge against float64, through the C ABI with every output inside a NaN-filled
guard band.

Dispatch targets (tests/test_post_instances_cpu.py parses the sets and the plan constants mirrored here out of the
sources, so a retuned launcher fails on CPU instead of moving these cases off their edges):
  istft       istft.cu       istft_kernel<N>, N = 256 / 512 / 1024: one CTA per (signal pair, chunk of hop blocks)
  band_stats  filterbank.cu  band_stats_kernel<NC>, NC = order + 1 for filter orders 2 / 4 / 8 / 16: lanes = 32
                             signals, 1..kBankWarps band-warps per CTA sharing one cp.async tile
  misc        misc.cu        tf_mask_kernel, apply_mask_kernel, transpose_kernel<float / float2>

iSTFT bound (u = 2^-24, w the periodic Hann window, H = N / 2).  Output sample s = (j - 1) H + n of hop block j is
    x[s] = (w[n] f_j[n] + w[n+H] f_{j-1}[n+H]) / wss[n],   wss[n] = w[n]^2 + w[n+H]^2
with f_t the inverse real FFT of frame t (including 1/N).  The kernel transforms the complex spectrum Z = A + iB of a
signal pair in one float32 FFT of log2 N radix-2-equivalent stages.  A stage rounds each butterfly output with at
most 4 roundings of a value bounded by the sum of the moduli of the inputs feeding it, and the nodes one output
depends on at a stage partition the inputs, so (as for the STFT, DESIGN §2)
    |Δ f_t[n]| <= eps * m_t,   m_t = (1/N) Σ_k |Z_t[k]|,   eps = sqrt(2) (4 log2 N + 6) u
(6: the gather of A + iB, the twiddle and 1/N roundings).  The window products, the float32 window itself, the sum of
the two halves, wss (two squares of rounded window values and their sum, 4u relative) and its reciprocal and product
add at most c = 10 roundings relative to the magnitudes, so entry-wise
    |Δx[s]| <= [eps (w[n] m_j + w[n+H] m_{j-1}) + c u (|w[n] f_j[n]| + |w[n+H] f_{j-1}[n+H]|)] / wss[n].
The tail block j = j_end has only the second term (wss = w[n+H]^2); samples past it are zero exactly.  m_t is taken over
the pair's combined spectrum, so the partner's magnitude enters.  The yardstick is oracle.librosa_np.istft in float64
of the same complex64 spectra.

tf_mask bound, in float32 ulps relative (rho = 2^-23): hypotf is within h = 3 ulps (CUDA Math API), the division and
each product round once (1/2 ulp), s + n rounds per component (1/2 ulp of |s + n|).  The ratio errs by 2h + 1/2
(irm / ibm) or 2h + 1 (iam), p - 1 rounded products raise it to the p-th power, and irm's 1 + xi and division add 1:
    |Δm| <= K(p) rho |m|,   K(p) = (2h + 3/2) p + 1 = 7.5 p + 1.
ibm decisions are exact wherever the float64 xi is further than K(p) + 2 ulps from the threshold.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import librosa_np, lfilter_np, tango_np

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
RHO = 2.0 ** -23
SENT32 = 0x7FC0DEAD               # a quiet-NaN bit pattern no kernel computes
SENT64 = 0x7FF8DEADDEADBEEF
GUARD = 1024                      # words of sentinel before and after every output

# ---- launch-plan constants mirrored from the sources (checked against them on CPU) --------------------------------
ISTFT_NFFTS = (256, 512, 1024)    # launch_istft's switch
ISTFT_ITEMS = 16                  # IGeom<N>::ITEMS: frames per shared-memory tile; fpc is a multiple of it
ISTFT_MIN_TILES = 4               # a chunk is split only while it keeps more than 4 * ITEMS hop blocks
ISTFT_CTAS_PER_SM = 2             # chunks double while pairs * chunks < sm_count() * 2
BANK_ORDERS = (2, 4, 8, 16)       # launch_band_stats' switch (filter orders; NC = order + 1)
BANK_WARPS = 8                    # kBankWarps: at most this many bands per CTA
BANK_CHUNK = 64                   # kBankChunk: samples per shared-memory chunk
GRID_YZ = 65535


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def cdiv(a, b):
    return -(-a // b)


# ---- launch plans -------------------------------------------------------------------------------------------------

def istft_plan(n_sig, T, L, n_fft, sms):
    """launch_n<N> of a whole-signal call: (j_end, chunks after doubling, chunks launched, fpc)."""
    H = n_fft // 2
    pairs = (n_sig + 1) // 2
    j_end = min(T, (L + n_fft + H - 1) // H)
    chunks = 1
    while pairs * chunks < sms * ISTFT_CTAS_PER_SM and cdiv(j_end, chunks) > ISTFT_MIN_TILES * ISTFT_ITEMS:
        chunks *= 2
    fpc = cdiv(cdiv(j_end, chunks), ISTFT_ITEMS) * ISTFT_ITEMS
    return j_end, chunks, cdiv(j_end, fpc), fpc


def bank_bpc(n_sig, n_band, sms):
    """launch_band_stats: bands (warps) per CTA."""
    sig_blocks = cdiv(n_sig, 32)
    b = min(n_band, BANK_WARPS)
    while b > 1 and sig_blocks * cdiv(n_band, b) < sms:
        b -= 1
    return b


# ---- guarded outputs ----------------------------------------------------------------------------------------------

class Guarded:
    """Outputs carved out of buffers filled with a NaN bit pattern; check() asserts that every output word was
    written and no guard word changed."""

    def __init__(self, dev):
        self.dev, self.bufs = dev, []

    def new(self, shape, dtype):
        n = int(np.prod(shape))
        if dtype == torch.float64:
            wdt, sent = torch.int64, SENT64
        else:
            wdt, sent = torch.int32, SENT32
            n *= 2 if dtype == torch.complex64 else 1
        buf = torch.full((n + 2 * GUARD,), sent, dtype=wdt, device=self.dev)
        self.bufs.append((buf, n, sent))
        return buf[GUARD:GUARD + n].view(dtype).view(shape)

    def check(self, what):
        torch.cuda.synchronize()
        for i, (buf, n, sent) in enumerate(self.bufs):
            assert bool((buf[:GUARD] == sent).all()), "%s: output %d: write before its start" % (what, i)
            assert bool((buf[GUARD + n:] == sent).all()), "%s: output %d: write past its end" % (what, i)
            left = int((buf[GUARD:GUARD + n] == sent).sum())
            assert left == 0, "%s: output %d: %d of %d words never written" % (what, i, left, n)
        self.bufs = []


def _call(fn, *args):
    from disco_b200 import _lib, ops
    _lib.check(getattr(_lib.load(), fn)(*args, ops._stream()))


def _p(t):
    from disco_b200 import ops
    return ops._ptr(t)


def cplx(rng, *s):
    return (rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)


# ==== A. iSTFT =====================================================================================================

def istft_dev(dev, Y, L, n_fft, what):
    """disco_istft of Y [n_sig, T, F] (device complex64) into a guarded [n_sig, L] output."""
    n_sig, T, _ = Y.shape
    g = Guarded(dev)
    x = g.new((n_sig, L), torch.float32)
    _call("disco_istft", _p(Y), _p(x), n_sig, T, L, n_fft)
    g.check(what)
    return x


def _pair_m(Yc):
    """m_t = (1/N) Σ_k |Z_t[k]| of the pair spectrum Z = A + iB of signals (2p, 2p + 1), for every signal of
    Yc [n_sig, T, F] (complex128); a last unpaired signal has B = 0."""
    n_sig, T, F = Yc.shape
    N = 2 * (F - 1)
    # Σ_k |Z[k]| is symmetric in A and B (|conj A + i conj B| = |A - iB| = |B + iA|), so each signal of a pair can
    # take the other as its B
    e = 2 * (n_sig // 2)
    B = np.zeros_like(Yc)
    B[0:e:2] = Yc[1:e:2]
    B[1:e:2] = Yc[0:e:2]
    A = Yc
    A_, B_ = A[..., 1:-1], B[..., 1:-1]
    m = (np.abs(A[..., 0].real + 1j * B[..., 0].real) + np.abs(A[..., -1].real + 1j * B[..., -1].real) +
         np.abs(A_ + 1j * B_).sum(-1) + np.abs(np.conj(A_) + 1j * np.conj(B_)).sum(-1)) / N
    return m


def istft_bound(Yh, L, n_fft, frame_window=None):
    """(float64 overlap-add of the frames, entry-wise bound) for Yh [n_sig, T, F] complex64 -> [n_sig, L] each.
    frame_window = (j, w_j) replaces the window of frame j (a negative control)."""
    n_sig, T, F = Yh.shape
    N, H = n_fft, n_fft // 2
    j_end = min(T, (L + N + H - 1) // H)
    Yc = Yh[:, :j_end].astype(np.complex128)
    fr = np.fft.irfft(Yc, n=N, axis=-1)                           # [n_sig, j_end, N]
    m = _pair_m(Yc)                                               # [n_sig, j_end]
    w = librosa_np.hann_periodic(N)
    W = np.broadcast_to(w, (j_end, N)).copy()
    if frame_window is not None:
        W[frame_window[0]] = frame_window[1]
    eps = math.sqrt(2) * (4 * math.log2(N) + 6) * U
    c = 10.0
    s = np.arange(L)
    j, n = s // H + 1, s % H
    inner, tail = j < j_end, j == j_end
    jc, jp = np.minimum(j, j_end - 1), np.minimum(j - 1, j_end - 1)
    a0 = np.where(inner, W[jc, n], 0.0)                            # window of frame j at n (0 past the frames)
    a1 = np.where(inner | tail, W[jp, n + H], 0.0)                 # window of frame j - 1 at n + H
    wss = np.where(inner, w[n] ** 2 + w[n + H] ** 2, np.where(tail, w[n + H] ** 2, 1.0))
    t0 = a0 * fr[:, jc, n]
    t1 = a1 * fr[:, jp, n + H]
    val = (t0 + t1) / wss
    bound = (eps * (a0 * m[:, jc] + a1 * m[:, jp]) + c * U * (np.abs(t0) + np.abs(t1))) / wss
    return val, bound


def check_istft(got, ref, bound, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= bound)
    assert not bad.any(), "%s: %d samples beyond the bound, first at %s: got %r want %r bound %r" % (
        what, int(bad.sum()), np.argwhere(bad)[0], got[bad][0], ref[bad][0], bound[bad][0])


def istft_check_batch(dev, Yh, L, n_fft, what, Y=None):
    """Run disco_istft on Yh and check every sample against librosa_np's float64 iSTFT under the bound."""
    n_sig = Yh.shape[0]
    if Y is None:
        Y = torch.from_numpy(Yh).to(dev)
    x = istft_dev(dev, Y, L, n_fft, what).cpu().numpy()
    H = n_fft // 2
    step = max(1, (1 << 24) // max(1, Yh.shape[1] * n_fft))        # signals per host batch (bounded memory)
    step += step % 2
    for s0 in range(0, n_sig, step):
        sl = slice(s0, min(n_sig, s0 + step))
        ref = np.stack([librosa_np.istft(Yh[s].T, hop_length=H, win_length=n_fft, length=L, dtype=np.float64)
                        for s in range(sl.start, sl.stop)])
        val, bound = istft_bound(Yh[sl], L, n_fft)
        # the bound's own overlap-add restates the oracle (a self-check of the formula the bound is built on)
        assert np.allclose(val, ref, rtol=0, atol=1e-12 * max(1.0, np.abs(ref).max()))
        check_istft(x[sl], ref, bound, what)
    return x


def istft_lengths(T, n_fft):
    """L = 1; L ending anywhere in the last hop of T frames; L that truncates the frames used; L past the tail."""
    H, N = n_fft // 2, n_fft
    out = {1}
    base = (T - 1) * H
    for r in (0, 1, H // 2, H - 1):
        if base + r >= 1:
            out.add(base + r)
    if T > 4:
        out.add((T - 4) * H + 7)       # ceil((L + N) / H) < T: j_end truncated
    out.add(T * H + N + 37)            # zero-filled tail
    return sorted(out)


ISTFT_FRAMES = (1, 2, 15, 16, 17, 64, 65, 4 * ISTFT_ITEMS * 2 - 1, 4 * ISTFT_ITEMS * 2 + 1,
                4 * ISTFT_ITEMS * 4 - 1, 4 * ISTFT_ITEMS * 4 + 1)


@pytest.mark.parametrize("n_fft", ISTFT_NFFTS)
def test_istft_frames_and_lengths(dev, sms, n_fft):
    """Every frame count edge at every length class, 3 signals (the last without a partner; chunked plans above 64
    blocks)."""
    rng = np.random.default_rng(n_fft)
    F = n_fft // 2 + 1
    for T in ISTFT_FRAMES:
        Yh = cplx(rng, 3, T, F)
        for L in istft_lengths(T, n_fft):
            istft_check_batch(dev, Yh, L, n_fft, ("frames", n_fft, T, L, istft_plan(3, T, L, n_fft, sms)))


def istft_plan_cases(n_fft, sms):
    """(label, n_sig, T) at the edges of launch_n's plan, each asserted to land where its label says."""
    target = sms * ISTFT_CTAS_PER_SM
    cases = [("one_chunk", 2 * target, 4 * ISTFT_ITEMS + 1),        # pairs = 2 SMs: no split despite 65 blocks
             ("two_chunks_odd", 2 * sms - 1, 8 * ISTFT_ITEMS + 1)]   # pairs = SMs: one doubling; odd signal count
    c_max = 1
    while 2 * c_max < target:
        c_max *= 2
    cases.append(("max_chunks_odd", 3, ISTFT_MIN_TILES * ISTFT_ITEMS * (c_max // 2) + 1))   # stopped by the SM bound
    found = {}
    for T in range(4 * ISTFT_ITEMS + 1, 4000):
        _, _, ch, fpc = istft_plan(2, T, (T - 1) * (n_fft // 2), n_fft, sms)
        last = T - (ch - 1) * fpc
        if ch > 1 and last == 1 and "last_one" not in found:
            found["last_one"] = T
        if ch > 1 and last > ISTFT_ITEMS and last % ISTFT_ITEMS == 1 and "last_items_plus_one" not in found:
            found["last_items_plus_one"] = T
    assert len(found) == 2, found
    cases += [("last_chunk_one_block", 2, found["last_one"]), ("last_chunk_items_plus_one", 1, found["last_items_plus_one"])]
    return cases


@pytest.mark.parametrize("n_fft", ISTFT_NFFTS)
def test_istft_plan_edges(dev, sms, n_fft):
    rng = np.random.default_rng(7 + n_fft)
    F, H = n_fft // 2 + 1, n_fft // 2
    target = sms * ISTFT_CTAS_PER_SM
    for label, n_sig, T in istft_plan_cases(n_fft, sms):
        L = (T - 1) * H + H // 2
        j_end, doubled, chunks, fpc = istft_plan(n_sig, T, L, n_fft, sms)
        pairs = (n_sig + 1) // 2
        if label == "one_chunk":
            assert chunks == 1 and j_end > ISTFT_MIN_TILES * ISTFT_ITEMS and pairs >= target
        elif label == "two_chunks_odd":
            assert chunks == 2 and n_sig % 2 == 1
        elif label == "max_chunks_odd":
            assert pairs * doubled >= target and pairs * doubled // 2 < target and n_sig % 2 == 1 and chunks > 1
        elif label == "last_chunk_one_block":
            assert chunks > 1 and j_end - (chunks - 1) * fpc == 1
        else:
            assert chunks > 1 and (j_end - (chunks - 1) * fpc) % ISTFT_ITEMS == 1
        Yh = cplx(rng, n_sig, T, F)
        istft_check_batch(dev, Yh, L, n_fft, (label, n_fft, n_sig, T, L, chunks, fpc))


@pytest.mark.parametrize("n_fft", ISTFT_NFFTS)
def test_istft_seam_and_batch_invariance(dev, sms, n_fft):
    """A signal pair gives the same bits at pair position 0 and later, in a one-chunk batch and in a many-chunk batch
    (the chunk seam recomputes the frame before its first block), and a whole batch equals one call per plan class."""
    rng = np.random.default_rng(11 + n_fft)
    F, H = n_fft // 2 + 1, n_fft // 2
    T = 8 * ISTFT_ITEMS + 1
    L = (T - 1) * H + 3
    pair = torch.from_numpy(cplx(rng, 2, T, F)).to(dev)
    target = sms * ISTFT_CTAS_PER_SM
    n_big = 2 * target + 2 * sms + 1          # odd: the last signal has no partner
    assert istft_plan(n_big, T, L, n_fft, sms)[2] == 1 and istft_plan(4, T, L, n_fft, sms)[2] > 1
    g = torch.Generator(device=dev).manual_seed(n_fft)
    big = torch.complex(torch.randn((n_big, T, F), device=dev, generator=g),
                        torch.randn((n_big, T, F), device=dev, generator=g))
    late = 2 * (sms + 3)
    big[0:2] = pair
    big[late:late + 2] = pair
    small = torch.cat([pair, pair])
    xb = istft_dev(dev, big, L, n_fft, "seam big")
    xs = istft_dev(dev, small, L, n_fft, "seam small")
    want = xb[0:2]
    for got in (xb[late:late + 2], xs[0:2], xs[2:4]):
        assert torch.equal(got, want)
    # the big batch cut into one call per plan class: 2 SMs of pairs (1 chunk), SMs pairs (2 chunks), the unpaired
    # last signal (3 chunks)
    cuts = [0, 2 * target, 2 * target + 2 * sms, n_big]
    parts = [istft_dev(dev, big[a:b].contiguous(), L, n_fft, "part") for a, b in zip(cuts[:-1], cuts[1:])]
    plans = [istft_plan(b - a, T, L, n_fft, sms)[2] for a, b in zip(cuts[:-1], cuts[1:])]
    assert len(set(plans)) == 3, plans
    assert torch.equal(torch.cat(parts), xb)


@pytest.mark.parametrize("n_fft", ISTFT_NFFTS)
def test_istft_negative_controls(dev, sms, n_fft):
    """The checker rejects what a subtly wrong kernel gives: a hop block from the neighbouring frame, one sample
    off by 1e-3, the partner's samples, the window of one frame shifted by a sample."""
    rng = np.random.default_rng(3 + n_fft)
    F, H = n_fft // 2 + 1, n_fft // 2
    T, L = 40, 39 * H + 5
    Yh = cplx(rng, 2, T, F)
    x = istft_check_batch(dev, Yh, L, n_fft, "controls")
    ref = np.stack([librosa_np.istft(Yh[s].T, hop_length=H, win_length=n_fft, length=L, dtype=np.float64)
                    for s in range(2)])
    _, bound = istft_bound(Yh, L, n_fft)
    j = 17
    blk = slice((j - 1) * H, j * H)
    bad = x.copy()
    bad[0, blk] = x[0, j * H:(j + 1) * H]
    with pytest.raises(AssertionError):
        check_istft(bad, ref, bound, "neighbouring block")
    bad = x.copy()
    k = int(np.argmax(np.abs(ref[0])))
    bad[0, k] = np.float32(x[0, k] * (1 + 1e-3))
    with pytest.raises(AssertionError):
        check_istft(bad, ref, bound, "scaled sample")
    with pytest.raises(AssertionError):
        check_istft(x[::-1].copy(), ref, bound, "partner")
    w = librosa_np.hann_periodic(n_fft)
    shifted, _ = istft_bound(Yh, L, n_fft, frame_window=(j, np.roll(w, 1)))
    with pytest.raises(AssertionError):
        check_istft(shifted.astype(np.float32), ref, bound, "shifted window")


# ==== B. band_stats ================================================================================================

def bank_ba(order, n_band, scale=1.0, fs=16000):
    """[n_band, 2, order + 1] (b, a) rows cycling over post's third-octave band-passes of filter order `order`
    (prototype order / 2).  Order 16 keeps the bands from 1 kHz up: below, its transfer-function form is unstable
    (pole radius > 1), as in the reference's helper."""
    from disco_b200 import post
    F, _ = post.third_octave_bands(fs)
    b, a = post.third_octave_filterbank(F, fs, order=order // 2)
    if order == 16:
        keep = np.array([i for i in range(len(F)) if np.abs(np.roots(a[i])).max() < 1.0])
        b, a = b[keep], a[keep]
    idx = np.arange(n_band) % len(b)
    return np.stack([b[idx], a[idx]], axis=1) * scale


def stats_ref(y, sel):
    """(cnt, sum, sq) of the restated outputs y [n_sig, n_band, L]: sequential sums over the selected samples."""
    take = (y != 0.0) if sel is None else np.broadcast_to((sel != 0)[:, None, :], y.shape)
    v = np.where(take, y, 0.0)
    return take.sum(-1).astype(np.float64), np.cumsum(v, axis=-1)[..., -1], np.cumsum(v * v, axis=-1)[..., -1]


def check_stats(got, cnt, sm, sq, what):
    """cnt exact; sum bit-equal to the sequential float64 sum of scipy-exact outputs; sq (fma-accumulated) within
    2 n 2^-53 sq."""
    assert np.array_equal(got[..., 0], cnt), (what, "count", np.argwhere(got[..., 0] != cnt)[:3])
    neq = got[..., 1] != sm
    assert not neq.any(), (what, "sum not bit-equal", np.argwhere(neq)[:3], got[..., 1][neq][:3], sm[neq][:3])
    err = np.abs(got[..., 2] - sq)
    assert np.all(err <= 2 * cnt * 2.0 ** -53 * sq), (what, "sum of squares", float((err / np.maximum(sq, 1e-300)).max()))


def band_stats_dev(dev, xh, ba, sel=None, ld=None, off=0, what=""):
    """disco_band_stats through the C ABI with rows `ld` floats apart and x starting `off` floats into its buffer."""
    n_sig, L = xh.shape
    ld = ld or L
    n_band, _, nc = ba.shape
    flat = np.zeros(off + n_sig * ld, np.float32)
    rows = flat[off:].reshape(n_sig, ld)
    rows[:, :L] = xh
    rows[:, L:] = np.nan                                   # the gaps between rows are never read
    xd = torch.from_numpy(flat).to(dev)
    sd = None
    if sel is not None:
        sflat = np.full(off + n_sig * ld, np.nan, np.float32)
        sflat[off:].reshape(n_sig, ld)[:, :L] = sel
        sd = torch.from_numpy(sflat).to(dev)
    bad = torch.from_numpy(np.ascontiguousarray(ba)).to(dev)
    g = Guarded(dev)
    st = g.new((n_sig, n_band, 3), torch.float64)
    _call("disco_band_stats", _p(xd[off:]), _p(sd[off:]) if sd is not None else None, _p(bad), _p(st), n_sig, L,
          ctypes.c_longlong(ld), n_band, nc - 1)
    g.check(what)
    return st.cpu().numpy()


def band_inputs(rng, n_sig, L):
    """Signals with an all-zero row (1) and an exactly zero prefix (2), and a selection with an all-zero row (3)."""
    x = rng.standard_normal((n_sig, L)).astype(np.float32)
    if n_sig > 2:
        x[1] = 0.0
        x[2, :min(L - 1, 37)] = 0.0
    sel = (rng.uniform(size=(n_sig, L)) > 0.4).astype(np.float32)
    if n_sig > 3:
        sel[3] = 0.0
    return x, sel


def run_band_case(dev, rng, n_sig, n_band, L, order, scale=1.0, ld=None, off=0, what=""):
    ba = bank_ba(order, n_band, scale)
    x, sel = band_inputs(rng, n_sig, L)
    y = lfilter_np.lfilter_plane(ba[:, 0], ba[:, 1], x)
    for s in (None, sel):
        got = band_stats_dev(dev, x, ba, s, ld=ld, off=off, what=what)
        check_stats(got, *stats_ref(y, s), (what, "sel" if s is not None else "nonzero"))
    if n_sig > 2:       # the zero prefix is excluded exactly, the zero signal has no sample
        cnt = band_stats_dev(dev, x, ba, None, ld=ld, off=off, what=what)[..., 0]
        assert np.all(cnt[1] == 0) and np.all(cnt[2] <= L - min(L - 1, 37))


def bank_geometries(sms):
    """(n_sig, n_band) for every bands-per-CTA value 1..8, preferring a dead-warp last CTA row and n_sig % 32 != 0."""
    out = {}
    for sb in range(1, 65):
        n_sig = 32 * sb - 5
        for n_band in range(1, 18):
            b = bank_bpc(n_sig, n_band, sms)
            dead = b > 1 and n_band % b != 0
            if b not in out or (dead and not out[b][2]):
                out[b] = (n_sig, n_band, dead)
    assert set(out) == set(range(1, BANK_WARPS + 1)), sorted(out)
    assert any(d for _, _, d in out.values())
    return {b: v[:2] for b, v in out.items()}


def test_band_stats_geometries(dev, sms):
    """Every bands-per-CTA value, each at a different filter order, on short signals."""
    rng = np.random.default_rng(1)
    for b, (n_sig, n_band) in sorted(bank_geometries(sms).items()):
        order = BANK_ORDERS[b % len(BANK_ORDERS)]
        run_band_case(dev, rng, n_sig, n_band, 150 if n_sig > 512 else 129, order, what=("bpc", b, n_sig, n_band, order))


@pytest.mark.parametrize("order", BANK_ORDERS)
def test_band_stats_lengths_and_layout(dev, order):
    """Lengths around the 64-sample chunk, strided rows and a misaligned x, a bank with a[0] != 1."""
    rng = np.random.default_rng(order)
    for L in (1, BANK_CHUNK - 1, BANK_CHUNK, BANK_CHUNK + 1, 2 * BANK_CHUNK, 2 * BANK_CHUNK + 1):
        run_band_case(dev, rng, 37, 5, L, order, what=("L", order, L))
    run_band_case(dev, rng, 35, 6, 200, order, ld=203, off=1, what=("strided", order))
    run_band_case(dev, rng, 33, 4, 130, order, ld=131, off=3, scale=3.7, what=("a0 = 3.7", order))


def test_band_stats_long(dev):
    """One long signal set (fw_snr's order-8 bank, all 17 bands)."""
    rng = np.random.default_rng(20000)
    run_band_case(dev, rng, 33, 17, 20011, 8, off=2, what="long")


def test_band_stats_negative_controls(dev):
    rng = np.random.default_rng(5)
    ba = bank_ba(8, 17)
    x, _ = band_inputs(rng, 34, 300)
    y = lfilter_np.lfilter_plane(ba[:, 0], ba[:, 1], x)
    got = band_stats_dev(dev, x, ba, what="controls")
    cnt, sm, sq = stats_ref(y, None)
    check_stats(got, cnt, sm, sq, "controls")
    v = np.where(y[0, 0] != 0, y[0, 0], 0.0)
    v[150] = 0.0
    bad_sum = sm.copy()
    bad_sum[0, 0] = np.cumsum(v)[-1]
    with pytest.raises(AssertionError):
        check_stats(got, cnt, bad_sum, sq, "dropped sample")
    bad_cnt = cnt.copy()
    bad_cnt[5, 3] += 1
    with pytest.raises(AssertionError):
        check_stats(got, bad_cnt, sm, sq, "count")
    yf = lfilter_np.lfilter_plane(ba[:, 0], ba[:, 1], x, fma=True)
    with pytest.raises(AssertionError):
        check_stats(got, *stats_ref(yf, None), "fma recurrence")


# ==== C. tf_mask, apply_mask, transpose ============================================================================

def k_ulps(p):
    return 7.5 * p + 1


def tf_mask_dev(dev, S, N, kind, p, thr_db=0.0, what=""):
    from disco_b200 import ops
    Sd, Nd = torch.from_numpy(S).to(dev), torch.from_numpy(N).to(dev)
    g = Guarded(dev)
    M = g.new(S.shape, torch.float32)
    _call("disco_tf_mask", _p(Sd), _p(Nd), _p(M), S.size, ops.MASK_KINDS[kind], p, ctypes.c_float(thr_db))
    g.check(what)
    return M.cpu().numpy()


def mask_f64(S, N, kind, p, thr_db=0.0):
    s, n = S.astype(np.complex128), N.astype(np.complex128)
    if kind == "iam":
        return (np.abs(s) / np.abs(s + n)) ** p
    xi = (np.abs(s) / np.maximum(np.abs(n), float(np.float32(2.220446049250313e-16)))) ** p
    return xi / (1 + xi) if kind == "irm" else xi


@pytest.mark.parametrize("kind", ["irm", "ibm", "iam"])
@pytest.mark.parametrize("p", [1, 2, 3])
def test_tf_mask_against_float64(dev, kind, p):
    rng = np.random.default_rng(p * 10 + len(kind))
    for n in (1, 255, 257, 1_000_003):
        S, N = cplx(rng, n), cplx(rng, n)
        for thr in ((0.0, 3.0, -5.0) if kind == "ibm" else (0.0,)):
            got = tf_mask_dev(dev, S, N, kind, p, thr, (kind, p, n, thr))
            ref = mask_f64(S, N, kind, p)
            if kind == "ibm":
                t = 10.0 ** (thr / 10.0)
                clear = np.abs(ref - t) > (k_ulps(p) + 2) * RHO * t
                assert np.array_equal(got[clear], (ref[clear] >= t).astype(np.float32)), (p, n, thr)
                assert np.all((got == 0) | (got == 1))
            else:
                err = np.abs(got - ref)
                assert np.all(err <= k_ulps(p) * RHO * np.abs(ref)), (kind, p, n, float((err / np.abs(ref)).max() / RHO))


def test_tf_mask_exact_ties(dev):
    """|s| / |n| = 1 exactly at 0 dB: s = 3 + 4i, n = 5 (and n = 5i) give 1 at every power."""
    S = np.array([3 + 4j, 3 - 4j, -4 + 3j], np.complex64)
    N = np.array([5 + 0j, 5j, 5 + 0j], np.complex64)
    for p in (1, 2, 3):
        np.testing.assert_array_equal(tf_mask_dev(dev, S, N, "ibm", p, 0.0), 1.0)


def _cls(v):
    """Special-value class of every entry: nan, +inf, -inf, 0, 1 or other."""
    c = np.full(v.shape, "x", dtype=object)
    c[v == 0] = "0"
    c[v == 1] = "1"
    c[np.isposinf(v)] = "+inf"
    c[np.isneginf(v)] = "-inf"
    c[np.isnan(v)] = "nan"
    return c


@pytest.mark.parametrize("kind", ["irm", "ibm", "iam"])
@pytest.mark.parametrize("p", [1, 2, 3])
def test_tf_mask_special_values(dev, kind, p):
    """NaN / inf / 0 / 1 where numpy's float32 evaluation of the reference formula has them: |n| = 0 (the eps clamp),
    s = 0, s = -n, |s| / eps overflowing at power 2, infinities."""
    inf = np.float32(np.inf)
    S = np.array([1 + 1j, 0, 0, 2 - 1j, 1e4, 1e4j, 1e-30, 0, inf, 1, 3e38, 1 + 1j, -2 + 5j], np.complex64)
    N = np.array([0, 1 + 1j, 0, -2 + 1j, 0, 0, 0, 1e-30, 1, inf, 3e38, 1e-45, 2 - 5j], np.complex64)
    got = tf_mask_dev(dev, S, N, kind, p, 0.0, (kind, p))
    with np.errstate(all="ignore"):
        want = np.asarray(tango_np.tf_mask(S, N, "%s%d" % (kind, p), 0.0)).astype(np.float32)
    np.testing.assert_array_equal(_cls(got), _cls(want), err_msg="%s%d: got %s want %s" % (kind, p, got, want))


def test_tf_mask_negative_control(dev):
    rng = np.random.default_rng(9)
    S, N = cplx(rng, 4096), cplx(rng, 4096)
    got = tf_mask_dev(dev, S, N, "irm", 2)
    ref = mask_f64(S, N, "irm", 2)
    bad = got.copy()
    k = int(np.argmax(ref))
    bad[k] *= np.float32(1 + 64 * RHO * k_ulps(2))
    assert np.all(np.abs(got - ref) <= k_ulps(2) * RHO * ref)
    assert not np.all(np.abs(bad - ref) <= k_ulps(2) * RHO * ref)


@pytest.mark.parametrize("one_minus", [False, True])
def test_apply_mask_both_entry_points(dev, one_minus):
    rng = np.random.default_rng(int(one_minus))
    om = 1 if one_minus else 0
    for shape in ((1,), (255,), (3, 7, 257)):
        X = torch.from_numpy(cplx(rng, *shape)).to(dev)
        m = torch.from_numpy(rng.uniform(-0.5, 1.5, size=shape).astype(np.float32)).to(dev)
        g = Guarded(dev)
        out = g.new(shape, torch.complex64)
        _call("disco_apply_mask", _p(X), _p(m), _p(out), X.numel(), om)
        g.check(("apply_mask", shape))
        w = (1 - m) if one_minus else m
        assert torch.equal(torch.view_as_real(out), torch.view_as_real(X) * w[..., None])
    for chans in range(1, 9):
        G, T, F = 3, 5, 129
        X = torch.from_numpy(cplx(rng, G, chans, T, F)).to(dev)
        m = torch.from_numpy(rng.uniform(size=(G, T, F)).astype(np.float32)).to(dev)
        g = Guarded(dev)
        out = g.new(X.shape, torch.complex64)
        _call("disco_apply_mask_channels", _p(X), _p(m), _p(out), G, chans, T * F, om)
        g.check(("apply_mask_channels", chans))
        w = (1 - m) if one_minus else m
        assert torch.equal(torch.view_as_real(out), torch.view_as_real(X) * w[:, None, :, :, None])


@pytest.mark.parametrize("dtype", [torch.complex64, torch.float32])
def test_transpose_shapes(dev, dtype):
    rng = np.random.default_rng(0)
    fn = "disco_transpose_c64" if dtype == torch.complex64 else "disco_transpose_f32"
    for batch in (1, 3):
        for rows in (1, 31, 32, 33, 257):
            for cols in (1, 31, 32, 33, 257):
                a = (cplx(rng, batch, rows, cols) if dtype == torch.complex64
                     else rng.standard_normal((batch, rows, cols)).astype(np.float32))
                ad = torch.from_numpy(a).to(dev)
                g = Guarded(dev)
                out = g.new((batch, cols, rows), dtype)
                _call(fn, _p(ad), _p(out), batch, rows, cols)
                g.check((fn, batch, rows, cols))
                assert torch.equal(out, ad.transpose(-1, -2).contiguous())


# ==== E. grid limits ===============================================================================================

def test_istft_beyond_grid_y_single_frame(dev):
    """131 073 signals (65 537 pairs, more than grid.y holds) of one frame, L = 1: equal to two calls split at an even
    signal index."""
    from disco_b200 import ops
    n = 2 * GRID_YZ + 3
    rng = np.random.default_rng(1)
    Y = torch.from_numpy(cplx(rng, n, 1, 129)).to(dev)
    x = ops.istft(Y, 1, 256)
    cut = 2 * 40000
    want = torch.cat([ops.istft(Y[:cut].contiguous(), 1, 256), ops.istft(Y[cut:].contiguous(), 1, 256)])
    torch.cuda.synchronize()
    assert torch.equal(x, want)
    assert bool(torch.isfinite(x).all())


def test_istft_beyond_grid_y_last_pairs(dev):
    """131 073 signals of 3 frames, L = 700: the pairs in the last launch against the float64 reference."""
    from disco_b200 import ops
    n, T, L = 2 * GRID_YZ + 3, 3, 700
    g = torch.Generator(device=dev).manual_seed(2)
    Y = torch.complex(torch.randn((n, T, 129), device=dev, generator=g), torch.randn((n, T, 129), device=dev, generator=g))
    x = ops.istft(Y, L, 256)
    tail = slice(n - 7, n)
    Yh = Y[tail].cpu().numpy()
    xs = x[tail].cpu().numpy()
    assert (n - 7) % 2 == 0        # the slice starts a pair: 2 pairs of the first launch, 1 pair and 1 lone signal of the second
    ref = np.stack([librosa_np.istft(Yh[s].T, hop_length=128, win_length=256, length=L, dtype=np.float64)
                    for s in range(7)])
    _, bound = istft_bound(Yh, L, 256)
    check_istft(xs, ref, bound, "last pairs")
    first = slice(0, 4)
    ref0 = np.stack([librosa_np.istft(Y[s].cpu().numpy().T, hop_length=128, win_length=256, length=L,
                                      dtype=np.float64) for s in range(4)])
    _, bound0 = istft_bound(Y[first].cpu().numpy(), L, 256)
    check_istft(x[first].cpu().numpy(), ref0, bound0, "first pairs")


@pytest.mark.parametrize("C", [1, 3])
def test_transpose_beyond_grid_y_rows(dev, C):
    """[1, 2 100 000, C] float32: 65 625 row tiles, more than grid.y holds."""
    from disco_b200 import ops
    a = torch.randn((1, 2_100_000, C), device=dev)
    out = ops.transpose_last2(a)
    torch.cuda.synchronize()
    assert torch.equal(out, a.transpose(-1, -2).contiguous())
