"""The length-aware STFT and iSTFT (lengths.cu: stft_lengths_kernel<N>; istft.cu: istft_lengths_kernel<N>) at every
instantiation, length class and launch-plan edge against float64, through the C ABI with every output inside a
NaN-filled guard band and every input poisoned with NaN past each signal's own end.

Dispatch targets (tests/test_lengths_stoi_instances_cpu.py parses the sets and the plan constants mirrored here out
of the sources, so a retuned launcher fails on CPU instead of moving these cases off their edges):
  stft_lengths   disco_stft_lengths   stft_lengths_kernel<N>, N = 256 / 512 / 1024: grid (frame groups, signal pairs);
                                      kLenWarps warp jobs of StftJob<N>::NB frames per CTA (16 / 8 / 4 frames)
  istft_lengths  disco_istft_lengths  istft_lengths_kernel<N>: grid (chunks, signal pairs), the chunk plan of
                                      disco_istft for the longest row (fpc hop blocks per chunk)
Both run pairs beyond grid.y (65 535) in further launches with x, Y and lengths advanced to an even signal.

STFT bound (DESIGN §2; u = 2^-24, w the periodic Hann window, H = N / 2).  Frame t < T_b = 1 + L_b // H of signal b
is one complex float32 FFT of (w / 2)(x_b + i x_p) over the reflect-padded frame, x_p the two-for-one partner
(signal b ^ 1; none for a lone last signal).  Each of the log2 N radix-2 stages rounds a butterfly output at most 4
times relative to the moduli feeding it, and the partial sums of a stage are bounded by the sum of the inputs' moduli;
the inter-pass twiddle (3), the window product and its table value (2) and the un-mixing add (1) come on top, and the
un-mixing adds two such errors, which doubles w / 2 to w.  So entry-wise
    |Y_b[t, f] - Y_b^f64[t, f]| <= tol_fft E_b[t],   tol_fft = sqrt(2) (4 log2 N + 6) u,
    E_b[t] = sum_n w_n |xpad_b[t H + n]| + [t < T_p] sum_n w_n |xpad_p[t H + n]|,
xpad the signal trimmed to its own length and reflect-padded at both ends (a partner that has ended contributes
exact zeros).  The yardstick is oracle.librosa_np.stft in float64 of the trimmed signal.  DC and Nyquist bins are real
by construction (imaginary part exactly 0), and frames T_b .. T - 1 are exactly 0.

iSTFT bound: istft_bound of tests/test_gpu_post_instances.py (derived there) on Y_b[:T'_b] with length L_b,
T'_b = min(T_b, y_frames): the same float32 inverse FFT, overlap-add and window-sum normalisation.  A pair of equal
lengths runs as one complex transform, so its partner's magnitudes enter m_t; a signal of a pair of different lengths,
or a lone last signal, runs alone.  Samples L_b .. L - 1 are exactly 0.

Bit-identity that the design promises (DESIGN "Uneven batches"): a frame of an equal-length pair or of a lone last
signal equals disco_stft of the trimmed signals; every iSTFT signal equals disco_istft of Y_b[:T'_b] at length L_b
(as a pair when the pair's lengths are equal, alone otherwise); and no result depends on the pair's position in the
batch.
"""
import numpy as np
import pytest
import torch

from oracle import librosa_np
from test_gpu_post_instances import (ISTFT_CTAS_PER_SM, ISTFT_ITEMS, ISTFT_MIN_TILES, Guarded, _call, _p,
                                     check_istft, cplx, istft_bound, istft_plan)
from test_gpu_stft_instances import hann, tol_fft

pytestmark = pytest.mark.gpu

# ---- launch-plan constants mirrored from the sources (checked against them on CPU) --------------------------------
LEN_NFFTS = (256, 512, 1024)      # launch_stft_lengths' and istft_lengths_kernel_for's switches
LEN_WARPS = 4                     # kLenWarps: warp jobs per stft_lengths CTA
JOB_NB = {256: 4, 512: 2, 1024: 1}   # StftJob<N>::NB = 32 / (N / 32): frames per warp job
GRID_YZ = 65535                   # kMaxGridYZ: signal pairs per launch


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def sms(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


def frames_per_cta(n_fft):
    return LEN_WARPS * JOB_NB[n_fft]


def n_frames(L, n_fft):
    return 1 + L // (n_fft // 2)


def first_end_reflected_frame(L, n_fft):
    """First frame t whose window [t H - H, t H + H) reaches past sample L - 1."""
    H = n_fft // 2
    return -(-(L - H + 1) // H)


def _len_with_frames(T, n_fft, r):
    """A length with T frames ending r samples into its last hop (r < H)."""
    return (T - 1) * (n_fft // 2) + r


# ---- cases ----------------------------------------------------------------------------------------------------------

def stft_cases(n_fft):
    """[(L_max, lengths, labels)] for stft_lengths: T_max on each side of a CTA's frame group, and in every batch the
    length classes, the pairings and T_b on each side of a frame group.  labels[s] names signal s's class; every label
    is asserted to land on its edge."""
    H, N = n_fft // 2, n_fft
    pc = frames_per_cta(n_fft)
    k = 5
    out = []
    for T_max, r in ((4 * pc - 1, 0), (4 * pc, H // 2 + 1), (4 * pc + 1, H - 1)):
        L_max = _len_with_frames(T_max, n_fft, r)
        pairs = [
            (("H+1", H + 1), ("H+1", H + 1)),                                # an equal-length pair
            (("H+2", H + 2), ("N-1", N - 1)),                                # partner longer / partner shorter
            (("N", N), ("N+1", N + 1)),
            (("kH-1", k * H - 1), ("kH+1", k * H + 1)),
            (("kH", k * H), ("kH", k * H)),                                  # last frame centred on the end
            (("L_max", L_max), ("L_max", L_max)),
            (("partner_ends_before_reflect", L_max - 3), ("H+1", H + 1)),
            (("Tb=2pc-1", _len_with_frames(2 * pc - 1, n_fft, H // 3)), ("Tb=2pc", _len_with_frames(2 * pc, n_fft, 1))),
            (("Tb=2pc+1", _len_with_frames(2 * pc + 1, n_fft, H - 2)),
             ("Tb=2pc+1", _len_with_frames(2 * pc + 1, n_fft, H - 2))),
        ]
        labels = [lab for pr in pairs for lab, _ in pr] + ["lone_last"]
        lengths = [L for pr in pairs for _, L in pr] + [k * H + 7]
        check_stft_labels(n_fft, L_max, lengths, labels)
        out.append((L_max, lengths, labels))
    assert {L_max % H == 0 for L_max, _, _ in out} == {True, False}
    assert sorted(n_frames(L_max, n_fft) % pc for L_max, _, _ in out) == [0, 1, pc - 1]
    return out


def check_stft_labels(n_fft, L_max, lengths, labels):
    H, N = n_fft // 2, n_fft
    pc = frames_per_cta(n_fft)
    n = len(lengths)
    assert n % 2 == 1 and labels[-1] == "lone_last"
    assert all(H < L <= L_max for L in lengths)
    want = {"H+1": H + 1, "H+2": H + 2, "N-1": N - 1, "N": N, "N+1": N + 1, "L_max": L_max}
    for s, (lab, L) in enumerate(zip(labels, lengths)):
        T = n_frames(L, n_fft)
        if lab in want:
            assert L == want[lab], (lab, L)
        elif lab == "kH":
            assert L % H == 0 and (T - 1) * H == L and T > 2            # the last frame is centred on sample L
        elif lab == "kH-1":
            assert L % H == H - 1
        elif lab == "kH+1":
            assert L % H == 1
        elif lab.startswith("Tb="):
            off = {"2pc-1": -1, "2pc": 0, "2pc+1": 1}[lab[3:]]
            assert T == 2 * pc + off and T <= n_frames(L_max, n_fft)
        elif lab == "partner_ends_before_reflect":
            Tp = n_frames(lengths[s ^ 1], n_fft)
            assert Tp <= first_end_reflected_frame(L, n_fft) and lengths[s ^ 1] != L
        else:
            assert lab == "lone_last" and s == n - 1
    pairs = [(lengths[2 * p], lengths[2 * p + 1]) for p in range(n // 2)]
    assert any(a == b for a, b in pairs) and any(a < b for a, b in pairs) and any(a > b for a, b in pairs)


def istft_classes(n_fft, L_max):
    """(label, length) of every length class of istft_lengths (its ABI accepts lengths in (0, L])."""
    H, N, k = n_fft // 2, n_fft, 5
    return [("1", 1), ("H-1", H - 1), ("H+1", H + 1), ("H+2", H + 2), ("N-1", N - 1), ("N", N), ("N+1", N + 1),
            ("kH-1", k * H - 1), ("kH", k * H), ("kH+1", k * H + 1), ("L_max", L_max)]


def istft_plan_cases(n_fft, sms):
    """[(label, n_sig, T, L_max, lengths)] at the edges of launch_istft_lengths' chunk plan; each label is asserted
    against the mirrored plan."""
    H = n_fft // 2
    target = sms * ISTFT_CTAS_PER_SM
    cases = []
    # one chunk: 2 SMs of pairs over 65 hop blocks (a smaller batch would split them); every length class, equal and
    # different pairs, repeated over the batch
    T = ISTFT_MIN_TILES * ISTFT_ITEMS + 1
    L_max = _len_with_frames(T, n_fft, H // 2)
    cls = [L for _, L in istft_classes(n_fft, L_max)]
    n_sig = 2 * target + 1
    lengths = [cls[(i // 2) % len(cls)] if (i // 2) % 3 else cls[i % len(cls)] for i in range(n_sig)]
    j_end, _, chunks, fpc = istft_plan(n_sig, T, L_max, n_fft, sms)
    assert chunks == 1 and j_end > ISTFT_MIN_TILES * ISTFT_ITEMS and (n_sig + 1) // 2 >= target
    cases.append(("one_chunk", n_sig, T, L_max, lengths))
    # many chunks: a few pairs over 513 hop blocks; T_b on and one past chunk boundaries, inside chunk 0, and a pair
    # of different lengths (the two-body path) in the many-chunk plan
    T = 8 * ISTFT_ITEMS * 4 + 1
    L_max = _len_with_frames(T, n_fft, H - 1)
    _, _, chunks, fpc = istft_plan(11, T, L_max, n_fft, sms)
    assert chunks >= 4, chunks
    at = lambda Tb, r: _len_with_frames(Tb, n_fft, r)
    lengths = [at(fpc, 3), at(fpc, 3),                       # an equal pair ending on a chunk boundary
               at(fpc + 1, H - 1), at(2 * fpc, 0),           # a pair of different lengths: one past / on a boundary
               at(2 * fpc + 1, 1), at(2 * fpc + 1, 1),       # an equal pair one past a boundary
               at(fpc // 2, H // 2), L_max,                  # inside chunk 0 / the longest
               1, H - 1,
               at(3 * fpc, H // 3)]                          # lone last, on a boundary
    tb = [min(T, n_frames(L, n_fft)) for L in lengths]
    assert tb[0] == fpc and tb[2] == fpc + 1 and tb[3] == 2 * fpc and tb[4] == 2 * fpc + 1 and tb[10] == 3 * fpc
    assert tb[6] < fpc and n_frames(L_max, n_fft) > 3 * fpc and lengths[2] != lengths[3]
    assert istft_plan(len(lengths), T, L_max, n_fft, sms)[2] == chunks
    cases.append(("many_chunks", len(lengths), T, L_max, lengths))
    # y_frames < 1 + L / H: the longer signals are cut to the frames given and zero-filled
    T_full = 40
    L_max = _len_with_frames(T_full, n_fft, H // 2 + 3)
    T = T_full - 3
    lengths = [L_max, L_max, L_max - 2 * H, _len_with_frames(T, n_fft, 5), _len_with_frames(T - 1, n_fft, 5), 1, n_fft]
    assert T < n_frames(L_max, n_fft) and n_frames(lengths[2], n_fft) > T and n_frames(lengths[4], n_fft) < T
    cases.append(("y_frames_short", len(lengths), T, L_max, lengths))
    return cases


# ---- device calls ---------------------------------------------------------------------------------------------------

def _lengths_ptrs(lengths, dev):
    from disco_b200 import _lib
    host = np.ascontiguousarray(lengths, dtype=np.int32)
    return torch.from_numpy(host).to(dev), host, host.ctypes.data_as(_lib.c_int_p)


def stft_lengths_dev(dev, xd, lengths, n_fft, what):
    n_sig, L = xd.shape
    g = Guarded(dev)
    Y = g.new((n_sig, n_frames(L, n_fft), n_fft // 2 + 1), torch.complex64)
    ld, _, hp = _lengths_ptrs(lengths, dev)
    _call("disco_stft_lengths", _p(xd), _p(ld), hp, _p(Y), n_sig, L, n_fft)
    g.check(what)
    return Y


def istft_lengths_dev(dev, Yd, lengths, L, n_fft, what):
    n_sig, T, _ = Yd.shape
    g = Guarded(dev)
    x = g.new((n_sig, L), torch.float32)
    ld, _, hp = _lengths_ptrs(lengths, dev)
    _call("disco_istft_lengths", _p(Yd), _p(ld), hp, _p(x), n_sig, T, L, n_fft)
    g.check(what)
    return x


def stft_dev(dev, xh, n_fft):
    """disco_stft of the rows xh (host float32), guarded."""
    xd = torch.from_numpy(np.ascontiguousarray(xh)).to(dev)
    n_sig, L = xh.shape
    g = Guarded(dev)
    Y = g.new((n_sig, n_frames(L, n_fft), n_fft // 2 + 1), torch.complex64)
    _call("disco_stft", _p(xd), _p(Y), n_sig, L, n_fft)
    g.check("disco_stft")
    return Y.cpu().numpy()


def istft_dev(dev, Yd, L, n_fft):
    n_sig, T, _ = Yd.shape
    g = Guarded(dev)
    x = g.new((n_sig, L), torch.float32)
    _call("disco_istft", _p(Yd.contiguous()), _p(x), n_sig, T, L, n_fft)
    g.check("disco_istft")
    return x.cpu().numpy()


def poisoned_signals(rng, lengths, L):
    """[n_sig, L] float32: N(0, 1) samples up to each length, NaN after."""
    x = np.full((len(lengths), L), np.nan, np.float32)
    for s, Lb in enumerate(lengths):
        x[s, :Lb] = rng.standard_normal(Lb).astype(np.float32)
    return x


def poisoned_spectra(rng, lengths, T, n_fft):
    """[n_sig, T, F] complex64: random up to each signal's frame count, NaN after."""
    Y = cplx(rng, len(lengths), T, n_fft // 2 + 1)
    for s, Lb in enumerate(lengths):
        Y[s, n_frames(Lb, n_fft):] = np.nan
    return Y


# ---- float64 checkers -----------------------------------------------------------------------------------------------

def frames_f64(x, n_fft):
    """Y [T, F] complex128 of the trimmed signal x (librosa_np in float64) and A[t] = sum_n w_n |xpad[t H + n]|."""
    H = n_fft // 2
    x = np.asarray(x, np.float64)
    Y = librosa_np.stft(x, n_fft, H, dtype=np.complex128).T
    pad = np.pad(np.abs(x), H, mode="reflect")
    T = n_frames(len(x), n_fft)
    idx = np.arange(n_fft)[None, :] + H * np.arange(T)[:, None]
    return Y, pad[idx] @ hann(n_fft)


def check_stft_signal(Yb, x, lengths, s, n_fft, what):
    """Signal s of a stft_lengths output (Yb [T, F] complex64) against float64 of x[s, :L_s] under the §2 bound; the
    partner's envelope counts while the partner lasts.  Frames past T_s exactly 0, DC / Nyquist real."""
    L_s = lengths[s]
    T_s = n_frames(L_s, n_fft)
    assert not np.any(Yb[T_s:]), (what, s, "frames from T_b on are not zero")
    assert not Yb[:T_s, 0].imag.any() and not Yb[:T_s, -1].imag.any(), (what, s, "DC / Nyquist bin not real")
    ref, A = frames_f64(x[s, :L_s], n_fft)
    E = A.copy()
    p = s ^ 1
    if p < len(lengths):
        _, Ap = frames_f64(x[p, :lengths[p]], n_fft)
        m = min(len(Ap), T_s)
        E[:m] += Ap[:m]
    err = np.abs(Yb[:T_s].astype(np.complex128) - ref)
    bad = ~(err <= tol_fft(n_fft) * E[:, None])
    assert not bad.any(), (what, s, L_s, "%d bins beyond the bound, first at %s" % (int(bad.sum()), np.argwhere(bad)[0]))


def istft_ref(Yh, lengths, s, n_fft):
    """(float64 iSTFT of signal s, entry-wise bound) as istft_lengths runs it: Y_s[:T'_s] at length L_s, with the
    partner's spectrum in the bound when the pair's lengths are equal."""
    n_sig, T, _ = Yh.shape
    L_s = lengths[s]
    Tb = min(T, n_frames(L_s, n_fft))
    p = s ^ 1
    rows = sorted((s, p)) if p < n_sig and lengths[p] == L_s else [s]
    val, bound = istft_bound(Yh[rows][:, :Tb], L_s, n_fft)
    i = rows.index(s)
    ref = librosa_np.istft(Yh[s, :Tb].T, hop_length=n_fft // 2, win_length=n_fft, length=L_s, dtype=np.float64)
    # the bound's own overlap-add restates the oracle (a self-check of the formula the bound is built on)
    assert np.allclose(val[i], ref, rtol=0, atol=1e-12 * max(1.0, np.abs(ref).max()))
    return ref, bound[i]


def check_istft_signal(xb, Yh, lengths, s, n_fft, what):
    L_s = lengths[s]
    assert not np.any(xb[L_s:]), (what, s, "samples from L_b on are not zero")
    ref, bound = istft_ref(Yh, lengths, s, n_fft)
    check_istft(xb[None, :L_s], ref[None], bound[None], (what, s, L_s))


# ==== A. stft_lengths ================================================================================================

@pytest.mark.parametrize("n_fft", LEN_NFFTS)
def test_stft_lengths_classes_pairs_and_grid(dev, n_fft):
    """Every length class and pairing at T_max on each side of a CTA's frame group, inputs NaN past each length:
    float64 within the §2 bound, exact zeros past T_b, bit-identical to disco_stft of the trimmed signals where the
    pairing is the same, and independent of the pair's position in the batch."""
    rng = np.random.default_rng(n_fft)
    for L_max, lengths, labels in stft_cases(n_fft):
        x = poisoned_signals(rng, lengths, L_max)
        xd = torch.from_numpy(x).to(dev)
        what = ("stft_lengths", n_fft, L_max)
        Y = stft_lengths_dev(dev, xd, lengths, n_fft, what)
        Yh = Y.cpu().numpy()
        assert np.isfinite(Yh.view(np.float32)).all(), what
        n = len(lengths)
        for s in range(n):
            check_stft_signal(Yh[s], x, lengths, s, n_fft, what + (labels[s],))
        for p in range(n // 2):
            a, b = 2 * p, 2 * p + 1
            if lengths[a] == lengths[b]:
                L_s = lengths[a]
                ref = stft_dev(dev, x[a:b + 1, :L_s], n_fft)
                assert np.array_equal(Yh[a:b + 1, :n_frames(L_s, n_fft)], ref), what + (labels[a], "not disco_stft's")
        L_s = lengths[-1]
        assert np.array_equal(Yh[-1, :n_frames(L_s, n_fft)], stft_dev(dev, x[-1:, :L_s], n_fft)[0]), what + ("lone",)
        # the pairs in reverse order (the lone signal stays last): the same bits
        perm = [i for p in reversed(range(n // 2)) for i in (2 * p, 2 * p + 1)] + [n - 1]
        Yp = stft_lengths_dev(dev, xd[perm].contiguous(), [lengths[i] for i in perm], n_fft, what + ("permuted",))
        assert torch.equal(Yp, Y[perm]), what + ("depends on the batch position",)


# ==== B. istft_lengths ===============================================================================================

@pytest.mark.parametrize("n_fft", LEN_NFFTS)
def test_istft_lengths_plan_edges(dev, sms, n_fft):
    """One-chunk and many-chunk plans, T_b on and one past a chunk boundary of the longest signal's plan and inside
    chunk 0, a different-length pair in a many-chunk plan, y_frames below 1 + L / H; spectra NaN past each signal's
    frames.  Float64 within istft_bound, exact zeros past L_b, bit-identical to disco_istft of the trimmed spectra."""
    rng = np.random.default_rng(100 + n_fft)
    for label, n_sig, T, L_max, lengths in istft_plan_cases(n_fft, sms):
        Yh = poisoned_spectra(rng, lengths, T, n_fft)
        Yd = torch.from_numpy(Yh).to(dev)
        plan = istft_plan(n_sig, T, L_max, n_fft, sms)
        what = (label, n_fft, n_sig, T, L_max, plan)
        xh = istft_lengths_dev(dev, Yd, lengths, L_max, n_fft, what).cpu().numpy()
        assert np.isfinite(xh).all(), what
        check = range(n_sig) if n_sig <= 64 else list(range(40)) + list(range(n_sig - 40, n_sig))
        for s in check:
            check_istft_signal(xh[s], Yh, lengths, s, n_fft, what)
        for s in check:
            L_s = lengths[s]
            Tb = min(T, n_frames(L_s, n_fft))
            p = s ^ 1
            if p < n_sig and lengths[p] == L_s:
                lo = min(s, p)
                ref = istft_dev(dev, Yd[lo:lo + 2, :Tb], L_s, n_fft)[s - lo]
            else:
                ref = istft_dev(dev, Yd[s:s + 1, :Tb], L_s, n_fft)[0]
            assert np.array_equal(xh[s, :L_s], ref), what + (s, "not disco_istft's")


@pytest.mark.parametrize("n_fft", LEN_NFFTS)
def test_istft_lengths_classes_and_position(dev, sms, n_fft):
    """Every length class of (0, L] in equal pairs, in different pairs and alone, at the head and at the tail of a
    one-chunk batch: the same bits at both positions."""
    rng = np.random.default_rng(200 + n_fft)
    H = n_fft // 2
    T = 12
    L_max = _len_with_frames(T, n_fft, H - 3)
    cls = [L for _, L in istft_classes(n_fft, L_max)]
    head = [L for L in cls for _ in range(2)] + cls                    # equal pairs, then different pairs (odd count)
    n_fill = 2 * sms * ISTFT_CTAS_PER_SM
    lengths = head[:-1] + [L_max] * n_fill + head
    assert len(head) % 2 == 1 and len(lengths) % 2 == 1
    Yh = poisoned_spectra(rng, lengths, T, n_fft)
    start = len(head) - 1 + n_fill
    Yh[start:start + len(head) - 1] = Yh[:len(head) - 1]
    Yd = torch.from_numpy(Yh).to(dev)
    assert istft_plan(len(lengths), T, L_max, n_fft, sms)[2] == 1
    xh = istft_lengths_dev(dev, Yd, lengths, L_max, n_fft, ("classes", n_fft)).cpu().numpy()
    for s in list(range(len(head))) + list(range(start, len(lengths))):
        check_istft_signal(xh[s], Yh, lengths, s, n_fft, ("classes", n_fft))
    assert np.array_equal(xh[start:start + len(head) - 1], xh[:len(head) - 1])


# ==== C. beyond grid.y ===============================================================================================

def beyond_grid_lengths(n, H, L_max):
    """Lengths of n = 2 * 65535 + 3 signals: pairs of equal and of different lengths cycling through (H, L_max], and
    the 3 signals of the second launch with lengths that differ from those at their positions in the first."""
    span = L_max - H
    p = np.arange(n) // 2
    lengths = (H + 1 + (p * 37) % span).astype(np.int32)
    odd = (np.arange(n) % 2 == 1) & (p % 3 == 0)                # every third pair of different lengths
    lengths[odd] = H + 1 + (p[odd] * 37 + 11) % span
    s0 = 2 * GRID_YZ
    lengths[s0:] = [L_max - 5, L_max - 5, H + 2]
    assert n - s0 == 3 and all(lengths[s0 + i] != lengths[i] for i in range(3))
    assert lengths.min() > H and lengths.max() <= L_max
    return lengths


# signals checked against float64 beyond grid.y: the first 4 pairs, pairs in the middle and at the end of the first
# launch, and the pair and the lone signal of the second launch (whole pairs, each starting at an even signal)
SAMPLE_BEYOND_GRID = list(range(8)) + [2 * 30011, 2 * 30011 + 1, 2 * GRID_YZ - 2, 2 * GRID_YZ - 1] + \
    [2 * GRID_YZ, 2 * GRID_YZ + 1, 2 * GRID_YZ + 2]


def test_stft_lengths_beyond_grid_y(dev):
    """131 073 signals (65 537 pairs): the second launch's signals against float64 and the first pairs bit for bit
    against a separate small call."""
    n_fft, H, L_max = 256, 128, 600
    n = 2 * GRID_YZ + 3
    lengths = beyond_grid_lengths(n, H, L_max)
    g = torch.Generator(device=dev).manual_seed(3)
    xd = torch.randn((n, L_max), device=dev, generator=g)
    ld = torch.from_numpy(lengths).to(dev)
    xd[torch.arange(L_max, device=dev)[None, :] >= ld[:, None].long()] = float("nan")
    Y = stft_lengths_dev(dev, xd, lengths, n_fft, "beyond grid.y")
    T = Y.shape[1]
    past = torch.arange(T, device=dev)[None, :] >= (1 + ld // H)[:, None].long()
    assert not bool(Y[past].abs().gt(0).any()), "frames past T_b not zero"
    assert bool(torch.isfinite(torch.view_as_real(Y)).all())
    # whole pairs from even signals, so that a signal's partner is its neighbour in the sample too
    sample = SAMPLE_BEYOND_GRID
    x, Yh, ls = xd[sample].cpu().numpy(), Y[sample].cpu().numpy(), lengths[sample]
    for i, s in enumerate(sample):
        check_stft_signal(Yh[i], x, ls, i, n_fft, ("beyond grid.y", s))
    small = stft_lengths_dev(dev, xd[:8].contiguous(), lengths[:8], n_fft, "small")
    assert torch.equal(small, Y[:8])


def test_istft_lengths_beyond_grid_y(dev):
    """131 073 signals: the second launch against float64 and the first pairs bit for bit against a small call."""
    n_fft, H, L_max, T = 256, 128, 600, 5
    n = 2 * GRID_YZ + 3
    lengths = beyond_grid_lengths(n, H, L_max)
    lengths[7] = 1                                      # a signal shorter than a hop among the first pairs
    lengths[6] = 1
    g = torch.Generator(device=dev).manual_seed(4)
    Y = torch.complex(torch.randn((n, T, H + 1), device=dev, generator=g),
                      torch.randn((n, T, H + 1), device=dev, generator=g))
    ld = torch.from_numpy(lengths).to(dev)
    Y[torch.arange(T, device=dev)[None, :] >= (1 + ld // H)[:, None].long()] = complex(float("nan"), float("nan"))
    x = istft_lengths_dev(dev, Y, lengths, L_max, n_fft, "beyond grid.y")
    past = torch.arange(L_max, device=dev)[None, :] >= ld[:, None].long()
    assert not bool(x[past].ne(0).any()), "samples past L_b not zero"
    assert bool(torch.isfinite(x).all())
    sample = SAMPLE_BEYOND_GRID
    xh, Yh, ls = x[sample].cpu().numpy(), Y[sample].cpu().numpy(), lengths[sample]
    for i, s in enumerate(sample):
        check_istft_signal(xh[i], Yh, ls, i, n_fft, ("beyond grid.y", s))
    small = istft_lengths_dev(dev, Y[:8].contiguous(), lengths[:8], L_max, n_fft, "small")
    assert torch.equal(small, x[:8])


# ==== D. negative controls ===========================================================================================

@pytest.mark.parametrize("n_fft", LEN_NFFTS)
def test_stft_lengths_negative_controls(dev, n_fft):
    """The checker rejects: the last frame reflected at L_max instead of L_b, T_b off by one either way, the partner's
    samples in place of the signal's."""
    H = n_fft // 2
    rng = np.random.default_rng(300 + n_fft)
    L_max = _len_with_frames(30, n_fft, H // 2)
    lengths = [11 * H + H // 3, 7 * H - 5, 9 * H, 9 * H, 4 * H + 1]
    x = poisoned_signals(rng, lengths, L_max)
    Yh = stft_lengths_dev(dev, torch.from_numpy(x).to(dev), lengths, n_fft, "controls").cpu().numpy()
    for s in range(len(lengths)):
        check_stft_signal(Yh[s], x, lengths, s, n_fft, "controls")
    s, L_s = 0, lengths[0]
    T_s = n_frames(L_s, n_fft)
    # reflected at L_max: the zero-filled row's STFT, cut to T_b frames
    row = np.where(np.isnan(x[s]), 0.0, x[s]).astype(np.float64)
    bad = Yh[s].copy()
    bad[:T_s] = librosa_np.stft(row, n_fft, H, dtype=np.complex128).T[:T_s].astype(np.complex64)
    with pytest.raises(AssertionError):
        check_stft_signal(bad, x, lengths, s, n_fft, "reflected at L_max")
    bad = Yh[s].copy()
    bad[T_s - 1] = 0
    with pytest.raises(AssertionError):
        check_stft_signal(bad, x, lengths, s, n_fft, "T_b - 1 frames")
    bad = Yh[s].copy()
    bad[T_s] = librosa_np.stft(row, n_fft, H, dtype=np.complex128).T[T_s].astype(np.complex64)
    assert np.any(bad[T_s])
    with pytest.raises(AssertionError):
        check_stft_signal(bad, x, lengths, s, n_fft, "T_b + 1 frames")
    with pytest.raises(AssertionError):
        check_stft_signal(Yh[1], x, lengths, s, n_fft, "partner's samples")


@pytest.mark.parametrize("n_fft", LEN_NFFTS)
def test_istft_lengths_negative_controls(dev, n_fft):
    """The checker rejects: an iSTFT normalised with the padded length's window sum, T_b off by one either way, the
    partner's samples in place of the signal's."""
    H = n_fft // 2
    rng = np.random.default_rng(400 + n_fft)
    T = 30
    L_max = _len_with_frames(T, n_fft, H // 2)
    lengths = [11 * H + H - 1, 7 * H - 5, 9 * H + 3, 9 * H + 3, 4 * H + 1]
    Yh = cplx(rng, len(lengths), T, H + 1)        # finite everywhere: the controls read frames past T_b
    xh = istft_lengths_dev(dev, torch.from_numpy(Yh).to(dev), lengths, L_max, n_fft, "controls").cpu().numpy()
    for s in range(len(lengths)):
        check_istft_signal(xh[s], Yh, lengths, s, n_fft, "controls")
    s, L_s = 0, lengths[0]
    T_s = n_frames(L_s, n_fft)
    kw = dict(hop_length=H, win_length=n_fft, dtype=np.float32)
    padded = Yh[s].copy()
    padded[T_s:] = 0
    bad = xh[s].copy()
    bad[:L_s] = librosa_np.istft(padded.T, length=L_max, **kw)[:L_s]     # window sum of the L_max-sample signal
    with pytest.raises(AssertionError):
        check_istft_signal(bad, Yh, lengths, s, n_fft, "padded window sum")
    for Tb in (T_s - 1, T_s + 1):
        bad = xh[s].copy()
        bad[:L_s] = librosa_np.istft(Yh[s, :Tb].T, length=L_s, **kw)
        with pytest.raises(AssertionError):
            check_istft_signal(bad, Yh, lengths, s, n_fft, ("T_b", Tb))
    with pytest.raises(AssertionError):
        check_istft_signal(xh[1], Yh, lengths, s, n_fft, "partner's samples")
