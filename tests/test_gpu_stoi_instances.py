"""The four STOI kernels (stoi.cu: resample_poly_kernel, stoi_select_kernel, stoi_bands_kernel, stoi_score_kernel)
and their per-signal-length modes at their launch-plan edges against float64, through the C ABI: d, n_sel and
n_frames inside NaN-filled guard bands, and the workspace itself filled with a NaN pattern so that its intermediates
(frame energies, kept-frame lists, band envelopes) are read back, compared with oracle/stoi_np.py and checked to be
written exactly where launch_stoi's layout puts them and nowhere else.

Plan constants (mirrored below; tests/test_lengths_stoi_instances_cpu.py parses them out of the sources):
  stoi_select_kernel  one CTA of kSelThreads = 256 per clean: a warp per frame (8 warps), then an in-order
                      ballot / popc scan over 256 frames per pass, `base` carried across passes
  stoi_bands_kernel   grid (n_clean + n_pair) * groups, groups = ceil((n_fr - 1) / kBandWarps): kBandWarps = 4 STFT
                      frames per CTA, a warp returns at t >= n_sel - 1
  stoi_score_kernel   one CTA of kScoreThreads = 256 per pair: 15 J (segment, band) items, J = n_sel - 1 - 29, taken
                      by thread it % 256 in order; below kStoiSeg = 30 STFT frames the score is 1e-5
  workspace           energy [n_clean][n_fr] float64, tob [n_clean + n_pair][n_fr][15] float64, sel [n_clean][n_fr]
                      int32, n_fr = (L - 256) // 128 + 1

Bounds (u = 2^-53; both the kernel and NumPy err from exact arithmetic, so each bound adds the two sides' errors).
  Window.  The kernel's 0.5 + 0.5 cospi((2n - 255) / 257) and np.hanning(258)[1:-1] are the same numbers.  cospi of a
    rounded argument of modulus < 1 errs by at most pi u + 2 ulp(1) = (pi + 4) u; NumPy's cos(pi k / 257) takes an
    argument with 3 roundings (pi, the product, the quotient: 3 pi u) and errs by at most 3 pi u + 2 u; halving is
    exact and 0.5 + v rounds once (u).  So each side's window value is within delta_w = 8 u of the exact one,
    absolutely (not relatively: near the window's ends the value is tiny).
  Energies.  s = sum_r (w_r x_r)^2 over 256 samples.  The kernel rounds each product once (2u on its square), then
    accumulates with fma, 8 terms per lane and a 5-level butterfly: 13 roundings of non-negative partial sums.  NumPy
    rounds each product and square (3u) and sums at most 256 terms (256u).  The window error moves a square by at most
    2 delta_w w_r x_r^2.  So
        |Δs| <= (15 + 259) u s + 4 delta_w sum_r w_r x_r^2.
    Then sqrt (u each side), + eps (u each side), log10 (1 ulp each side) and the factor 20 (u):
        |Δe| <= (20 / ln 10) (|Δs| / (2 sqrt(s)) + 4 u (sqrt(s) + eps)) / (sqrt(s) + eps) + 6 u |e|.
  Kept-frame list.  Equal element for element (and n_sel equal) on inputs whose energies stay at least 1e-9 dB from
    the 40 dB threshold (energy_margin), which is far beyond the bound above.
  Band envelopes.  Sample n of STFT frame t is z_n = w_n (w_r x[sel_j 128 + r] + w_(128+r) x[sel_(j-1) 128 + 128 + r]),
    j = t + n // 128, r = n % 128 (the overlap-add of the kept frames, the second term absent for j = 0).  Each side
    forms it with at most 4 roundings along any term and the window error above, so with a_n = w_n (w_r |x_a| +
    w_(128+r) |x_b|) and b_n = |x_a| + |x_b|:  |Δz_n| <= d_n = 4 u a_n + delta_w (1 + w_n) b_n.  A radix-2 stage
    (butterfly u +- w v: the complex product 2 sqrt(2) u |w||v|, the twiddle's sincospi value (2 ulp per component,
    4 sqrt(2) u), the complex add u) errs by at most 10 u relative to |u| + |v|, and the nodes one output depends on
    partition the inputs, so a 512-point FFT of 9 stages (NumPy's real FFT: at most one more stage's worth) errs per
    bin by at most eps_fft sum_n a_n with eps_fft = 100 u, plus sum_n d_n from the inputs.  Band b sums m_b = edges
    [b + 1] - edges[b] bins: B = ||X_band||_2 moves by at most sqrt(m_b) max_k |ΔX_k| (triangle inequality), and its
    squares, sum and sqrt round within (m_b + 6) u B over both sides:
        |ΔB| <= 2 sqrt(m_b) (eps_fft sum_n a_n + sum_n d_n) + (m_b + 6) u B.
  Scores.  Within 1e-9 of the oracle's (a mean of 15 J items summed in different orders), as in test_gpu_stoi.py.
  Resampler.  test_gpu_stoi.resample_ok's bound against scipy.signal.resample_poly of the trimmed row, and exact zeros
    from ceil(L_b up / down) on.
"""
import math
import warnings

import numpy as np
import pytest
import torch

from oracle import stoi_np
from test_gpu_post_instances import GUARD, SENT32, Guarded, _call, _p
from test_gpu_stoi import energy_margin, resample_ok, speechlike

pytestmark = pytest.mark.gpu

U64 = 2.0 ** -53
DELTA_W = 8 * U64
EPS_FFT = 100 * U64
SENT_WS64 = (SENT32 << 32) | SENT32     # two int32 sentinels read as one float64 (a NaN)

# ---- plan constants mirrored from the sources (checked against them on CPU) ----------------------------------------
STOI_FRAME = 256          # kStoiFrame
STOI_HOP = STOI_FRAME // 2
STOI_BANDS = 15           # kStoiBands
STOI_SEG = 30             # kStoiSeg
SEL_THREADS = 256         # kSelThreads: frames per scan pass
SEL_WARPS = SEL_THREADS // 32
BAND_WARPS = 4            # kBandWarps: STFT frames per stoi_bands CTA
SCORE_THREADS = 256       # kScoreThreads: (segment, band) items per pass of a score CTA


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def n_fr_of(L):
    return 0 if L < STOI_FRAME else (L - STOI_FRAME) // STOI_HOP + 1


def ws_layout(n_clean, n_pair, L):
    """launch_stoi's workspace: (n_fr, energy offset, tob offset, sel offset) in bytes, and the total size."""
    n_fr = n_fr_of(L)
    e_off = 0
    tob_off = e_off + 8 * n_clean * n_fr
    sel_off = tob_off + 8 * (n_clean + n_pair) * n_fr * STOI_BANDS
    return n_fr, e_off, tob_off, sel_off, sel_off + 4 * n_clean * n_fr


def loud(seed, n_sel, extra=0):
    """A clean whose every frame is kept (n_sel = its frame count), extra < 128 samples past its last full frame."""
    return speechlike(seed, STOI_FRAME + STOI_HOP * (n_sel - 1) + extra, period=1 << 30).astype(np.float64)


# ---- the call --------------------------------------------------------------------------------------------------------

def stoi_run(dev, cleans, degraded, pairs, lengths=None, what=""):
    """disco_stoi (lengths None) or disco_stoi_lengths with guarded d / n_sel / n_frames and a sentinel-filled,
    guard-banded workspace.  Returns a dict of host arrays: d, n_sel, n_frames, and the workspace split by launch_stoi's
    layout into energy [C, n_fr], tob [C + P, n_fr, 15], sel [C, n_fr] and their 'written' masks."""
    from disco_b200 import _lib
    lib = _lib.load()
    C, L = cleans.shape
    D, P = degraded.shape[0], len(pairs)
    T = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    xc, xd, pr = T(cleans, np.float64), T(degraded, np.float64), T(np.asarray(pairs).reshape(-1, 2), np.int32)
    g = Guarded(dev)
    d = g.new((P,), torch.float64)
    n_sel = g.new((C,), torch.int32)
    n_frames = g.new((P,), torch.int32)
    ws_bytes = lib.disco_stoi_workspace(C, P, L)
    n_fr, e_off, tob_off, sel_off, total = ws_layout(C, P, L)
    assert ws_bytes == total, (ws_bytes, total)
    wbuf = torch.full((ws_bytes // 4 + 2 * GUARD,), SENT32, dtype=torch.int32, device=dev)
    ws = wbuf[GUARD:GUARD + ws_bytes // 4]
    if lengths is None:
        _call("disco_stoi", _p(xc), _p(xd), _p(pr), _p(d), _p(n_sel), _p(n_frames), C, D, P, L, _p(ws), ws_bytes)
    else:
        lh = np.ascontiguousarray(lengths, dtype=np.int32)
        ld = T(lh, np.int32)
        _call("disco_stoi_lengths", _p(xc), _p(xd), _p(pr), _p(d), _p(n_sel), _p(n_frames), C, D, P, L,
              _p(ld), lh.ctypes.data_as(_lib.c_int_p), _p(ws), ws_bytes)
    g.check(what)
    assert bool((wbuf[:GUARD] == SENT32).all()) and bool((wbuf[GUARD + ws_bytes // 4:] == SENT32).all()), \
        (what, "workspace guard word changed")
    w = ws.cpu().numpy()
    f64 = lambda a, b, shape: w[a // 4:b // 4].view(np.float64).reshape(shape)
    out = dict(d=d.cpu().numpy(), n_sel=n_sel.cpu().numpy(), n_frames=n_frames.cpu().numpy(), ws=ws.clone(), n_fr=n_fr,
               energy=f64(e_off, tob_off, (C, n_fr)), tob=f64(tob_off, sel_off, (C + P, n_fr, STOI_BANDS)),
               sel=w[sel_off // 4:].reshape(C, n_fr))
    out["energy_w"] = out["energy"].view(np.int64) != SENT_WS64
    out["tob_w"] = out["tob"].view(np.int64) != SENT_WS64
    out["sel_w"] = out["sel"] != SENT32
    return out


# ---- float64 checkers ------------------------------------------------------------------------------------------------

def check_energy(got, x, what):
    """got [n_fr(x)] against stoi_np.frame_energies(x) under the derived bound."""
    want = stoi_np.frame_energies(x)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    w = stoi_np.hann()
    fr = np.stack([x[i:i + STOI_FRAME] for i in range(0, len(x) - STOI_FRAME + 1, STOI_HOP)])
    s = ((w * fr) ** 2).sum(1)
    ds = (15 + 259) * U64 * s + 4 * DELTA_W * (w * fr ** 2).sum(1)
    r = np.sqrt(s)
    lin = np.where(s > 0, ds / (2 * np.where(s > 0, r, 1.0)), 0.0) + 4 * U64 * (r + stoi_np.EPS)
    bound = 20 / math.log(10) * lin / (r + stoi_np.EPS) + 6 * U64 * np.abs(want)
    bad = ~(np.abs(got - want) <= bound)
    assert not bad.any(), (what, "energy", np.flatnonzero(bad)[:5], got[bad][:3], want[bad][:3])


def check_selection(sel, n_sel, x, what):
    keep = stoi_np.selection(x)
    assert n_sel == len(keep), (what, "n_sel", n_sel, len(keep))
    assert np.array_equal(sel[:n_sel], keep), (what, "kept frames", np.flatnonzero(sel[:n_sel] != keep)[:5])


def tob_bound(x, keep):
    """Per (STFT frame, band) bound of the band envelopes of x under the kept-frame list keep."""
    w = stoi_np.hann()
    nf = len(keep) - 1
    n = np.arange(STOI_FRAME)
    j = np.arange(nf)[:, None] + n[None, :] // STOI_HOP
    r = n % STOI_HOP
    xa = np.abs(x[keep[j] * STOI_HOP + r])
    xb = np.where(j >= 1, np.abs(x[keep[np.maximum(j - 1, 0)] * STOI_HOP + STOI_HOP + r]), 0.0)
    a = w * (w[r] * xa + w[STOI_HOP + r] * xb)
    d = 4 * U64 * a + DELTA_W * (1 + w) * (xa + xb)
    per = EPS_FFT * a.sum(1) + d.sum(1)                                  # [nf]: max_k |ΔX_k| of one side
    m = np.array([b - a_ for a_, b in stoi_np.band_edges()], np.float64)
    return 2 * np.sqrt(m)[None, :] * per[:, None], (m + 6) * U64


def check_tob(got, x, y, what):
    """got [n_sel - 1, 15]: the band envelopes of y (None: of x) under x's selection, against stoi_np.tob."""
    keep = stoi_np.selection(x)
    xt, yt = stoi_np.tob(x, x if y is None else y)
    want = (xt if y is None else yt).T
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ab, rel = tob_bound(x if y is None else y, keep)
    bound = ab + rel * want
    bad = ~(np.abs(got - want) <= bound)
    assert not bad.any(), (what, "band envelopes", np.argwhere(bad)[:3], got[bad][:3], want[bad][:3])


def check_run(out, cleans, degraded, pairs, lengths, what):
    """Every intermediate and score of a stoi_run against the oracle on the trimmed signals, and the workspace written
    exactly where the layout puts this call's values."""
    C = cleans.shape[0]
    Ls = [cleans.shape[1]] * C if lengths is None else list(lengths)
    for c in range(C):
        x = cleans[c, :Ls[c]]
        assert energy_margin(x) >= 1e-9, (what, c, "input too close to the 40 dB threshold")
        nfc, ns = n_fr_of(Ls[c]), int(out["n_sel"][c])
        assert np.array_equal(np.flatnonzero(out["energy_w"][c]), np.arange(nfc)), (what, c, "energy write set")
        assert np.array_equal(np.flatnonzero(out["sel_w"][c]), np.arange(ns)), (what, c, "sel write set")
        assert np.array_equal(out["tob_w"][c].all(1), out["tob_w"][c].any(1)), (what, c, "partial tob row")
        assert np.array_equal(np.flatnonzero(out["tob_w"][c].any(1)), np.arange(max(ns - 1, 0))), (what, c, "tob rows")
        check_energy(out["energy"][c, :nfc], x, (what, c))
        check_selection(out["sel"][c], ns, x, (what, c))
        if ns > 1:
            check_tob(out["tob"][c, :ns - 1], x, None, (what, c))
    for p, (c, g) in enumerate(pairs):
        row = out["tob"][C + p]
        if not (0 <= c < C and 0 <= g < degraded.shape[0]):
            assert np.isnan(out["d"][p]) and out["n_frames"][p] == -1, (what, p)
            assert not out["tob_w"][C + p].any(), (what, p, "a bad pair wrote band envelopes")
            continue
        x, y = cleans[c, :Ls[c]], degraded[g, :Ls[c]]
        ns = int(out["n_sel"][c])
        assert np.array_equal(np.flatnonzero(out["tob_w"][C + p].any(1)), np.arange(max(ns - 1, 0))), (what, p)
        if ns > 1:
            check_tob(row[:ns - 1], x, y, (what, "pair", p))
        assert out["n_frames"][p] == ns - 1, (what, p)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            # a single kept frame leaves no STFT frame, where the oracle's (and pystoi's) matmul has no operand:
            # below 30 frames the score is 1e-5 either way
            want = stoi_np.stoi_10k(x, y) if ns > 1 else 1e-5
        assert abs(out["d"][p] - want) <= 1e-9, (what, p, out["d"][p], want)
        if ns - 1 < STOI_SEG:
            assert out["d"][p] == 1e-5


def degraded_of(rng, cleans, k=1):
    """Noisy, silent and sign-flipped versions, float32-representable."""
    rows = []
    for x in cleans:
        sd = max(float(x.std()), 1e-3)
        rows += [x + 0.4 * sd * rng.standard_normal(len(x)), np.zeros_like(x), -x][:k + 2]
    return np.stack(rows).astype(np.float32).astype(np.float64)


# ==== A. stoi_select_kernel ==========================================================================================

SELECT_NFR = (1, 8, 15, 17, 255, 256, 257, 511, 512, 513)


def select_cases():
    """(n_fr, cleans [3, L]): every frame loud; silence runs straddling frames 256 and 512 (where they exist); silent."""
    out = []
    for n_fr in SELECT_NFR:
        L = STOI_FRAME + STOI_HOP * (n_fr - 1)
        a = loud(n_fr, n_fr)
        b = speechlike(1000 + n_fr, L, period=1 << 30).astype(np.float64)
        for f0, f1 in ((250, 262), (506, 515)):         # frames f0 .. f1 - 2 silent (those that exist)
            if f0 < n_fr - 1:
                b[STOI_HOP * f0:STOI_HOP * f1] = 0.0
        out.append((n_fr, np.stack([a, b, np.zeros(L)])))
    return out


def check_select_labels(cases):
    """Every n_fr of SELECT_NFR on its edge: one warp's frame, the warps' multiples +- 1, one scan pass +- 1, two."""
    nfr = [n for n, _ in cases]
    assert any(n % SEL_WARPS == 0 for n in nfr) and any(n % SEL_WARPS == 1 for n in nfr)
    assert any(n % SEL_WARPS == SEL_WARPS - 1 for n in nfr)
    for k in (1, 2):
        assert {k * SEL_THREADS - 1, k * SEL_THREADS, k * SEL_THREADS + 1} <= set(nfr)
    for n, cl in cases:
        assert cl.shape[1] == STOI_FRAME + STOI_HOP * (n - 1) and n_fr_of(cl.shape[1]) == n
        keep_b = stoi_np.selection(cl[1])
        for edge in (SEL_THREADS, 2 * SEL_THREADS):
            if n > edge:       # a silence run straddles the scan pass boundary: frames edge - 1 and edge dropped
                assert edge not in keep_b and edge - 1 not in keep_b and len(keep_b) < n
        assert len(stoi_np.selection(cl[0])) == n and len(stoi_np.selection(cl[2])) == n


def test_select_edges(dev):
    """n_fr at one warp, the warps' multiples +- 1, one and two scan passes +- 1; silence across a pass boundary; an
    all-silent clean; pairs that share a clean and a degraded signal used with several cleans."""
    cases = select_cases()
    check_select_labels(cases)
    rng = np.random.default_rng(5)
    for n_fr, cleans in cases:
        deg = degraded_of(rng, cleans[:2])                             # 6 rows
        pairs = [(0, 0), (0, 1), (0, 2), (1, 3), (1, 4), (2, 0), (1, 0), (2, 5)]
        out = stoi_run(dev, cleans, deg, pairs, what=("select", n_fr))
        check_run(out, cleans, deg, pairs, None, ("select", n_fr))


# ==== B. stoi_bands_kernel / stoi_score_kernel, lengths mode =========================================================

BAND_SCORE_NSEL = {"one_frame": 1, "nf%4=0": 41, "nf%4=1": 42, "nf%4=3": 44, "nf=29": 30, "nf=30": 31,
                   "J=17": 47, "J=18": 48, "J=170": 200}


def band_score_cases():
    """{label: (n_sel, extra samples)}: every clean loud, so n_sel is its frame count."""
    return {lab: (ns, (7 * i) % STOI_HOP) for i, (lab, ns) in enumerate(BAND_SCORE_NSEL.items())}


def check_band_score_labels(labels):
    for lab, ns in labels.items():
        nf = ns - 1
        J = nf - STOI_SEG + 1
        if lab.startswith("nf%4="):
            assert nf % BAND_WARPS == int(lab[-1]) and nf >= STOI_SEG
        elif lab.startswith("nf="):
            assert nf == int(lab[3:]) and nf in (STOI_SEG - 1, STOI_SEG)     # the 1e-5 branch and its edge
        elif lab == "J=17":
            assert J * STOI_BANDS == SCORE_THREADS - 1                  # 255 items: the last thread idle
        elif lab == "J=18":
            assert SCORE_THREADS < J * STOI_BANDS < 2 * SCORE_THREADS  # 270 items: the item loop wraps
        elif lab == "J=170":
            assert J * STOI_BANDS > 8 * SCORE_THREADS                   # several items per thread
        else:
            assert lab == "one_frame" and ns == 1
    assert {(ns - 1) % BAND_WARPS for lab, ns in labels.items() if ns > 1} == {0, 1, 2, 3}


def lengths_batch(rng):
    """Cleans of their own lengths (from 256 samples up to L) in rows of L, NaN past each; degraded rows NaN past the
    longest clean they are paired with; pairs sharing cleans and a degraded row used by cleans of two lengths."""
    cases = band_score_cases()
    labels = list(cases)
    xs = [loud(20 + i, ns, extra) for i, (ns, extra) in enumerate(cases.values())]
    xs.append(speechlike(99, 30000, period=4000).astype(np.float64))   # gated speech, the longest row
    labels.append("L")
    lengths = [len(x) for x in xs]
    L = max(lengths)
    C = len(xs)
    cleans = np.full((C, L), np.nan)
    for c, x in enumerate(xs):
        cleans[c, :len(x)] = x
    deg = np.full((2 * C, L), np.nan)
    pairs = []
    for c, x in enumerate(xs):
        sd = max(float(x.std()), 1e-3)
        deg[2 * c, :len(x)] = (x + 0.5 * sd * rng.standard_normal(len(x))).astype(np.float32)
        deg[2 * c + 1, :len(x)] = (0.3 * x + 2.0 * sd * rng.standard_normal(len(x))).astype(np.float32)
        pairs += [(c, 2 * c), (c, 2 * c + 1)]
    # degraded row 2 (finite up to clean 1's length) is also scored against the shorter clean 0, and a pair repeats
    assert lengths[0] < lengths[1]
    pairs += [(0, 2), (1, 2), (C - 1, 2 * (C - 1))]
    return cleans, deg, pairs, lengths, labels


def test_bands_and_score_edges_with_lengths(dev):
    """disco_stoi_lengths at every bands-group and score-loop edge: intermediates and scores against the oracle on the
    trimmed signals, nothing written past each clean's frames, NaN inputs past each length never read."""
    rng = np.random.default_rng(8)
    cleans, deg, pairs, lengths, labels = lengths_batch(rng)
    check_band_score_labels(BAND_SCORE_NSEL)
    assert min(lengths) == STOI_FRAME and max(lengths) == cleans.shape[1]
    out = stoi_run(dev, cleans, deg, pairs, lengths, what="lengths")
    assert np.isfinite(out["d"]).all()
    check_run(out, cleans, deg, pairs, lengths, "lengths")
    for c, lab in enumerate(labels[:-1]):
        assert out["n_sel"][c] == BAND_SCORE_NSEL[lab], (lab, out["n_sel"][c])


def test_lengths_all_full_equal_null_call(dev):
    """Every length equal to L: the same bits as the call without lengths, workspace included."""
    rng = np.random.default_rng(9)
    x = np.stack([speechlike(s, 20000, period=3000 + 700 * s) for s in range(3)]).astype(np.float64)
    deg = degraded_of(rng, x)
    pairs = [(0, 0), (1, 3), (2, 6), (0, 7), (2, 2)]
    a = stoi_run(dev, x, deg, pairs, what="null")
    b = stoi_run(dev, x, deg, pairs, [x.shape[1]] * 3, what="all L")
    for k in ("d", "n_sel", "n_frames"):
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k
    assert torch.equal(a["ws"], b["ws"])
    check_run(a, x, deg, pairs, None, "null")


def test_bad_pairs_leave_the_others_unchanged(dev):
    """A pair naming a clean or degraded row out of range gives NaN and n_frames = -1 and writes no band envelope; the
    other pairs' scores, frame counts and envelopes keep their bits."""
    rng = np.random.default_rng(10)
    x = np.stack([speechlike(s, 15000, period=2500 + 500 * s) for s in range(2)]).astype(np.float64)
    deg = degraded_of(rng, x)
    good = [(0, 0), (1, 4), (0, 2), (1, 0)]
    bad = [(-1, 0), (2, 1), (0, -1), (1, 6)]
    mixed = [good[0], bad[0], good[1], bad[1], bad[2], good[2], good[3], bad[3]]
    ref = stoi_run(dev, x, deg, good, what="good")
    out = stoi_run(dev, x, deg, mixed, what="mixed")
    check_run(out, x, deg, mixed, None, "mixed")
    C = x.shape[0]
    for i, pr in enumerate(mixed):
        if pr in good:
            k = good.index(pr)
            assert out["d"][i].tobytes() == ref["d"][k].tobytes() and out["n_frames"][i] == ref["n_frames"][k]
            assert np.array_equal(out["tob"][C + i].view(np.int64), ref["tob"][C + k].view(np.int64))
        else:
            assert np.isnan(out["d"][i]) and out["n_frames"][i] == -1
    assert np.array_equal(out["n_sel"], ref["n_sel"])


# ==== C. resampler with lengths ======================================================================================

def resample_lengths(fs):
    """Lengths whose L_b up mod down is 0, 1 and down - 1, L_b = 1, and L_b shorter than one polyphase filter."""
    from disco_b200 import stoi
    taps, up, down = stoi.resample_taps(fs)
    per_phase = -(-len(taps) // up)
    out = []
    for r in (0, 1, down - 1):
        L = next(L for L in range(3 * down + 17, 3 * down + 17 + down) if L * up % down == r)
        out.append(L)
    out += [1, max(2, per_phase // 2), 5 * down + 3 * per_phase + 1]
    assert min(out) == 1 and any(1 < L < per_phase for L in out)
    assert {L * up % down for L in out[:3]} == {0, 1, down - 1}
    return out


@pytest.mark.parametrize("fs", [8000, 16000, 22050, 44100, 48000])
def test_resample_poly_lengths(dev, fs):
    from disco_b200 import _lib, stoi
    taps, up, down = stoi.resample_taps(fs)
    lengths = resample_lengths(fs)
    L = max(lengths) + 11
    rng = np.random.default_rng(fs)
    x = np.full((len(lengths), L), np.nan, np.float32)
    for s, Lb in enumerate(lengths):
        x[s, :Lb] = rng.standard_normal(Lb)
    n_out = -(-L * up // down)
    g = Guarded(dev)
    y = g.new((len(lengths), n_out), torch.float64)
    xt, tt = torch.from_numpy(x).to(dev), torch.from_numpy(taps).to(dev)
    lh = np.ascontiguousarray(lengths, dtype=np.int32)
    ld = torch.from_numpy(lh).to(dev)
    _call("disco_resample_poly_lengths", _p(xt), _p(y), _p(tt), len(taps), up, down, len(lengths), L, _p(ld),
          lh.ctypes.data_as(_lib.c_int_p))
    g.check(("resample lengths", fs))
    got = y.cpu().numpy()
    for s, Lb in enumerate(lengths):
        n10 = -(-Lb * up // down)
        assert not np.any(got[s, n10:]), (fs, Lb, "not zero past ceil(L_b up / down)")
        ok, worst = resample_ok(got[s:s + 1, :n10], x[s:s + 1, :Lb], taps, up, down)
        assert ok, (fs, Lb, worst)


# ==== D. negative controls ===========================================================================================

def score_from_tob(X, Y):
    """stoi_np.stoi_10k's steps 4-5 on band envelopes X, Y [15, nf]."""
    J = X.shape[1] - STOI_SEG + 1
    xs = np.array([X[:, m:m + STOI_SEG] for m in range(J)])
    ys = np.array([Y[:, m:m + STOI_SEG] for m in range(J)])
    yp = np.minimum(ys * np.linalg.norm(xs, axis=2, keepdims=True) / (np.linalg.norm(ys, axis=2, keepdims=True)
                                                                        + stoi_np.EPS), xs * (1 + 10 ** 0.75))
    yp = yp - yp.mean(2, keepdims=True)
    xc = xs - xs.mean(2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + stoi_np.EPS
    xc /= np.linalg.norm(xc, axis=2, keepdims=True) + stoi_np.EPS
    return np.sum(yp * xc) / (J * STOI_BANDS)


def test_intermediate_checkers_reject_subtly_wrong_values(dev):
    """The energy checker rejects the energy of the frame one hop off, the selection checker two swapped entries, the
    band checker one envelope off by 1e-9 relative -- which moves the score by far less than the score check's 1e-9."""
    rng = np.random.default_rng(12)
    x = speechlike(31, 25000, period=4000).astype(np.float64)
    y = degraded_of(rng, x[None])[:1]
    out = stoi_run(dev, x[None], y, [(0, 0)], what="controls")
    check_run(out, x[None], y, [(0, 0)], None, "controls")
    e = out["energy"][0].copy()
    f = int(np.argmax(np.abs(np.diff(e))))
    e[f] = e[f + 1]
    with pytest.raises(AssertionError):
        check_energy(e, x, "frame one hop off")
    ns = int(out["n_sel"][0])
    sel = out["sel"][0].copy()
    sel[[3, 4]] = sel[[4, 3]]
    with pytest.raises(AssertionError):
        check_selection(sel, ns, x, "two entries swapped")
    tob = out["tob"][0, :ns - 1].copy()
    t, b = np.unravel_index(np.argmax(tob), tob.shape)
    tob[t, b] *= 1 + 1e-9
    with pytest.raises(AssertionError):
        check_tob(tob, x, None, "one envelope off by 1e-9")
    X, Y = stoi_np.tob(x, y[0])
    Xb = X.copy()
    Xb[b, t] *= 1 + 1e-9
    assert abs(score_from_tob(X, Y) - stoi_np.stoi_10k(x, y[0])) <= 1e-12       # the restatement is faithful
    assert abs(score_from_tob(Xb, Y) - score_from_tob(X, Y)) < 1e-10            # invisible to the score check
