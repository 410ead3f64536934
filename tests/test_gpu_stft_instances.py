"""Every instantiation of the fused STFT kernel (stft_scm.cu) and of the consumers of its partial-sum workspace against
float64, at the frame counts, signal lengths and launch geometries where its tiling and segment layout have edges,
through the C ABI with every output and the workspace inside NaN-filled guard bands.

Dispatch targets (INSTANCES below; tests/test_stft_instances_cpu.py parses the dispatch sets out of the sources and
requires this table to cover exactly them):
  stft              disco_stft           stft_scm_kernel<N, C, 0, OUT_Y>, C = min(4, n_sig)
  stft_scm          disco_stft_scm       stft_scm_kernel<N, C, 1, OUT_Y>
  stft_scm2         disco_stft_scm2      stft_scm_kernel<N, C, 2, OUT_Y>        (Y given)
  stft_scm2_none    disco_stft_scm2      stft_scm_kernel<N, C, 2, OUT_NONE>     (Y = NULL)
  stft_filter_dual  disco_stft_filter_dual  stft_scm_kernel<N, C, 0, OUT_FILTER / OUT_FILTER_FT>
  scm_finalize      disco_scm_from_workspace (and disco_stft_scm with Rss, Rnn)  scm_finalize_kernel<C>
  solve_workspace   disco_mwf_solve_workspace / _workspace2: mwf_solve_kernel reading the partial sums (load_part)
  filter_dual       disco_filter_dual    filter_dual_kernel<C, OUT_FT>

Tolerances are entry-wise first-order float32 bounds (u = 2^-24), derived from the kernels' arithmetic:
  Y        |Y - Y^f64| <= tol_fft * E, E = sum_n w_n (|x_a[n]| + |x_b[n]|) over the padded frame of the channel's
           two-for-one pair (a lone channel of an odd group: its own samples only).  One complex FFT transforms
           (w/2)(x_a + i x_b); a radix-2 stage rounds each output at most 4 times relative to |a| + |b| of its
           butterfly (the two ffma2 of x = a + w b, the float table value of w, the ffma2 of y = 2a - x, fft_reg.cuh;
           trivial twiddles round once), and the partial sums of a stage are bounded by the sum of the inputs' moduli,
           so log2 N stages err by at most 4 log2 N u sum |w/2||x_a + i x_b|.  On top: the inter-pass twiddle
           product (cmul: 2 roundings + the table value), the window product and its table value (2), and the
           un-mixing fadd2 (1), which adds two such errors (A = Z[f] + conj(Z[N - f])) and so doubles the w/2 envelope
           to w.  tol_fft = sqrt(2) (4 log2 N + 6) u, sqrt(2) for the complex modulus.  Bins 0 and F - 1 are real by
           construction: their imaginary parts must be exactly 0.
  Rss/Rnn  against the complex128 masked SCM of the kernel's own stored Y (for OUT_NONE the Y of the OUT_Y twin,
           whose workspace must be bit-identical):  |R - R^f64| <= tol * (1/T) sum_t w_t |y_i||y_j|,
           tol = sqrt(2) (T + n_slot + 6) u: the frames of a (group, CTA) segment are summed sequentially and the
           n_slot segments of the group in slot order (finalize, load_part), and 6 covers one term (m^2 or (1 - m)
           and its square, the two roundings of the product y_i conj(y_j)) and the 1/T scale (1/T and the product).
  filters  filter_dual: check_filter of test_gpu_kernel_instances (D = C).  The filter pass must equal
           filter_dual(W1, W2, Y_g) bit for bit, Y_g = disco_stft of the group's C signals (same pairing).
  solver   W, T1 from the workspace solve bit-identical to mwf_solve on the finalized matrices.
These are bounds, not fits: a wrong sample, twiddle, pair index or slot is an O(1) error against them.

Workspace write set: the partial sums live in a buffer pre-filled with the NaN sentinel.  By the segment contract
(kernels.h) CTA b of n_cta = min(total, SMs - reserved) owns tiles [total b / n_cta, total (b + 1) / n_cta); the CTAs
whose range meets group g write its slots 0 .. n_slot(g) - 1.  Every word of those slots must be written, every word
of the slots behind them and of the guard bands must keep the sentinel, and finalize and the solver, run on that
poisoned workspace, must give finite results within the bounds above: they read only written slots.
"""
import ctypes
import functools
import math

import numpy as np
import pytest
import torch

from test_gpu_kernel_instances import GUARD, SENTINEL, U, Guarded, assert_bounded, check_filter, ref_scm

pytestmark = pytest.mark.gpu

ERR_UNSUPPORTED = -2
N_FFTS = (256, 512, 1024)
C1_4 = tuple(range(1, 5))
C1_8 = tuple(range(1, 9))
# one row per dispatch target: n_fft -> channel counts (or the channel counts of an n_fft-independent kernel)
INSTANCES = {
    "stft": {256: C1_4, 512: C1_4, 1024: C1_4},
    "stft_scm": {256: C1_8, 512: C1_8, 1024: C1_4},
    "stft_scm2": {256: C1_4, 512: C1_4},
    "stft_scm2_none": {256: C1_4, 512: C1_4},
    "stft_filter_dual": {256: C1_4, 512: C1_4},      # both layouts each
    "scm_finalize": {"C": C1_8},
    "solve_workspace": {"C": C1_4, "n_set": (1, 2)},
    "filter_dual": {"C": C1_4, "layout": ("TF", "FT")},
}
# n_mask of each stft_scm_kernel row
NM_OF = {"stft": 0, "stft_scm": 1, "stft_scm2": 2, "stft_scm2_none": 2, "stft_filter_dual": 0}


def tile_frames(n_fft, C):
    """stft_tile_frames: TT = 8 (32 / RA) / ceil(C / 2), RA = n_fft / 32."""
    return 8 * (32 // (n_fft // 32)) // ((C + 1) // 2)


# ---- the segment contract of kernels.h, restated ------------------------------------------------------------------

def segments(n_grp, tp, sms):
    """(n_cta, lo, hi, n_slot): CTA b owns tiles [lo[b], hi[b]); n_slot[g] CTAs meet group g."""
    total = n_grp * tp
    n_cta = min(total, sms)
    b = np.arange(n_cta, dtype=np.int64)
    lo, hi = total * b // n_cta, total * (b + 1) // n_cta
    d = np.zeros(n_grp + 1, np.int64)
    np.add.at(d, lo // tp, 1)
    np.add.at(d, (hi - 1) // tp + 1, -1)
    return n_cta, lo, hi, np.cumsum(d)[:n_grp]


def slots_bound(n_grp, tp, n_cta):
    """stft_slots_per_grp."""
    min_range = n_grp * tp // n_cta
    return tp + 1 if min_range == 0 else tp // min_range + 2


def geometry_classes(n_grp, tp, sms):
    """Which of the launch-geometry classes a batch of n_grp groups of tp tiles falls in."""
    n_cta, lo, hi, n_slot = segments(n_grp, tp, sms)
    total = n_grp * tp
    out = set()
    if total < sms and np.all(hi - lo == 1) and np.all(n_slot == tp):
        out.add("one tile per CTA")
    if total == sms:
        out.add("total = S")
    if total == sms + 1:
        out.add("total = S + 1")
    if tp == 1 and n_grp == 3 * sms + 1:
        out.add("CTA walks whole groups")
    if n_grp == 1 and tp >= 5 * sms and n_slot[0] == sms:
        out.add("one group over every CTA")
    if n_slot.max() == slots_bound(n_grp, tp, n_cta):
        out.add("slots bound tight")
    if np.any((hi - lo >= 2) & (lo % tp != 0)):
        out.add("multi-tile range from mid-group")
    return out


ALL_CLASSES = {"one tile per CTA", "total = S", "total = S + 1", "CTA walks whole groups", "one group over every CTA",
               "slots bound tight", "multi-tile range from mid-group"}


@functools.lru_cache(maxsize=None)
def tight_shape(sms):
    """The smallest (n_grp, tp) with n_grp, tp > 1 whose largest slot count equals slots_per_grp."""
    best = None
    for g in range(2, 80):
        for tp in range(2, 60):
            if g * tp > sms and (best is None or g * tp < best[0] * best[1]):
                n_cta, _, _, n_slot = segments(g, tp, sms)
                if n_slot.max() == slots_bound(g, tp, n_cta):
                    best = (g, tp)
    return best


def geometry_shapes(sms):
    """(n_grp, tp) of the six geometry cases for S = sms CTAs."""
    return [((sms - 1) // 3, 3),            # total < S: one tile per CTA, a group over 3 CTAs
            (sms, 1), (sms + 1, 1),         # total = S, S + 1
            (3 * sms + 1, 1),               # a CTA walks several whole groups
            (1, 5 * sms),                   # one group over every CTA, n_slot = S
            tight_shape(sms),               # max n_slot = slots_per_grp
            (7, (5 * sms) // 14)]           # ranges of 2-3 tiles starting inside groups


# ---- device helpers ---------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _lib():
    from disco_b200 import _lib as lib_mod
    return lib_mod.load()


def _call(fn, *args):
    from disco_b200 import _lib as lib_mod, ops
    lib_mod.check(getattr(_lib(), fn)(*args, ops._stream()))


def _p(t):
    from disco_b200 import ops
    return ops._ptr(t)


def ws_bytes_unreserved():
    """(library, segment contract with no SM reserved) workspace bytes of one 4-channel group of 20 000 frames at
    n_fft 512: its n_cta is the number of SMs the kernel may use, so the bytes change with the reserved-SM setting."""
    L = 256 * 19999
    tp = -(-(1 + L // 256) // tile_frames(512, 4))
    n_cta = segments(1, tp, n_sms())[0]
    return _lib().disco_stft_scm_workspace(1, 4, L, 512), slots_bound(1, tp, n_cta) * 2 * 4 * 4 * 257 * 4


@pytest.fixture(scope="module")
def reserved(request, dev):
    """disco_set_reserved_sms(r) for the tests of this module that ask for it; always restored to 0."""
    r = getattr(request, "param", 0)
    lib = _lib()
    assert lib.disco_set_reserved_sms(r) == 0
    try:
        yield r
    finally:
        assert lib.disco_set_reserved_sms(0) == 0
        got, want = ws_bytes_unreserved()
        assert got == want, "reserved SMs not restored to 0"


class Workspace:
    """Partial-sum workspace inside a sentinel-filled buffer with guard bands."""

    def __init__(self, dev, nbytes):
        assert nbytes % 4 == 0
        self.n = nbytes // 4
        self.buf = torch.full((self.n + 2 * GUARD,), SENTINEL, dtype=torch.int32, device=dev)
        self.ws = self.buf[GUARD:GUARD + self.n].view(torch.float32)
        self.nbytes = nbytes


def check_write_set(ws, n_grp, spg, n_slot, what):
    """Every word of slots < n_slot[g] written, every word of slots >= n_slot[g] and of the guards untouched."""
    torch.cuda.synchronize()
    buf = ws.buf.cpu().numpy()
    assert np.all(buf[:GUARD] == SENTINEL) and np.all(buf[GUARD + ws.n:] == SENTINEL), \
        what + ": workspace guard band written"
    w = buf[GUARD:GUARD + ws.n].reshape(n_grp, spg, -1) == SENTINEL
    used = np.arange(spg)[None, :] < n_slot[:, None]
    unwritten = w[used].sum()
    assert unwritten == 0, "%s: %d words of written slots never written" % (what, unwritten)
    stray = (~w[~used]).sum()
    assert stray == 0, "%s: %d words written into slots no CTA owns" % (what, stray)


# ---- inputs and float64 references ------------------------------------------------------------------------------

def hann(n_fft):
    n = np.arange(n_fft, dtype=np.float64)
    return 0.5 - 0.5 * np.cos(2.0 * np.pi * n / n_fft)


def ref_stft(x, n_fft):
    """x (n_sig, L) float32 -> Y (n_sig, T, F) complex128 and the per-(signal, frame) sum_n w_n |x[n]|, via
    oracle.librosa_np.stft for the spectrum."""
    from oracle import librosa_np
    hop = n_fft // 2
    n_sig, L = x.shape
    T = 1 + L // hop
    xd = x.astype(np.float64)
    Y = np.stack([librosa_np.stft(xd[i], n_fft, hop, dtype=np.complex128).T for i in range(n_sig)])
    pad = np.pad(np.abs(xd), ((0, 0), (hop, hop)), mode="reflect")
    idx = np.arange(n_fft)[None, :] + hop * np.arange(T)[:, None]
    A = pad[:, idx] @ hann(n_fft)                                   # (n_sig, T)
    return Y, A


def pair_envelope(A, n_sig, C):
    """E of every signal: its own sum_n w |x| plus that of its two-for-one partner (signals grouped by C, channels
    (0, 1), (2, 3), ... of a group paired; the partner must exist, the last group may be short)."""
    E = A.copy()
    for s in range(n_sig):
        c = s % C
        partner = s + 1 if c % 2 == 0 else s - 1
        if c % 2 == 1 or (c + 1 < C and partner < n_sig):
            E[s] += A[partner]
    return E


def tol_fft(n_fft):
    return math.sqrt(2) * (4 * math.log2(n_fft) + 6) * U


def tol_scm1(T, n_slot):
    return math.sqrt(2) * (T + n_slot + 6) * U


def check_Y(Y, x, n_fft, C, what):
    """Y (n_sig, T, F) complex64 of signals grouped by C against float64, entry-wise; Nyquist and DC real."""
    Yh = Y.cpu().numpy()
    n_sig = x.shape[0]
    assert not Yh[..., 0].imag.any() and not Yh[..., -1].imag.any(), what + ": DC / Nyquist bin not real"
    Yr, A = ref_stft(x, n_fft)
    E = pair_envelope(A, n_sig, C)
    assert_bounded(Yh, Yr, np.broadcast_to(E[:, :, None], Yr.shape), tol_fft(n_fft), what + " Y")


def make_x(rng, dev, n_sig, L, misaligned=False):
    x = rng.standard_normal((n_sig, L)).astype(np.float32)
    if not misaligned:
        return x, torch.from_numpy(x).to(dev)
    buf = torch.zeros(n_sig * L + 4, dtype=torch.float32, device=dev)
    xd = buf[1:1 + n_sig * L]
    xd.copy_(torch.from_numpy(x.reshape(-1)))
    assert xd.data_ptr() % 16 == 4
    return x, xd


def make_mask(rng, dev, G, T, F, binary, layout):
    m = rng.uniform(size=(G, T, F)).astype(np.float32)
    if binary:
        m = (m > 0.5).astype(np.float32)
    mh = m if layout == "TF" else np.ascontiguousarray(m.transpose(0, 2, 1))
    return m, torch.from_numpy(mh).to(dev)


def checked_groups(n_grp, tp, sms, limit=12):
    """All groups of a small batch; of a large one the first and last group of every CTA range."""
    if n_grp <= limit:
        return list(range(n_grp))
    _, lo, hi, _ = segments(n_grp, tp, sms)
    return sorted(set((lo // tp).tolist()) | set(((hi - 1) // tp).tolist()))


# ---- one run of an instantiation --------------------------------------------------------------------------------

def run_stft(dev, rng, n_fft, n_sig, L, misaligned=False):
    """disco_stft (NM = 0, OUT_Y): Y against float64."""
    x, xd = make_x(rng, dev, n_sig, L, misaligned)
    T, F = 1 + L // (n_fft // 2), n_fft // 2 + 1
    o = Guarded(dev)
    Y = o.new((n_sig, T, F))
    _call("disco_stft", _p(xd), _p(Y), n_sig, L, n_fft)
    what = "stft N=%d n_sig=%d L=%d T=%d%s" % (n_fft, n_sig, L, T, " misaligned" if misaligned else "")
    o.check(what)
    check_Y(Y, x, n_fft, min(4, n_sig), what)


def check_scm_groups(Rss, Rnn, Yh, masks, groups, n_slot, T, what):
    """Rss, Rnn [G, F, C, C] of the listed groups against the complex128 SCMs of Yh [G, C, T, F] under masks
    [G, T, F]; exact mirrors and real diagonals everywhere."""
    for R in (Rss, Rnn):
        assert torch.equal(R, R.conj().transpose(-1, -2)), what + ": mirrors not exactly conjugate"
        assert not bool(torch.diagonal(torch.view_as_real(R), dim1=-3, dim2=-2)[..., 1, :].any()), \
            what + ": diagonal with an imaginary part"
    Rs, Rn = Rss.cpu().numpy(), Rnn.cpu().numpy()
    for g in groups:
        ws_, wn_, es, en = ref_scm(Yh[g], masks[g])
        tol = tol_scm1(T, int(n_slot[g]))
        assert_bounded(Rs[g], ws_, es, tol, "%s Rss group %d" % (what, g))
        assert_bounded(Rn[g], wn_, en, tol, "%s Rnn group %d" % (what, g))


def solve_checks(dev, ws, Rs_list, G, C, L, n_fft, what):
    """The workspace solve (one or two mask sets) against mwf_solve on the finalized matrices, bit for bit."""
    F = n_fft // 2 + 1
    n_set = len(Rs_list)
    o = Guarded(dev)
    W, T1 = o.new((n_set, G, F, C)), o.new((n_set, G, F, C))
    if n_set == 1:
        Rso, Rno = o.new((G, F, C, C)), o.new((G, F, C, C))
        _call("disco_mwf_solve_workspace", _p(ws.ws), _p(W), _p(T1), _p(Rso), _p(Rno), G, C, L, n_fft, 0, 1,
              ctypes.c_double(1.0))
    else:
        _call("disco_mwf_solve_workspace2", _p(ws.ws), _p(W), _p(T1), G, C, L, n_fft, 0, 1, ctypes.c_double(1.0))
    o.check("solve_workspace " + what)
    Rss = torch.stack([r[0] for r in Rs_list]).contiguous()
    Rnn = torch.stack([r[1] for r in Rs_list]).contiguous()
    if n_set == 1:
        assert torch.equal(Rso, Rss[0]) and torch.equal(Rno, Rnn[0]), what + ": want_scm matrices differ from finalize"
    o = Guarded(dev)
    W0, T10 = o.new((n_set, G, F, C)), o.new((n_set, G, F, C))
    _call("disco_mwf_solve", _p(Rss), _p(Rnn), _p(W0), _p(T10), n_set * G * F, C, 0, 1, ctypes.c_double(1.0))
    o.check("mwf_solve " + what)
    assert bool(torch.isfinite(torch.view_as_real(W)).all()), what + ": workspace solve not finite"
    assert torch.equal(W, W0) and torch.equal(T1, T10), what + ": workspace solve differs from mwf_solve"


def run_scm(dev, rng, kind, n_fft, C, G, L, layout="TF", binary=False, misaligned=False, sms=None):
    """stft_scm (NM = 1) or stft_scm2 (NM = 2, with Y and without): Y against float64, the workspace write set,
    finalize against float64 on the poisoned workspace, the workspace solve against mwf_solve."""
    lib = _lib()
    sms = sms or n_sms()
    hop, F = n_fft // 2, n_fft // 2 + 1
    T = 1 + L // hop
    tp = -(-T // tile_frames(n_fft, C))
    n_cta, _, _, n_slot = segments(G, tp, sms)
    nm = 1 if kind == "stft_scm" else 2
    x, xd = make_x(rng, dev, G * C, L, misaligned)
    masks = [make_mask(rng, dev, G, T, F, binary, layout) for _ in range(nm)]
    lay = 0 if layout == "TF" else 1
    nbytes = (lib.disco_stft_scm_workspace if nm == 1 else lib.disco_stft_scm2_workspace)(G, C, L, n_fft)
    spg = nbytes // (G * nm * 2 * C * C * F * 4)
    assert spg * G * nm * 2 * C * C * F * 4 == nbytes and spg == slots_bound(G, tp, n_cta)
    what = "%s N=%d C=%d G=%d L=%d T=%d tiles/grp=%d n_cta=%d %s%s%s" % (
        kind, n_fft, C, G, L, T, tp, n_cta, layout, " binary" if binary else "", " misaligned" if misaligned else "")
    o = Guarded(dev)
    Y = o.new((G, C, T, F))
    ws = Workspace(dev, nbytes)
    if nm == 1:
        Rss, Rnn = o.new((G, F, C, C)), o.new((G, F, C, C))
        _call("disco_stft_scm", _p(xd), _p(masks[0][1]), lay, _p(Y), _p(Rss), _p(Rnn), G, C, L, n_fft, _p(ws.ws),
              nbytes)
    else:
        _call("disco_stft_scm2", _p(xd), _p(masks[0][1]), _p(masks[1][1]), lay, _p(Y), G, C, L, n_fft, _p(ws.ws),
              nbytes)
    o.check(what)
    check_write_set(ws, G, spg, n_slot, what)
    groups = checked_groups(G, tp, sms)
    sig = np.array([g * C + c for g in groups for c in range(C)])
    Ysel = Y.view(G * C, T, F)[torch.from_numpy(sig).to(dev)]
    check_Y(Ysel, x[sig], n_fft, C, what)
    if nm == 2:
        ws0 = Workspace(dev, nbytes)       # OUT_NONE twin: the same partial sums, slot for slot, guards included
        _call("disco_stft_scm2", _p(xd), _p(masks[0][1]), _p(masks[1][1]), lay, None, G, C, L, n_fft, _p(ws0.ws),
              nbytes)
        torch.cuda.synchronize()
        assert torch.equal(ws0.buf, ws.buf), what + ": OUT_NONE workspace differs from the run that stores Y"
    Yh = Y.cpu().numpy()
    mats = []
    for q in range(nm):
        o = Guarded(dev)
        Rs2, Rn2 = o.new((G, F, C, C)), o.new((G, F, C, C))
        _call("disco_scm_from_workspace", _p(ws.ws), nm, q, _p(Rs2), _p(Rn2), G, C, L, n_fft)
        o.check("scm_finalize " + what)
        if nm == 1:
            assert torch.equal(Rs2, Rss) and torch.equal(Rn2, Rnn), what + ": finalize differs from the fused call"
        check_scm_groups(Rs2, Rn2, Yh, masks[q][0], groups, n_slot, T, "%s set %d" % (what, q))
        mats.append((Rs2, Rn2))
    if C <= 4:
        solve_checks(dev, ws, mats, G, C, L, n_fft, what)
    else:
        o = Guarded(dev)
        W, T1 = o.new((G, F, C)), o.new((G, F, C))
        from disco_b200 import ops
        rc = lib.disco_mwf_solve_workspace(_p(ws.ws), _p(W), _p(T1), None, None, G, C, L, n_fft, 0, 1,
                                           ctypes.c_double(1.0), ops._stream())
        assert rc != 0, what + ": workspace solve accepted C > 4"
        torch.cuda.synchronize()
        assert all(bool((b[GUARD:GUARD + n] == SENTINEL).all()) for b, n in o.bufs), what + ": rejected call wrote"


def run_filter(dev, rng, n_fft, C, G, L, layout, ref, misaligned=False, sms=None):
    """stft_filter_dual (OUT_FILTER / OUT_FILTER_FT): bit-identical to filter_dual(W1, W2, Y_g), Y_g from disco_stft
    per group; filter_dual against float64 on Y_g."""
    hop, F = n_fft // 2, n_fft // 2 + 1
    T = 1 + L // hop
    sms = sms or n_sms()
    tp = -(-T // tile_frames(n_fft, C))
    x, xd = make_x(rng, dev, G * C, L, misaligned)
    cplx = lambda *s: (rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)
    W1, W2 = cplx(G, F, C), cplx(G, F, C)
    W1d, W2d = torch.from_numpy(W1).to(dev), torch.from_numpy(W2).to(dev)
    lay = 0 if layout == "TF" else 1
    shape = (G, T, F) if layout == "TF" else (G, F, T)
    what = "stft_filter_dual N=%d C=%d G=%d L=%d T=%d %s ref=%d%s" % (n_fft, C, G, L, T, layout, ref,
                                                                     " misaligned" if misaligned else "")
    o = Guarded(dev)
    z, zn, yf = o.new(shape), o.new(shape), o.new(shape)
    _call("disco_stft_filter_dual", _p(xd), _p(W1d), _p(W2d), _p(z), _p(zn), _p(yf), ref, lay, G, C, L, n_fft)
    o.check(what)
    xg = torch.from_numpy(x).to(dev).view(G, C, L)
    Y = torch.empty((G, C, T, F), dtype=torch.complex64, device=dev)
    for g in range(G):
        _call("disco_stft", _p(xg[g]), _p(Y[g]), C, L, n_fft)
    o = Guarded(dev)
    z0, zn0, yf0 = o.new(shape), o.new(shape), o.new(shape)
    _call("disco_filter_dual", _p(W1d), _p(W2d), _p(Y), _p(z0), _p(zn0), _p(yf0), ref, lay, G, C, T, n_fft)
    o.check("filter_dual " + what)
    assert torch.equal(z, z0) and torch.equal(zn, zn0) and torch.equal(yf, yf0), what + ": differs from filter_dual"
    Yh = Y.cpu().numpy()
    zh, znh, yfh = (a.cpu().numpy() for a in (z0, zn0, yf0))
    if layout == "FT":
        zh, znh, yfh = (a.transpose(0, 2, 1) for a in (zh, znh, yfh))
    for g in checked_groups(G, tp, sms, limit=6):
        check_filter(zh[g], znh[g], W1[g], Yh[g], True, ref, "filter_dual %s group %d z" % (what, g))
        check_filter(yfh[g], None, W2[g], Yh[g], True, ref, "filter_dual %s group %d yf" % (what, g))


# ---- frame and length edges -------------------------------------------------------------------------------------

def edge_lengths(n_fft, C):
    """(L, misaligned) of the frame edges T = 2, 3, TT - 1, TT, TT + 1, 2 TT + 1, 300 with L = (T - 1) hop + r,
    r rotating over 0, 1, 3, hop - 1; the shortest signal L = hop + 1; one 16-byte-misaligned x with L % 4 == 0."""
    hop, tt = n_fft // 2, tile_frames(n_fft, C)
    rs = (0, 1, 3, hop - 1)
    out = []
    for i, T in enumerate(sorted({2, 3, tt - 1, tt, tt + 1, 2 * tt + 1, 300})):
        r = rs[i % 4]
        if (T - 1) * hop + r <= hop:
            r = 1
        out.append(((T - 1) * hop + r, False))
    out.append((hop + 1, False))
    out.append((tt * hop, True))                   # T = TT + 1, L % 4 == 0, x 4 bytes past a 16-byte boundary
    return out


def kinds_and_shapes():
    out = []
    for kind in ("stft_scm", "stft_scm2", "stft_filter_dual"):
        for n_fft, cs in INSTANCES[kind].items():
            out += [(kind, n_fft, C) for C in cs]
    return out


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("n_sig", (1, 2, 3, 4, 5, 6, 7, 9))
def test_stft_edges(dev, reserved, n_fft, n_sig):
    """The plain STFT: C = min(4, n_sig) channels per group, the last group 1..3 channels short for n_sig 5, 6, 7, 9,
    at every frame and length edge; L = hop must be rejected."""
    C = min(4, n_sig)
    rng = np.random.default_rng(100 * n_fft + n_sig)
    for L, mis in edge_lengths(n_fft, C):
        run_stft(dev, rng, n_fft, n_sig, L, mis)
    o = Guarded(dev)
    Y = o.new((n_sig, 2, n_fft // 2 + 1))
    x = torch.zeros(n_sig * n_fft, device=dev)
    from disco_b200 import ops
    assert _lib().disco_stft(_p(x), _p(Y), n_sig, n_fft // 2, n_fft, ops._stream()) == -1, "L = hop accepted"


@pytest.mark.parametrize("kind,n_fft,C", kinds_and_shapes())
def test_fused_edges(dev, reserved, kind, n_fft, C):
    """The fused kernels at every frame and length edge, masks uniform and binary in both layouts (filter pass: both
    output layouts, references rotating); L = hop must be rejected."""
    rng = np.random.default_rng(1000 * n_fft + 10 * C + len(kind))
    hop = n_fft // 2
    for i, (L, mis) in enumerate(edge_lengths(n_fft, C)):
        G = 2 if L > 100 * hop else 3
        if kind == "stft_filter_dual":
            run_filter(dev, rng, n_fft, C, G, L, ("TF", "FT")[i % 2], (C - 1, 0, C // 2)[i % 3], mis)
        else:
            run_scm(dev, rng, kind, n_fft, C, G, L, layout=("TF", "FT")[i % 2], binary=(i // 2) % 2 == 1,
                    misaligned=mis)
    lib = _lib()
    from disco_b200 import ops
    x = torch.zeros(C * n_fft, device=dev)
    if kind == "stft_scm":
        rc = lib.disco_stft_scm(_p(x), _p(x), 0, _p(x), None, None, 1, C, hop, n_fft, _p(x), 1 << 20, ops._stream())
    elif kind == "stft_scm2":
        rc = lib.disco_stft_scm2(_p(x), _p(x), _p(x), 0, None, 1, C, hop, n_fft, _p(x), 1 << 20, ops._stream())
    else:
        rc = lib.disco_stft_filter_dual(_p(x), _p(x), _p(x), _p(x), None, _p(x), 0, 0, 1, C, hop, n_fft,
                                        ops._stream())
    assert rc == -1, "L = hop accepted"


# ---- launch geometry --------------------------------------------------------------------------------------------

def geometry_params():
    """Every instantiation at reserved = 0; the first channel count of each (n_fft, kind) at 16 and 64."""
    out = []
    for r in (0, 16, 64):
        for n_fft in N_FFTS:
            for kind in ("stft", "stft_scm", "stft_scm2", "stft_filter_dual"):
                cs = INSTANCES[kind].get(n_fft, ())
                for C in (cs if r == 0 else cs[:1]):
                    out.append(pytest.param(r, kind, n_fft, C, id="r%d-%s-%d-%d" % (r, kind, n_fft, C)))
    return out


@pytest.mark.parametrize("reserved,kind,n_fft,C", geometry_params(), indirect=["reserved"])
def test_geometry(dev, reserved, kind, n_fft, C):
    """Every geometry class on S = SMs - reserved CTAs.  The plain STFT takes its groups from n_sig (C = 4: n_sig =
    4 G; C < 4: one group only, so it runs the single-group classes)."""
    sms = n_sms() - reserved
    hop, tt = n_fft // 2, tile_frames(n_fft, C)
    rng = np.random.default_rng(7 * n_fft + C + reserved)
    for i, (G, tp) in enumerate(geometry_shapes(sms)):
        T = max(2, tp * tt - (i % 2))             # the last tile of a group full or one frame short
        L = (T - 1) * hop + (0, 1, 3)[i % 3] if T > 2 else hop + 1
        if kind == "stft":
            if C < 4 and G > 1:
                continue
            run_stft(dev, rng, n_fft, G * C, L)
        elif kind == "stft_filter_dual":
            run_filter(dev, rng, n_fft, C, G, L, ("TF", "FT")[i % 2], i % C, sms=sms)
        else:
            run_scm(dev, rng, kind, n_fft, C, G, L, layout=("TF", "FT")[i % 2], binary=i % 3 == 2, sms=sms)


# ---- unsupported combinations -----------------------------------------------------------------------------------

def test_unsupported_combinations_rejected(dev):
    """Outside the table the ABI returns DISCO_ERR_UNSUPPORTED and writes nothing; ops raises NotImplementedError."""
    from disco_b200 import ops
    lib = _lib()
    table = {(n, c, NM_OF[k]) for k in NM_OF for n, cs in INSTANCES[k].items() for c in cs}
    L = 4000
    x = torch.zeros((1, 9, L), device=dev)
    for n_fft in N_FFTS:
        F, T = n_fft // 2 + 1, 1 + L // (n_fft // 2)
        for C in range(1, 9):
            for nm in (0, 1, 2):
                assert bool(lib.disco_stft_scm_supported(n_fft, C, nm)) == ((n_fft, C, nm) in table), (n_fft, C, nm)
            m = torch.zeros((1, T, F), device=dev)
            xc = x[:, :C].contiguous()
            W = torch.zeros((1, F, C), dtype=torch.complex64, device=dev)
            if (n_fft, C, 1) not in table:
                o = Guarded(dev)
                Y, R = o.new((1, C, T, F)), o.new((1, F, C, C))
                ws = torch.zeros(1 << 20, device=dev)
                rc = lib.disco_stft_scm(_p(xc), _p(m), 0, _p(Y), _p(R), _p(R), 1, C, L, n_fft, _p(ws), 1 << 22,
                                        ops._stream())
                assert rc == ERR_UNSUPPORTED, (n_fft, C, rc)
                torch.cuda.synchronize()
                assert all(bool((b == SENTINEL).all()) for b, _ in o.bufs), (n_fft, C)
                with pytest.raises(NotImplementedError):
                    ops.stft_scm(xc, m, n_fft)
            if (n_fft, C, 2) not in table:
                o = Guarded(dev)
                Y, z = o.new((1, C, T, F)), o.new((1, T, F))
                ws = Workspace(dev, 1 << 20)
                rc = lib.disco_stft_scm2(_p(xc), _p(m), _p(m), 0, _p(Y), 1, C, L, n_fft, _p(ws.ws), ws.nbytes,
                                         ops._stream())
                assert rc == ERR_UNSUPPORTED, (n_fft, C, rc)
                rc = lib.disco_stft_filter_dual(_p(xc), _p(W), _p(W), _p(z), _p(z), _p(z), 0, 0, 1, C, L, n_fft,
                                                ops._stream())
                assert rc == ERR_UNSUPPORTED, (n_fft, C, rc)
                torch.cuda.synchronize()
                assert all(bool((b == SENTINEL).all()) for b, _ in o.bufs) and bool((ws.buf == SENTINEL).all())
                with pytest.raises(NotImplementedError):
                    ops.stft_scm2(xc, m, m, n_fft)
                with pytest.raises(NotImplementedError):
                    ops.stft_filter_dual(xc, W, W, n_fft=n_fft)
