"""BSS-eval on the device (csrc/bss.cu, disco_b200/bss_eval.py, post.tango_scores) against the float64 oracle
(oracle/bss_np.py, mir_eval's published algorithm).

Tolerance: |ΔdB| <= 1e-6 + 4 |LU - SVD|, where LU (np.linalg.solve, as mir_eval) and SVD (least squares) are the
oracle's two float64 solves of the same normal equations: where they agree to 1e-8 dB the bound is ~1e-6 dB, where
conditioning or the cancellation in ‖e‖² - ‖P e‖² (about eps 10^(SAR/10) relative) separates them the bound follows.
A singular G (L + flen - 1 < nsrc flen) sends both oracle routes through the same least-squares solve, so their
disagreement says nothing; there the device's dependent-column rule and the SVD's rank cut-off drop different
rounding-level directions of an ill-conditioned span, and the floor is 1e-5 dB.

Correlation kernel edges (bss.cu): 256-sample shared-memory chunks, 4096-sample time segments, 8 lags per thread and
4 signals per CTA (the last CTA of a set takes 1..4 signals: nsrc + rows covers every remainder below)."""
import numpy as np
import pytest
import torch
from scipy.signal import butter, lfilter

from oracle import bss_np

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def refs_of(rng, nsrc, L, kind):
    x = rng.standard_normal((nsrc, L))
    if kind == "lowpass":     # Gaussian noise through a 4th-order 1 kHz low-pass (16 kHz) plus a -40 dB white floor
        b, a = butter(4, 1000 / 8000)
        x = lfilter(b, a, x, axis=1) + 1e-2 * rng.standard_normal((nsrc, L))
    return x.astype(np.float32)


def ests_of(rng, refs, E, snrs):
    """E estimate sets: a filtered mixture of the references plus white noise at the SNRs `snrs` (cycled)."""
    nsrc, L = refs.shape
    out = np.empty((E, nsrc, L), np.float32)
    for e in range(E):
        mixing = np.eye(nsrc) + 0.05 * rng.standard_normal((nsrc, nsrc))
        mixed = np.stack([lfilter([1.0, 0.3, -0.1], [1.0], m) for m in mixing @ refs.astype(np.float64)])
        snr = snrs[e % len(snrs)]
        noise = rng.standard_normal(mixed.shape) * np.sqrt(np.mean(mixed ** 2)) * 10 ** (-snr / 20)
        out[e] = (mixed + noise).astype(np.float32)
    return out


def oracle(refs, ests, flen, perm):
    """(LU result, SVD result) of the oracle for one estimate set."""
    r, e = refs.astype(np.float64), ests.astype(np.float64)
    return (bss_np.bss_eval_sources(r, e, perm, flen, "lu"), bss_np.bss_eval_sources(r, e, perm, flen, "svd"))


def assert_scores(got, lu, svd, what, floor=1e-6):
    for name, g, a, b in zip(("sdr", "sir", "sar"), got[:3], lu[:3], svd[:3]):
        assert not np.any(np.isnan(g)), (what, name, g)
        big = b > 100          # rounding-level residual energies: both beyond 100 dB (or +inf)
        assert np.all(g[big] > 100), (what, name, g, b)
        with np.errstate(invalid="ignore"):
            dis = np.where(np.isfinite(a) & np.isfinite(b), np.abs(a - b), 0.0)
            err = np.abs(g - b)
        tol = floor + 4 * dis
        assert np.all(err[~big] <= tol[~big]), (what, name, g, b, a)


CASES = [   # nsrc, E, L, flen, kind
    (1, 1, 1000, 512, "white"),
    (1, 3, 257, 64, "lowpass"),
    (2, 1, 4095, 512, "white"),
    (2, 3, 4097, 512, "lowpass"),
    (2, 1, 255, 512, "white"),       # L + flen - 1 < nsrc flen: singular G
    (3, 1, 256, 64, "white"),
    (3, 3, 8193, 512, "lowpass"),
    (4, 1, 1, 16, "white"),          # one sample: every G singular beyond rank 16
    (4, 3, 5000, 512, "white"),
    (4, 1, 300, 512, "lowpass"),     # singular
    # appended estimate rows (E nsrc) spanning 2 and 3 64-row blocks of the factor kernel
    (2, 33, 1000, 64, "white"),
    (2, 66, 700, 64, "white"),
    # nsrc flen around multiples of 64 (the factor's column blocks), flen 1, and M = nsrc (1 + E) at every
    # remainder mod 4 (the last 4-signal CTA of the correlation kernel)
    (1, 1, 500, 1, "white"),
    (4, 1, 2000, 7, "lowpass"),      # 28
    (4, 2, 3000, 9, "white"),        # 36
    (1, 2, 3000, 63, "white"),       # 63, M = 3
    (1, 4, 3000, 65, "lowpass"),     # 65, M = 5
    (2, 1, 3000, 63, "white"),       # 126
    (2, 2, 3000, 65, "lowpass"),     # 130
    (2, 1, 8191, 511, "white"),      # 1022; L one below two 4096-sample segments
    (3, 2, 8192, 65, "lowpass"),     # 195, M = 9; exactly two segments
    (3, 4, 12289, 63, "white"),      # 189, M = 15; one sample into a fourth segment
]


@pytest.mark.parametrize("nsrc,E,L,flen,kind", CASES)
@pytest.mark.parametrize("perm", [True, False])
def test_against_oracle(dev, nsrc, E, L, flen, kind, perm):
    from disco_b200 import bss_eval
    rng = np.random.default_rng(nsrc * 100 + E * 10 + L + flen)
    refs = refs_of(rng, nsrc, L, kind)
    ests = ests_of(rng, refs, E, snrs=(-10.0, 20.0, 60.0))
    got = bss_eval.bss_eval_sources(torch.from_numpy(refs).to(dev), torch.from_numpy(ests).to(dev),
                                    compute_permutation=perm, flen=flen)
    got = [g.cpu().numpy() for g in got]
    for e in range(E):
        lu, svd = oracle(refs, ests[e], flen, perm)
        singular = L + flen - 1 < nsrc * flen
        assert_scores([g[e] for g in got], lu, svd, (nsrc, E, L, flen, kind, e), floor=1e-5 if singular else 1e-6)
        if perm and not singular:
            np.testing.assert_array_equal(got[3][e], svd[3])


def test_full_length_lowpass_high_scores(dev):
    """tango.main's shape (144 000 samples, 2 references) with cond(G) ~ 5e6 and scores up to ~100 dB."""
    from disco_b200 import bss_eval
    rng = np.random.default_rng(11)
    refs = refs_of(rng, 2, 144000, "lowpass")
    ests = ests_of(rng, refs, 3, snrs=(100.0, 40.0, 0.0))
    got = bss_eval.bss_eval_sources(torch.from_numpy(refs).to(dev), torch.from_numpy(ests).to(dev),
                                    compute_permutation=False)
    got = [g.cpu().numpy() for g in got]
    for e in range(3):
        lu, svd = oracle(refs, ests[e], 512, False)
        assert_scores([g[e] for g in got], lu, svd, ("144000", e))


def test_estimate_equal_to_reference(dev):
    from disco_b200 import bss_eval
    rng = np.random.default_rng(5)
    for nsrc in (1, 2, 4):
        refs = refs_of(rng, nsrc, 3000, "white")
        t = torch.from_numpy(refs).to(dev)
        sdr, sir, sar, perm = (x.cpu().numpy() for x in bss_eval.bss_eval_sources(t, t.clone()))
        for x in (sdr, sar) + ((sir,) if nsrc > 1 else ()):
            assert not np.any(np.isnan(x)) and np.all(x >= 100), (nsrc, x)
        np.testing.assert_array_equal(perm, np.arange(nsrc))


def test_batch_position_and_rerun_bit_identical(dev):
    from disco_b200 import ops
    rng = np.random.default_rng(9)
    refs = torch.from_numpy(np.stack([refs_of(rng, 2, 9000, "white") for _ in range(3)])).to(dev)
    ests = torch.from_numpy(np.stack([ests_of(rng, refs[i].cpu().numpy(), 1, (10.0,))[0] for i in range(3)])).to(dev)
    a = ops.bss_eval(refs, ests)
    b = ops.bss_eval(refs[[2, 0]].contiguous(), ests[[2, 0]].contiguous())
    c = ops.bss_eval(refs, ests)
    torch.cuda.synchronize()
    assert torch.equal(a, c)
    assert torch.equal(a[2], b[0]) and torch.equal(a[0], b[1])
    old = ops.BSS_WORKSPACE_CAP
    try:
        ops.BSS_WORKSPACE_CAP = 1          # one set per chunk
        d = ops.bss_eval(refs, ests)
    finally:
        ops.BSS_WORKSPACE_CAP = old
    assert torch.equal(a, d)


def test_poisoned_outputs_and_workspace(dev):
    """Norms inside NaN-patterned guard bands, the workspace filled with NaN: every output word written, no guard word
    changed, no NaN read from unwritten workspace."""
    from disco_b200 import _lib, ops
    SENT = 0x7FF8DEADDEADBEEF
    G = 512
    lib = _lib.load()
    rng = np.random.default_rng(2)
    for nsrc, R, L, flen in ((2, 3, 5000, 512), (3, 2, 300, 64), (1, 5, 4096, 100), (2, 66, 1000, 64)):
        refs = torch.from_numpy(np.stack([refs_of(rng, nsrc, L, "white") for _ in range(2)])).to(dev)
        ests = torch.from_numpy(rng.standard_normal((2, R, L)).astype(np.float32)).to(dev)
        n = 2 * R * (1 + 2 * nsrc)
        buf = torch.full((n + 2 * G,), SENT, dtype=torch.int64, device=dev)
        out = buf[G:G + n].view(torch.float64)
        ws_bytes = lib.disco_bss_eval_workspace(2, nsrc, R, L, flen)
        ws = torch.full((ws_bytes // 8,), float("nan"), dtype=torch.float64, device=dev)
        _lib.check(lib.disco_bss_eval(ops._ptr(refs), ops._ptr(ests), ops._ptr(out), 2, nsrc, R, L, flen,
                                      ops._ptr(ws), ws_bytes, ops._stream()))
        torch.cuda.synchronize()
        assert bool((buf[:G] == SENT).all()) and bool((buf[G + n:] == SENT).all())
        assert int((buf[G:G + n] == SENT).sum()) == 0
        assert not bool(torch.isnan(out).any())
        want = ops.bss_eval(refs, ests, flen=flen).reshape(-1)
        assert torch.equal(out, want)


def exact_normal_equations(refs, ests, flen):
    """G = AᵀA and D = Aᵀe of the delayed references, assembled from correctly rounded correlations
    Q[i][s][k] = Σ_t x_s(t) r_i(t - k) (math.fsum of float64 products of float32 inputs, each exact)."""
    import math
    r, e = refs.astype(np.float64), ests.astype(np.float64)
    nsrc, L = r.shape
    n = nsrc * flen
    corr = lambda x, y, k: math.fsum(x[k:] * y[:L - k]) if k < L else 0.0
    Q = {(i, j, k): corr(r[j], r[i], k) for i in range(nsrc) for j in range(nsrc) for k in range(flen)}
    G = np.empty((n, n))
    for i in range(nsrc):
        for j in range(nsrc):
            for a in range(flen):
                for b in range(flen):
                    G[i * flen + a, j * flen + b] = Q[i, j, a - b] if a >= b else Q[j, i, b - a]
    D = np.array([[corr(e[q], r[j], b) for q in range(len(e))] for j in range(nsrc) for b in range(flen)])
    ee = np.array([math.fsum(x * x) for x in e])
    return G, D, ee


@pytest.mark.parametrize("nsrc,R,flen,L", [(1, 3, 64, 700), (2, 4, 64, 1400), (3, 2, 32, 1000), (4, 2, 16, 700)])
def test_norms_against_float64_cholesky(dev, nsrc, R, flen, L):
    """The raw norms of ops.bss_eval, entry-wise, against float64 Cholesky of the exactly assembled G and D, for
    white references (L >= 10 nsrc flen, so G is well conditioned).

    ‖e‖²: a sum of L positive terms, |Δ| <= L 2⁻⁵³ ‖e‖².  Block norms ‖y_b‖², y = L_G⁻¹ D: the device's correlations
    perturb G and D by at most L 2⁻⁵³ |A|ᵀ|A| and L 2⁻⁵³ |A|ᵀ|e| (n = nsrc flen columns, ‖|A|‖ <= √n ‖A‖), and the
    Cholesky with its appended rows is backward stable with (n + 1) 2⁻⁵³ n ‖G‖, so with η = (L + n + 1) n 2⁻⁵³ each
    side errs by at most (η κ(G) + 2 η √(n κ(G))) ‖e‖² <= 3 η κ(G) ‖e‖² (‖y‖ <= ‖e‖); device and host together:
    |Δ‖y_b‖²| <= 6 η κ(G) ‖e‖².  The dB comparison above cannot see this: its 1e-6 dB floor is ~2e-7 relative."""
    import scipy.linalg
    from disco_b200 import ops
    rng = np.random.default_rng(nsrc * 1000 + R)
    n = nsrc * flen
    assert L >= 10 * n
    refs = refs_of(rng, nsrc, L, "white")
    ests = np.concatenate([ests_of(rng, refs, 1, (10.0,))[0], rng.standard_normal((R - nsrc, L)).astype(np.float32)]
                          if R > nsrc else [ests_of(rng, refs, 1, (10.0,))[0][:R]])
    got = ops.bss_eval(torch.from_numpy(refs[None]).to(dev), torch.from_numpy(ests[None]).to(dev), flen=flen)
    got = got[0].cpu().numpy()                                           # [R, 1 + 2 nsrc]
    G, D, ee = exact_normal_equations(refs, ests, flen)
    kappa = np.linalg.cond(G)
    eta = (L + n + 1) * n * 2.0 ** -53
    tol = 6 * eta * kappa * ee
    np.testing.assert_array_less(np.abs(got[:, 0] - ee), L * 2.0 ** -53 * ee + 1e-300)
    y = scipy.linalg.solve_triangular(np.linalg.cholesky(G), D, lower=True)            # [n, R]
    for b in range(nsrc):
        blk = (y[b * flen:(b + 1) * flen] ** 2).sum(0)
        assert np.all(np.abs(got[:, 1 + b] - blk) <= tol), (b, got[:, 1 + b], blk, tol)
        sl = slice(b * flen, (b + 1) * flen)
        ys = scipy.linalg.solve_triangular(np.linalg.cholesky(G[sl, sl]), D[sl], lower=True)
        single = (ys ** 2).sum(0)
        assert np.all(np.abs(got[:, 1 + nsrc + b] - single) <= tol), (b, got[:, 1 + nsrc + b], single, tol)
    # negative control: an error of 100 times the bound in one block norm is caught
    assert not np.all(np.abs(got[:, 1] + 100 * tol - (y[:flen] ** 2).sum(0)) <= tol)


def test_tango_scores_against_numpy_loop(dev):
    """post.tango_scores on synth utterances through tango_batched against a NumPy loop restating tango.py:541-593
    with the oracle (fw_snr / fw_sd through the same post functions, one node at a time)."""
    from disco_b200 import post
    from disco_b200.synth import make_batch
    from disco_b200.tango import tango_batched
    fs, L = 16000, 3 * 16000
    B, K, C = 2, 2, 2
    y, s, n = make_batch(B, K, C, L, seed0=31)
    rng = np.random.default_rng(4)
    s_dry = (0.1 * rng.standard_normal((B, L + 100))).astype(np.float32)
    n_dry = (0.05 * rng.standard_normal((B, L + 100))).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = tango_batched(T(y), T(s), T(n))
    times = post.to_time(out, L)
    res, resz = post.tango_scores(T(y[:, :, 0]), T(s[:, :, 0]), T(n[:, :, 0]), T(s_dry), T(n_dry), times, fs)
    tn = {k: v.cpu().numpy() for k, v in times.items()}
    for b in range(B):
        for k in range(K):
            min_len = min(L, tn["yf"].shape[-1], s_dry.shape[1], n_dry.shape[1])
            cut = lambda x: x[fs:min_len]
            sh, szh, yk = cut(tn["yf"][b, k]), cut(tn["z_y"][b, k]), cut(y[b, k, 0])
            refs_dry = np.vstack((cut(s_dry[b]), cut(n_dry[b])))
            refs = np.vstack((cut(s[b, k, 0]), cut(n[b, k, 0])))
            ests = np.vstack((sh, yk - sh))
            ests_z = np.vstack((szh, yk - szh))
            ests_i = np.vstack((yk, yk - sh))
            for rs, es, keys, d in ((refs_dry, ests, ("sdr_dry", "sir_dry", "sar_dry"), res),
                                    (refs_dry, ests_z, ("sdr_dry", "sir_dry", "sar_dry"), resz),
                                    (refs_dry, ests_i, ("sdr_in_dry", "sir_in_dry", "sar_in_dry"), res),
                                    (refs, ests, ("sdr_cnv", "sir_cnv", "sar_cnv"), res),
                                    (refs, ests_z, ("sdr_cnv", "sir_cnv", "sar_cnv"), resz),
                                    (refs, ests_i, ("sdr_in_cnv", "sir_in_cnv"), res)):
                lu, svd = oracle(rs, es, 512, False)
                for i, key in enumerate(keys):
                    g, a_, b_ = d[key][b, k].item(), lu[i][0], svd[i][0]
                    if b_ > 100:
                        assert g > 100, (b, k, key, g, b_)
                    else:
                        assert abs(g - b_) <= 1e-6 + 4 * abs(a_ - b_), (b, k, key, g, b_, a_)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
            want = {
                "snr_out": post.fw_snr(t(cut(tn["sf"][b, k])), t(cut(tn["nf"][b, k])), fs)[1],
                "snr_in_cnv": post.fw_snr(t(refs[0]), t(refs[1]), fs)[1],
                "snr_in_dry": post.fw_snr(t(refs_dry[0]), t(refs_dry[1]), fs)[1],
                "fw_sd_cnv": post.fw_sd(t(cut(tn["sf"][b, k])), t(refs[0]), fs)[1],
                "fw_sd_dry": post.fw_sd(t(cut(tn["sf"][b, k])), t(refs_dry[0]), fs)[1],
            }
            for key, w in want.items():
                assert abs(res[key][b, k].item() - w.item()) <= 1e-9 * max(1.0, abs(w.item())), key
            assert abs(resz["snr_out"][b, k].item() -
                       post.fw_snr(t(cut(tn["z_s"][b, k])), t(cut(tn["z_n"][b, k])), fs)[1].item()) <= 1e-9
    assert "delta_stoi" not in res and "snr_in_raw" not in res
