"""Float64 NumPy restatement of BSS-eval's source scores (mir_eval.separation.bss_eval_sources, the algorithm of
Vincent, Gribonval and Fevotte, "Performance measurement in blind audio source separation", IEEE TASLP 2006, as
mir_eval publishes it), written from that description:

  * Gram matrix of the references delayed by 0 .. flen-1 samples and their correlation with the estimate, both by FFT;
  * filter coefficients by np.linalg.solve, falling back to np.linalg.lstsq when the solve raises (solver='lu'), or by
    SVD least squares throughout (solver='svd');
  * the projection by FFT filtering, the distortion components as differences of projections, energies in dB with a
    zero denominator giving +inf;
  * optionally the permutation with the largest mean SIR.

`brute_force` is the definition itself for small sizes: the explicit delayed-copy matrix A and an SVD least-squares
projection.  `gram_norms` is the route the device kernels take (‖P e‖² = ‖y‖², L y = D, G = L L^T), for the identity
checks.
"""
import itertools

import numpy as np
import scipy.linalg
from scipy.signal import fftconvolve


def _safe_db(num, den):
    if den == 0:
        return np.inf
    return 10 * np.log10(num / den)


def gram(refs, est, flen):
    """G = A^T A [nsrc flen, nsrc flen] and D = A^T e [nsrc flen] by FFT (exact up to rounding: the FFT length covers
    the full linear correlation)."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    est = np.asarray(est, dtype=np.float64)
    nsrc, L = refs.shape
    n_fft = int(2 ** np.ceil(np.log2(L + flen - 1.0)))
    sf = np.fft.fft(refs, n=n_fft, axis=1)
    sef = np.fft.fft(est, n=n_fft)
    G = np.zeros((nsrc * flen, nsrc * flen))
    for i in range(nsrc):
        for j in range(i, nsrc):
            ssf = np.real(np.fft.ifft(sf[i] * np.conj(sf[j])))
            blk = scipy.linalg.toeplitz(np.hstack((ssf[0], ssf[-1:-flen:-1])), r=ssf[:flen])
            G[i * flen:(i + 1) * flen, j * flen:(j + 1) * flen] = blk
            G[j * flen:(j + 1) * flen, i * flen:(i + 1) * flen] = blk.T
    D = np.zeros(nsrc * flen)
    for i in range(nsrc):
        ssef = np.real(np.fft.ifft(sf[i] * np.conj(sef)))
        D[i * flen:(i + 1) * flen] = np.hstack((ssef[0], ssef[-1:-flen:-1]))
    return G, D


def _solve(G, D, solver):
    if solver == "svd":
        return np.linalg.lstsq(G, D, rcond=None)[0]
    try:
        return np.linalg.solve(G, D)
    except np.linalg.LinAlgError:
        return np.linalg.lstsq(G, D, rcond=None)[0]


def project(refs, est, flen, solver="lu"):
    """Least-squares projection of the zero-padded estimate onto the delayed references, [L + flen - 1]."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    nsrc, L = refs.shape
    G, D = gram(refs, est, flen)
    C = _solve(G, D, solver).reshape(flen, nsrc, order="F")
    sproj = np.zeros(L + flen - 1)
    for i in range(nsrc):
        sproj += fftconvolve(C[:, i], refs[i])[:L + flen - 1]
    return sproj


def decompose(refs, est, j, flen, solver="lu"):
    """s_true, e_spat, e_interf, e_artif of estimate `est` against reference j."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    est = np.asarray(est, dtype=np.float64)
    L = est.size
    s_true = np.hstack((refs[j], np.zeros(flen - 1)))
    e_spat = project(refs[j:j + 1], est, flen, solver) - s_true
    e_interf = project(refs, est, flen, solver) - s_true - e_spat
    e_artif = -s_true - e_spat - e_interf
    e_artif[:L] += est
    return s_true, e_spat, e_interf, e_artif


def source_crit(s_true, e_spat, e_interf, e_artif):
    s_filt = s_true + e_spat
    sdr = _safe_db(np.sum(s_filt ** 2), np.sum((e_interf + e_artif) ** 2))
    sir = _safe_db(np.sum(s_filt ** 2), np.sum(e_interf ** 2))
    sar = _safe_db(np.sum((s_filt + e_interf) ** 2), np.sum(e_artif ** 2))
    return sdr, sir, sar


def _select(sdr, sir, sar, nsrc, compute_permutation):
    if not compute_permutation:
        d = np.arange(nsrc)
        return sdr[d, d], sir[d, d], sar[d, d], d
    perms = list(itertools.permutations(range(nsrc)))
    dum = np.arange(nsrc)
    mean_sir = np.array([np.mean(sir[list(p), dum]) for p in perms])
    popt = perms[int(np.argmax(mean_sir))]
    idx = (list(popt), dum)
    return sdr[idx], sir[idx], sar[idx], np.asarray(popt)


def bss_eval_sources(refs, ests, compute_permutation=True, flen=512, solver="lu"):
    """(nsrc, L) references and estimates -> sdr, sir, sar, perm (mir_eval's outputs)."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    ests = np.atleast_2d(np.asarray(ests, dtype=np.float64))
    nsrc = refs.shape[0]
    sdr, sir, sar = (np.full((nsrc, nsrc), np.nan) for _ in range(3))
    pairs = [(j, k) for j in range(nsrc) for k in range(nsrc)] if compute_permutation else [(j, j) for j in range(nsrc)]
    for j, k in pairs:
        sdr[j, k], sir[j, k], sar[j, k] = source_crit(*decompose(refs, ests[j], k, flen, solver))
    return _select(sdr, sir, sar, nsrc, compute_permutation)


def delay_matrix(refs, flen, cols=None):
    """Explicit A [L + flen - 1, |cols| flen]: the references `cols` delayed by 0 .. flen-1, zero-padded."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    nsrc, L = refs.shape
    cols = range(nsrc) if cols is None else cols
    A = np.zeros((L + flen - 1, len(cols) * flen))
    for c, i in enumerate(cols):
        for k in range(flen):
            A[k:k + L, c * flen + k] = refs[i]
    return A


def brute_force(refs, ests, compute_permutation=True, flen=512):
    """The definition: P_S e by SVD least squares on the explicit delay matrix (small L and flen only)."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    ests = np.atleast_2d(np.asarray(ests, dtype=np.float64))
    nsrc, L = refs.shape

    def proj(cols, e):
        A = delay_matrix(refs, flen, cols)
        return A @ np.linalg.lstsq(A, e, rcond=None)[0]

    sdr, sir, sar = (np.full((nsrc, nsrc), np.nan) for _ in range(3))
    pairs = [(j, k) for j in range(nsrc) for k in range(nsrc)] if compute_permutation else [(j, j) for j in range(nsrc)]
    for j, k in pairs:
        e = np.hstack((ests[j], np.zeros(flen - 1)))
        p_k, p_all = proj([k], e), proj(None, e)
        sdr[j, k] = _safe_db(np.sum(p_k ** 2), np.sum((e - p_k) ** 2))
        sir[j, k] = _safe_db(np.sum(p_k ** 2), np.sum((p_all - p_k) ** 2))
        sar[j, k] = _safe_db(np.sum(p_all ** 2), np.sum((e - p_all) ** 2))
    return _select(sdr, sir, sar, nsrc, compute_permutation)


def gram_norms(refs, est, flen, delta=1e-10):
    """The kernels' route in float64: ‖e‖², ‖y_all‖² per reference block and ‖y_k‖² of each reference alone, with
    y = L^-1 D from a Cholesky factor whose pivots <= delta * max diag G drop their column (layout of
    disco_bss_eval's norms row)."""
    refs = np.atleast_2d(np.asarray(refs, dtype=np.float64))
    est = np.asarray(est, dtype=np.float64)
    nsrc = refs.shape[0]
    G, D = gram(refs, est, flen)

    def fwd(Gs, Ds):
        n = Gs.shape[0]
        Lf = np.zeros_like(Gs)
        thr = delta * np.max(np.diag(Gs))
        y = np.zeros(n)
        for j in range(n):
            d = Gs[j, j] - Lf[j, :j] @ Lf[j, :j]
            if not d > thr:
                continue
            Lf[j, j] = np.sqrt(d)
            Lf[j + 1:, j] = (Gs[j + 1:, j] - Lf[j + 1:, :j] @ Lf[j, :j]) / Lf[j, j]
            y[j] = (Ds[j] - Lf[j, :j] @ y[:j]) / Lf[j, j]
        return y

    y_all = fwd(G, D)
    out = [float(est @ est)] + [float(np.sum(y_all[b * flen:(b + 1) * flen] ** 2)) for b in range(nsrc)]
    for k in range(nsrc):
        s = slice(k * flen, (k + 1) * flen)
        out.append(float(np.sum(fwd(G[s, s], D[s]) ** 2)))
    return np.array(out)


def scores_from_norms(norms, nsrc):
    """(sdr, sir [nsrc (reference k)], sar) of one estimate row from its gram_norms / disco_bss_eval norms row."""
    ee, blocks, single = norms[0], norms[1:1 + nsrc], norms[1 + nsrc:1 + 2 * nsrc]
    p_all = blocks.sum()
    db = lambda a, b: 10 * np.log10(a / b) if b > 0 else np.inf
    interf = [blocks[1:].sum() if k == 0 else p_all - single[k] for k in range(nsrc)]
    sdr = np.array([db(single[k], ee - single[k]) for k in range(nsrc)])
    sir = np.array([db(single[k], interf[k]) for k in range(nsrc)])
    return sdr, sir, db(p_all, ee - p_all)
