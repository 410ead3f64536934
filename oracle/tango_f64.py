"""Vectorised float64 evaluation of the reference's MWF mathematics — TEST INFRASTRUCTURE.

Same algorithm as oracle/tango_np.py (reference tango.py:252-457 and
internal_formulas.py:31-81) but evaluated in complex128 with whole-array contractions
and a Cholesky-whitened Hermitian eigen-solve instead of LAPACK ggev.  It serves as
"truth" when budgeting the fp32 error of both the reference and the CUDA path
(SURVEY.md §6: the reference itself sits 1e-7 .. 5e-6 rel-L2 from this), and as the
fast CPU baseline ("vectorised port") next to the loop-faithful one.

The rank-r GEVD-MWF closed form used here (SURVEY.md §8a-5, verified against
intern_filter to 2e-16): with (lambda_i, q_i) the generalised eigenpairs of
(Rss, Rnn), q_i^H Rnn q_i = 1, eigenvalues clamped to [eps, 1e6] and sorted descending,

    w  = sum_{i<r} q_i * lambda_i / (lambda_i + mu) * conj((Rnn q_i)[0])
    t1 = q_0 * conj((Rnn q_0)[0])
"""
import sys

import numpy as np

from oracle import librosa_np

EPS = sys.float_info.epsilon
ETA = 1e6


def masked_scm(X, m):
    """X (D,F,T) complex, m (F,T) real -> Rss, Rnn (F,D,D): mean_t (m x)(m x)^H, ((1-m) x)(...)^H."""
    X = X.astype(np.complex128)
    m = np.asarray(m, np.float64)
    a, b = m * m, (1 - m) * (1 - m)
    T = X.shape[-1]
    Rss = np.einsum("ft,ift,jft->fij", a, X, X.conj()) / T
    Rnn = np.einsum("ft,ift,jft->fij", b, X, X.conj()) / T
    return Rss, Rnn


def scm(A):
    """A (D,F,T) -> (F,D,D): mean_t a a^H."""
    A = A.astype(np.complex128)
    return np.einsum("ift,jft->fij", A, A.conj()) / A.shape[-1]


def gevd_filter(Rss, Rnn, mu=1.0, rank=1, loading=1e-12):
    """Batched rank-r GEVD-MWF: Rss, Rnn (F,D,D) -> w (F,D), t1 (F,D), lam (F,D) descending."""
    D = Rss.shape[-1]
    Rnn = 0.5 * (Rnn + Rnn.conj().swapaxes(-1, -2))
    Rss = 0.5 * (Rss + Rss.conj().swapaxes(-1, -2))
    tr = np.real(np.trace(Rnn, axis1=-2, axis2=-1)) / D
    Rl = Rnn + (loading * tr + 1e-300)[:, None, None] * np.eye(D)
    L = np.linalg.cholesky(Rl)
    Li = np.linalg.inv(L)
    A = Li @ Rss @ Li.conj().swapaxes(-1, -2)
    A = 0.5 * (A + A.conj().swapaxes(-1, -2))
    lam, V = np.linalg.eigh(A)
    lam, V = lam[:, ::-1], V[:, :, ::-1]
    Q = Li.conj().swapaxes(-1, -2) @ V                       # Rnn-orthonormal
    lam = np.clip(lam, EPS, ETA)
    g = lam / (lam + mu)
    if rank not in ("full", "Full"):
        g[:, rank:] = 0
    c = np.conj((Rnn @ Q)[:, 0, :])                          # conj((Rnn q_i)[0]) per i
    w = np.einsum("fdi,fi->fd", Q, g * c)
    t1 = Q[:, :, 0] * c[:, 0:1]
    return w, t1, lam


def mwf_filter(Rss, Rnn):
    """internal_formulas.py:74-76: first column of (Rnn + Rss)^-1 Rss."""
    return np.linalg.solve(Rnn + Rss, Rss)[:, :, 0]


def r1_mwf_filter(Rss, Rnn, mu=1.0):
    """internal_formulas.py:45-54 in closed form (SURVEY.md §8a-5)."""
    lam, V = np.linalg.eigh(0.5 * (Rss + Rss.conj().swapaxes(-1, -2)))
    l, v = np.abs(lam[:, -1]), V[:, :, -1]
    u = np.linalg.solve(Rnn, v[:, :, None])[:, :, 0]
    den = mu + l * np.einsum("fd,fd->f", v.conj(), u)
    return (l / den)[:, None] * u * np.conj(v[:, 0:1])


def solve(Rss, Rnn, mu=1.0, filter_type="gevd", rank=1):
    if filter_type == "gevd":
        return gevd_filter(Rss, Rnn, mu, rank)[0]
    if filter_type == "mwf":
        return mwf_filter(Rss, Rnn)
    if filter_type == "r1-mwf":
        return r1_mwf_filter(Rss, Rnn, mu)
    raise AttributeError("Unknown filter reference")


def filter_sum(w, X):
    """w (F,D), X (D,F,T) -> (F,T): w^H x."""
    return np.einsum("fd,dft->ft", w.conj(), X.astype(np.complex128))


def irm(s, n, power=1):
    xi = (np.abs(s) / np.maximum(np.abs(n), EPS)) ** power
    return xi / (1 + xi)


def stft64(x, n_fft=512, hop=256):
    return librosa_np.stft(np.asarray(x, np.float64), n_fft, hop, dtype=np.complex128)


def offline_tango(y, s=None, n=None, masks=None, n_fft=512, n_hop=256, mu=1.0,
                  filter_type="gevd", rank=1, mask_for_z="local", mask_power=1, solve=solve, ref_mic=0):
    """Two-step Tango in float64.  y (K,C,L).  Either (s, n) for oracle irm masks or
    masks=(mask_z (K,F,T), mask_w (K,F,T)).  `solve(Rss, Rnn, mu, filter_type, rank) -> w` is the per-bin
    filter (e.g. the solver-policy oracle of oracle/solve_f64.py).  Returns dict of (K,F,T) arrays.

    ref_mic: the reference microphone of every node.  Its oracle mask is the step-1 mask of all the node's
    channels and zn = Y[ref_mic] - z_y; the step-2 oracle mask is that of microphone 0 (as oracle/tango_np.py
    states it; the reference itself fails for ref_mic != 0, see DESIGN §2).  The filters still estimate the
    speech at microphone 0 (intern_filter's e_0 selector)."""
    y = np.asarray(y)
    K, C, _ = y.shape
    Y = np.array([[stft64(c, n_fft, n_hop) for c in y[k]] for k in range(K)])
    have_sn = s is not None
    if have_sn:
        S = np.array([[stft64(c, n_fft, n_hop) for c in s[k]] for k in range(K)])
        N = np.array([[stft64(c, n_fft, n_hop) for c in n[k]] for k in range(K)])
    if masks is None:
        mz = np.array([irm(S[k, ref_mic], N[k, ref_mic], mask_power) for k in range(K)])
        mw = mz if ref_mic == 0 else np.array([irm(S[k, 0], N[k, 0], mask_power) for k in range(K)])
    else:
        mz, mw = np.asarray(masks[0], np.float64), np.asarray(masks[1], np.float64)
    out = {}
    z_y = np.empty(Y.shape[:1] + Y.shape[2:], np.complex128)
    z_s, z_n = np.empty_like(z_y), np.empty_like(z_y)
    for k in range(K):
        Rss, Rnn = masked_scm(Y[k], mz[k])
        w = solve(Rss, Rnn, mu, filter_type, rank)
        z_y[k] = filter_sum(w, Y[k])
        if have_sn:
            z_s[k], z_n[k] = filter_sum(w, S[k]), filter_sum(w, N[k])
    yf, sf, nf = np.empty_like(z_y), np.empty_like(z_y), np.empty_like(z_y)
    for k in range(K):
        others = [j for j in range(K) if j != k]
        X = np.concatenate([Y[k], z_y[others]], axis=0)
        if mask_for_z == "local":
            Rss, Rnn = masked_scm(X, mw[k])
        elif mask_for_z == "distant":
            a = np.concatenate([mw[k][None] * Y[k], mw[others] * z_y[others]], axis=0)
            b = np.concatenate([(1 - mw[k])[None] * Y[k], (1 - mw[others]) * z_y[others]], axis=0)
            Rss, Rnn = scm(a), scm(b)
        else:
            raise NotImplementedError(mask_for_z)
        w = solve(Rss, Rnn, mu, filter_type, rank)
        yf[k] = filter_sum(w, X)
        if have_sn:
            sf[k] = filter_sum(w, np.concatenate([S[k], z_s[others]], axis=0))
            nf[k] = filter_sum(w, np.concatenate([N[k], z_n[others]], axis=0))
    out.update(yf=yf, z_y=z_y, zn=Y[:, ref_mic] - z_y, masks_z=mz, mask_w=mw, Y=Y)
    if have_sn:
        out.update(sf=sf, nf=nf, z_s=z_s, z_n=z_n)
    return out
