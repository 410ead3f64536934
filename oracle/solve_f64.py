"""Float64 statement of the per-bin MWF solver's policy (`mwf_solve_kernel`) — TEST INFRASTRUCTURE.

A batched NumPy restatement of what the kernels promise, not a port of how they compute it: the
eigenproblem is solved with LAPACK (`np.linalg.eigh`) instead of repeated squaring or Jacobi, so a
kernel that converges to the wrong eigenpair disagrees with it.  What it shares with the kernels is
the policy for the inputs LAPACK would turn into inf/NaN:

1. Both matrices are Hermitian-symmetrised, (R + R^H) / 2.
2. Both are multiplied by one power of two, 2^-s with 2^s <= t < 2^(s+1), where
   t = max(sum|diag Rss| + sum|diag Rnn|, largest |Re| or |Im| of any entry): the sum for PSD input, the
   maximum for indefinite input with a zero diagonal; no scaling when t is 0.  The scaling is exact, every
   filter below is invariant under a common scale, and inputs that differ by a power of two are solved as
   the same matrices, bit for bit.
3. Cholesky of the (scaled) Rnn -- of Rnn + Rss for 'mwf' -- with every running pivot
   d_j = M_jj - sum_k |L_jk|^2 floored at 1e-13 * tr(M) / D + 1e-300, and the column below a floored
   pivot set to zero.  A singular direction of Rnn (Rnn == 0, a dead or duplicated microphone, a bin
   whose mask is 1 in every frame or 0 in all but one) becomes a direction of tiny, uncoupled noise
   power instead of a division by zero, and the rounding noise of a numerically singular complex64
   Rnn (slightly indefinite) cannot grow from column to column.
4. 'gevd': eigenpairs of the whitened A = L^-1 Rss L^-H, q = L^-H v (so q^H Rnn q = 1 up to the floor),
   eigenvalues clamped to [eps, 1e6], the r LARGEST SIGNED ones taken (descending; the reference's
   argsort order), and
       w  = sum_{i<r} q_i * lambda_i / (lambda_i + mu) * conj((Rnn q_i)[0])
       t1 = q_0 * conj((Rnn q_0)[0]).
   Rnn == 0 gives w = t1 = 0 (row 0 of Rnn is zero); Rss == 0 gives every lambda = eps, so w is of
   order eps.
5. 'r1-mwf': (l, v) = (|lambda|, v) of the largest eigenvalue of Rss, u = Rnn^-1 v through the floored
   factor, w = l u conj(v_0) / (mu + l v^H u); Rnn == 0 gives w ~ v conj(v_0), the limit as Rnn -> 0.
6. 'mwf': w = (Rnn + Rss)^-1 Rss e_0 through the floored factor of Rnn + Rss.
"""
import sys

import numpy as np

EPS = sys.float_info.epsilon      # internal_formulas.py:6
ETA = 1e6                         # internal_formulas.py:7
FLOOR_REL = 1e-13
FLOOR_ABS = 1e-300


def herm(R):
    return 0.5 * (R + np.conj(np.swapaxes(R, -1, -2)))


def _diag_abs_sum(R):
    return np.sum(np.abs(np.real(np.diagonal(R, axis1=-2, axis2=-1))), axis=-1)


def common_scale(Rss, Rnn):
    """The power of two 2^-s the solver multiplies both matrices by (1 where both matrices are 0)."""
    m = np.maximum(np.max(np.maximum(np.abs(Rss.real), np.abs(Rss.imag)), axis=(-2, -1)),
                   np.max(np.maximum(np.abs(Rnn.real), np.abs(Rnn.imag)), axis=(-2, -1)))
    t = np.maximum(_diag_abs_sum(Rss) + _diag_abs_sum(Rnn), m)
    _, e = np.frexp(t)                      # t = m 2^e, m in [0.5, 1): 2^(e-1) <= t < 2^e
    return np.where(t > 0, np.ldexp(1.0, 1 - e), 1.0)


def cholesky_floor(M):
    """Lower Cholesky factor of the Hermitian batch M (n, D, D), running pivots floored at
    1e-13 * tr(M) / D + 1e-300 per matrix."""
    n, D, _ = M.shape
    floor = FLOOR_REL * np.real(np.trace(M, axis1=-2, axis2=-1)) / D + FLOOR_ABS
    L = np.zeros_like(M)
    for j in range(D):
        d = np.real(M[:, j, j]) - np.sum(np.abs(L[:, j, :j]) ** 2, axis=-1)
        lj = np.sqrt(np.maximum(d, floor))
        L[:, j, j] = lj
        s = M[:, j + 1:, j] - np.einsum("nik,nk->ni", L[:, j + 1:, :j], np.conj(L[:, j, :j]))
        L[:, j + 1:, j] = np.where((d >= floor)[:, None], s / lj[:, None], 0.0)
    return L


def _lower_solve(L, B):
    """L^-1 B for lower-triangular L (n, D, D), B (n, D, k)."""
    n, D, _ = L.shape
    X = np.zeros(B.shape, np.complex128)
    for i in range(D):
        X[:, i] = (B[:, i] - np.einsum("nk,nkc->nc", L[:, i, :i], X[:, :i])) / np.real(L[:, i, i])[:, None]
    return X


def _upper_solve_h(L, B):
    """L^-H B for lower-triangular L."""
    n, D, _ = L.shape
    X = np.zeros(B.shape, np.complex128)
    for i in range(D - 1, -1, -1):
        X[:, i] = (B[:, i] - np.einsum("nk,nkc->nc", np.conj(L[:, i + 1:, i]), X[:, i + 1:])) \
            / np.real(L[:, i, i])[:, None]
    return X


def prepare(Rss, Rnn):
    """Steps 1-2: symmetrised, commonly scaled complex128 copies (n, D, D)."""
    Rss = herm(np.asarray(Rss, np.complex128))
    Rnn = herm(np.asarray(Rnn, np.complex128))
    sc = common_scale(Rss, Rnn)[..., None, None]
    return Rss * sc, Rnn * sc


def gevd(Rss, Rnn, mu=1.0, rank=1):
    """Rank-r GEVD-MWF.  Rss, Rnn (n, D, D) -> w, t1 (n, D), lam (n, D) clamped and descending,
    Q (n, D, D) with the matching generalised eigenvectors as columns."""
    Rss, Rnn = prepare(Rss, Rnn)
    D = Rss.shape[-1]
    L = cholesky_floor(Rnn)
    A = herm(_lower_solve(L, np.conj(np.swapaxes(_lower_solve(L, Rss), -1, -2))))   # L^-1 (L^-1 Rss)^H
    m = np.max(np.abs(A), axis=(1, 2))[:, None, None]      # Rnn == 0 puts A near 1e300: keep LAPACK in range
    m = np.where(m > 0, m, 1.0)
    lam, V = np.linalg.eigh(A / m)
    lam = lam * m[:, :, 0]
    order = np.argsort(-lam, axis=-1, kind="stable")          # largest signed first
    lam = np.take_along_axis(lam, order, axis=-1)
    V = np.take_along_axis(V, order[:, None, :], axis=-1)
    Q = _upper_solve_h(L, V)
    lam = np.clip(lam, EPS, ETA)
    g = lam / (lam + mu)
    r = D if rank in ("full", "Full", None, 0) else min(int(rank), D)
    g[:, r:] = 0.0
    c = np.conj(np.einsum("nj,nji->ni", Rnn[:, 0, :], Q))     # conj((Rnn q_i)[0])
    w = np.einsum("ndi,ni->nd", Q, g * c)
    t1 = Q[:, :, 0] * c[:, 0:1]
    return w, t1, lam, Q


def r1_mwf(Rss, Rnn, mu=1.0):
    Rss, Rnn = prepare(Rss, Rnn)
    lam, V = np.linalg.eigh(Rss)
    l, v = np.abs(lam[:, -1]), V[:, :, -1]
    L = cholesky_floor(Rnn)
    u = _upper_solve_h(L, _lower_solve(L, v[:, :, None]))[:, :, 0]
    den = mu + l * np.einsum("nd,nd->n", np.conj(v), u)
    return (l / den)[:, None] * u * np.conj(v[:, 0:1])


def mwf(Rss, Rnn):
    Rss, Rnn = prepare(Rss, Rnn)
    L = cholesky_floor(Rnn + Rss)
    return _upper_solve_h(L, _lower_solve(L, Rss[:, :, 0:1]))[:, :, 0]


def solve(Rss, Rnn, mu=1.0, filter_type="gevd", rank=1):
    """(w, t1) like ops.mwf_solve, for any leading batch shape; t1 = e_0 for 'r1-mwf' and 'mwf'."""
    Rss = np.asarray(Rss)
    D = Rss.shape[-1]
    lead = Rss.shape[:-2]
    Rs, Rn = Rss.reshape(-1, D, D), np.asarray(Rnn).reshape(-1, D, D)
    if filter_type == "gevd":
        w, t1 = gevd(Rs, Rn, mu, rank)[:2]
    elif filter_type in ("r1-mwf", "mwf"):
        w = r1_mwf(Rs, Rn, mu) if filter_type == "r1-mwf" else mwf(Rs, Rn)
        t1 = np.zeros_like(w)
        t1[:, 0] = 1.0
    else:
        raise AttributeError("Unknown filter reference")
    return w.reshape(lead + (D,)), t1.reshape(lead + (D,))
