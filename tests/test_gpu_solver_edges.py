"""The per-bin MWF solve (`mwf_solve_kernel`: the register solver for D <= 4, the cooperative one for D = 5..16) on
ill-conditioned, singular, tied, indefinite and extreme-scale bins, against oracle/solve_f64.py.

Every input is built in float64 and rounded to complex64; the truth is the oracle evaluated on those complex64
matrices upcast, so the rounding of the input is not an error source."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import rel_l2
from oracle import solve_f64
from test_gpu_solver_instances import ALL_D, mpb

pytestmark = pytest.mark.gpu

DS = list(ALL_D)        # every instantiation of both engines (tests/test_gpu_solver_instances.py INSTANCES)
EPS64 = np.finfo(np.float64).eps
FILTERS = [("gevd", 1, 1.0), ("gevd", 2, 2.5), ("gevd", "full", 1.0), ("r1-mwf", 1, 2.5), ("mwf", 1, 1.0)]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _c64(a):
    return np.ascontiguousarray(a, dtype=np.complex64)


def _c64h(R):
    """Exactly Hermitian complex64 (real diagonal, conjugate mirrors)."""
    R = 0.5 * (R + R.conj().swapaxes(-1, -2))
    return _c64(R)


def _unitary(rng, n, D):
    z = rng.standard_normal((n, D, D)) + 1j * rng.standard_normal((n, D, D))
    q, r = np.linalg.qr(z)
    return q * (np.diagonal(r, axis1=-2, axis2=-1) / np.abs(np.diagonal(r, axis1=-2, axis2=-1)))[:, None, :]


def _hpd(rng, n, D, r):
    a = rng.standard_normal((n, D, r)) + 1j * rng.standard_normal((n, D, r))
    return a @ a.conj().transpose(0, 2, 1) / r


def _solve(dev, Rss, Rnn, typ, rank, mu):
    from disco_b200 import ops
    W, T1 = ops.mwf_solve(torch.from_numpy(_c64(Rss)).to(dev), torch.from_numpy(_c64(Rnn)).to(dev), mu, typ, rank)
    return W.cpu().numpy(), T1.cpu().numpy()


def _truth(Rss, Rnn, typ, rank, mu):
    return solve_f64.solve(_c64(Rss).astype(np.complex128), _c64(Rnn).astype(np.complex128), mu, typ, rank)


def _rank(rank, D):
    return min(rank, D) if isinstance(rank, int) else rank


def _cond_family(rng, n, D, cond):
    """Rnn = U diag(sigma) U^H with sigma log-spaced from 1 to 1/cond; Rss = strong rank-1 plus diffuse."""
    sig = np.logspace(0, -np.log10(cond), D) if D > 1 else np.ones(1)
    U = _unitary(rng, n, D)
    Rnn = (U * sig[None, None, :]) @ U.conj().transpose(0, 2, 1)
    Rss = 10 * _hpd(rng, n, D, 1) + 0.1 * _hpd(rng, n, D, D + 2)
    return Rss, Rnn


def _err_bound(cond, gap, D):
    """Bar for the float32 output of a float64 solve: 2e-6 (float32 output rounding plus the squaring's stopping
    rule), plus the float64 forward bound kappa * eps64 / gap with a 10 D constant for the D-term sums, plus
    kappa * 1e-13 for the Jacobi paths: their sweeps stop at an off-diagonal energy of 1e-26 of the total, i.e.
    eigenvectors accurate to ~1e-13, which the whitening q = L^-H v amplifies by up to kappa(Rnn)."""
    return 2e-6 + 10 * D * cond * EPS64 / gap + cond * 1e-13


def _cond_draws(seeds):
    """(generator, cond) for cond = 1 ... 1e10 under each seed, one generator per seed drawn in that order."""
    for seed in seeds:
        rng = np.random.default_rng(seed)
        for cond in (1e0, 1e2, 1e4, 1e6, 1e8, 1e10):
            yield rng, cond


@pytest.mark.parametrize("D", DS)
def test_conditioning(dev, D):
    """cond(Rnn) = 1 ... 1e10 as constructed.  Rounding to complex64 perturbs Rnn by ~6e-8 of its norm, so from
    cond ~1e7 on the matrix the solver sees has its own (larger, or no) condition number: the forward check takes
    only the bins whose complex64 Rnn keeps lambda_min >= 1e-10 tr (far above the 1e-13 pivot floor), with
    kappa of those matrices in the bound, and requires every other bin to be finite.  Two draws per D: 'full' also
    sums the small eigenpairs of the whitened matrix, whose norm reaches 1e9 here, so it checks that the Jacobi sweeps
    resolve them relative to their own size (at D = 11 and 15 they did not before the per-pair stopping rule)."""
    for rng, cond in _cond_draws((100 + D, 1700 + D)):
        Rss, Rnn = _cond_family(rng, 48, D, cond)
        Rss, Rnn = _c64h(Rss), _c64h(Rnn)
        ev = np.linalg.eigvalsh(Rnn.astype(complex))
        ok = ev[:, 0] >= 1e-10 * ev.sum(axis=1)
        if cond <= 1e6:
            assert np.all(ok)
        kappa = float(np.max(ev[ok, -1] / ev[ok, 0])) if ok.any() else 1.0
        for typ, rank, mu in FILTERS:
            rank = _rank(rank, D)
            W, T1 = _solve(dev, Rss, Rnn, typ, rank, mu)
            assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1)), (cond, typ, rank)
            if not ok.any():
                continue
            w, t1 = _truth(Rss[ok], Rnn[ok], typ, rank, mu)
            gap = 1.0
            if typ == "gevd" and rank != "full" and rank < D:
                lam = solve_f64.gevd(Rss[ok].astype(complex), Rnn[ok].astype(complex), mu, rank)[2]
                gap = float(np.min((lam[:, rank - 1] - lam[:, rank]) / lam[:, 0]))
            tol = 2e-6 if cond <= 1e6 else _err_bound(kappa, gap, D)
            assert rel_l2(W[ok], w) <= tol, (cond, typ, rank, rel_l2(W[ok], w), tol)
            if typ == "gevd":
                assert rel_l2(T1[ok], t1) <= tol, (cond, typ, rank, rel_l2(T1[ok], t1), tol)


@pytest.mark.parametrize("D", DS)
def test_small_pivot_is_used_as_is(dev, D):
    """A Cholesky pivot of 1.2e-10 tr(Rnn), a thousand times above the 1e-13 tr / D floor, is used as it is:
    Rnn = diag(1, ..., 1, p) with p exact in complex64, generic Rss.  'full' is left out: its Jacobi sweeps stop
    relative to ||A|| ~ 1 / p, so the small eigenpairs it also sums carry an error no tight bar covers."""
    rng = np.random.default_rng(1000 + D)
    n = 16
    p = float(np.float32(1.2e-10 * D))
    Rnn = np.broadcast_to(np.diag(np.r_[np.ones(D - 1), p]), (n, D, D)).astype(complex)
    Rss = _c64h(10 * _hpd(rng, n, D, 1) + 0.1 * _hpd(rng, n, D, D + 2))
    kappa = 1.0 / p
    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        if rank == "full":
            continue
        W, T1 = _solve(dev, Rss, Rnn, typ, rank, mu)
        w, t1 = _truth(Rss, Rnn, typ, rank, mu)
        gap = 1.0
        if typ == "gevd" and rank < D:
            lam = solve_f64.gevd(Rss.astype(complex), Rnn, mu, rank)[2]
            gap = float(np.min((lam[:, rank - 1] - lam[:, rank]) / lam[:, 0]))
        tol = _err_bound(kappa, gap, D)
        assert np.all(np.isfinite(W)) and rel_l2(W, w) <= tol, (typ, rank, rel_l2(W, w), tol)


def _gap_family(rng, n, D, delta):
    """Whitened pencil with lambda_1 / lambda_2 = 1 + delta: Rss = L A L^H, A = V diag(lam) V^H, Rnn = L L^H."""
    lam = np.concatenate([[2.0 * (1 + delta), 2.0], np.linspace(1.0, 0.1, max(D - 2, 0))])[:D]
    V = _unitary(rng, n, D)
    A = (V * lam[None, None, :]) @ V.conj().transpose(0, 2, 1)
    Lc = np.linalg.cholesky(_hpd(rng, n, D, D + 4))
    return Lc @ A @ Lc.conj().transpose(0, 2, 1), Lc @ Lc.conj().transpose(0, 2, 1)


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_eigen_gap(dev, D):
    """Forward error against the oracle for relative gaps down to 1e-7 (above the complex64 rounding of the input,
    so the gap survives it); the squaring needs ~log2(40 / delta) steps, within its 40-step cap."""
    rng = np.random.default_rng(200 + D)
    for delta in (1e-1, 1e-3, 1e-5, 1e-7):
        Rss, Rnn = _gap_family(rng, 32, D, delta)
        Rss, Rnn = _c64h(Rss), _c64h(Rnn)
        lam = solve_f64.gevd(_c64(Rss).astype(complex), _c64(Rnn).astype(complex))[2]
        gap = float(np.min((lam[:, 0] - lam[:, 1]) / lam[:, 0]))
        cond = float(np.max(np.linalg.cond(_c64(Rnn).astype(complex))))
        for rank, mu in ((1, 1.0), (1, 2.5), (2, 1.0)):
            W, T1 = _solve(dev, Rss, Rnn, "gevd", rank, mu)
            w, t1 = _truth(Rss, Rnn, "gevd", rank, mu)
            tol = _err_bound(cond, gap if rank == 1 else 1.0, D)
            assert rel_l2(W, w) <= tol, (delta, rank, mu, rel_l2(W, w), tol)
            assert rel_l2(T1, t1) <= _err_bound(cond, gap, D), (delta, rank, mu, rel_l2(T1, t1))


def _backward_check(Rss, Rnn, W, T1, mu, tol):
    """t1 ~ q and g = w / t1 = lam / (lam + mu): the pair (lam, t1) must satisfy Rss t1 = lam Rnn t1 and lam must be
    the largest generalised eigenvalue."""
    Rs, Rn = _c64(Rss).astype(complex), _c64(Rnn).astype(complex)
    lmax = np.linalg.eigvalsh(np.linalg.solve(np.linalg.cholesky(Rn), Rs) @
                              np.linalg.inv(np.linalg.cholesky(Rn)).conj().transpose(0, 2, 1))[:, -1]
    W, T1 = W.astype(complex), T1.astype(complex)
    # a top eigenspace orthogonal to e_0 makes every valid choice give (Rnn q)[0] = 0, so w = t1 = 0
    zero = np.all(T1 == 0, axis=1)
    assert np.all(W[zero] == 0)
    Rs, Rn, lmax, W, T1 = Rs[~zero], Rn[~zero], lmax[~zero], W[~zero], T1[~zero]
    k = np.argmax(np.abs(T1), axis=1)
    g = np.real(W[np.arange(len(k)), k] / T1[np.arange(len(k)), k])
    lam = g * mu / (1 - g)
    res = np.einsum("nij,nj->ni", Rs, T1) - lam[:, None] * np.einsum("nij,nj->ni", Rn, T1)
    scale = np.linalg.norm(Rs, axis=(1, 2)) * np.linalg.norm(T1, axis=1)
    assert np.all(np.linalg.norm(res, axis=1) <= tol * np.maximum(scale, 1e-30)), np.max(np.linalg.norm(res, axis=1) / scale)
    assert np.all(lam >= lmax * (1 - tol)), np.min(lam / lmax)


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_ties_and_tiny_gaps(dev, D):
    """Exact ties (any vector of the top eigenspace is right) and a relative gap of 2^-39, which the 40-step
    squaring cap cannot resolve: judged by backward error.  The inputs are exact in complex64: Rnn = 4 I, Rss
    diagonal with the tie at the front, at the back or behind a smaller entry, or a [[1, e], [e, 1]] block with
    e = 2^-40 on channels 0 and 1."""
    n = 4
    Rss = np.zeros((n, D, D), complex)
    base = np.linspace(1.0, 0.25, D)
    Rss[0] = np.diag(np.r_[2.0, 2.0, base[2:]])                      # tie at the front
    Rss[1] = np.diag(np.r_[base[2:], 2.0, 2.0][:D] if D > 2 else [2.0, 2.0])   # tie at the back
    Rss[2] = np.diag(np.r_[0.5, 2.0, 2.0, base[3:]][:D])              # tie behind a smaller entry
    e = 2.0 ** -40
    Rss[3] = np.diag(np.r_[1.0, 1.0, np.linspace(0.5, 0.25, D)[2:]])
    Rss[3, 0, 1], Rss[3, 1, 0] = e * (1 + 1j), e * (1 - 1j)
    Rnn = np.broadcast_to(4.0 * np.eye(D), (n, D, D)).copy()
    for mu in (1.0, 2.5):
        W, T1 = _solve(dev, Rss, Rnn, "gevd", 1, mu)
        assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1))
        _backward_check(Rss, Rnn, W, T1, mu, 2e-6 * (1 + 2.0 / mu) * D)


def _embed(R, D, d):
    keep = [i for i in range(D) if i != d]
    out = np.zeros(R.shape[:-2] + (D, D), R.dtype)
    out[..., np.ix_(keep, keep)[0], np.ix_(keep, keep)[1]] = R
    return out


@pytest.mark.parametrize("D", DS)
def test_dead_microphone(dev, D):
    """Row and column d of both matrices zero: W is the (D-1)-microphone solve with a zero tap at d; d = 0 (the
    reference microphone) gives W = 0."""
    rng = np.random.default_rng(300 + D)
    if D == 1:
        for typ, rank, mu in FILTERS:
            W, T1 = _solve(dev, np.zeros((4, 1, 1)), np.zeros((4, 1, 1)), typ, rank, mu)
            assert np.all(W == 0) and np.all(np.isfinite(T1)), typ
        return
    Rss, Rnn = _cond_family(rng, 32, D - 1, 1e2)
    Rss, Rnn = _c64h(Rss), _c64h(Rnn)
    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        for d in sorted({0, D // 2, D - 1}):
            W, T1 = _solve(dev, _embed(Rss, D, d), _embed(Rnn, D, d), typ, rank, mu)
            assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1)), (typ, rank, d)
            if d == 0:
                assert np.all(W == 0), (typ, rank)
                continue
            if typ == "r1-mwf":
                continue        # solves with the singular Rnn itself: finiteness only (DESIGN.md section 2)
            Ws, _ = _solve(dev, Rss, Rnn, typ, _rank(rank, D - 1), mu)
            assert np.all(W[:, d] == 0), (typ, rank, d)
            assert rel_l2(np.delete(W, d, axis=1), Ws) <= 1e-6, (typ, rank, d, rel_l2(np.delete(W, d, axis=1), Ws))


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_duplicated_microphone(dev, D):
    """Channel D-1 is an exact copy of channel 0 in both matrices.  Only w_0 + w_{D-1} acts on the signal, so the
    comparison with the oracle collapses the two taps."""
    rng = np.random.default_rng(400 + D)
    Rss, Rnn = _cond_family(rng, 32, D - 1, 1e2)
    idx = list(range(D - 1)) + [0]
    Rss = _c64h(Rss)[:, idx][:, :, idx]
    Rnn = _c64h(Rnn)[:, idx][:, :, idx]

    def collapse(w):
        c = w[:, :D - 1].astype(complex).copy()
        c[:, 0] += w[:, D - 1]
        return c

    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        W, T1 = _solve(dev, Rss, Rnn, typ, rank, mu)
        assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1)), (typ, rank)
        if (typ, rank) in (("gevd", 1), ("mwf", 1)):
            w, _ = _truth(Rss, Rnn, typ, rank, mu)
            assert rel_l2(collapse(W), collapse(w)) <= 1e-5, (typ, rel_l2(collapse(W), collapse(w)))


@pytest.mark.parametrize("D", DS)
def test_singular_statistics(dev, D):
    """Bins of binary masks.  Rnn == 0 (mask 1 in every frame): the gevd filter is exactly 0, 'mwf' and 'r1-mwf'
    agree with the oracle (r1-mwf tends to v conj(v_0) as Rnn -> 0).  Rss == 0 (mask 0 in every frame): lambda
    clamps to eps, so w = eps / (eps + mu) t1 for rank 1.  Rnn = c e_k e_k^H (rank one, exact zero pivots):
    agrees with the oracle."""
    rng = np.random.default_rng(500 + D)
    Rss, Rnn = _cond_family(rng, 16, D, 1e2)
    Rss, Rnn = _c64h(Rss), _c64h(Rnn)
    Z = np.zeros_like(Rss)
    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        W, T1 = _solve(dev, Rss, Z, typ, rank, mu)
        assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1)), (typ, rank)
        if typ == "gevd":
            assert np.all(W == 0) and np.all(T1 == 0), (typ, rank)
        else:
            assert rel_l2(W, _truth(Rss, Z, typ, rank, mu)[0]) <= 2e-6, (typ, rel_l2(W, _truth(Rss, Z, typ, rank, mu)[0]))
        W, T1 = _solve(dev, Z, Rnn, typ, rank, mu)
        assert np.all(np.isfinite(W)) and np.all(np.isfinite(T1)), (typ, rank)
        if typ == "mwf":
            assert np.all(W == 0)
        elif typ == "gevd" and rank == 1:
            assert np.allclose(W, EPS64 / (EPS64 + mu) * T1, rtol=1e-6, atol=1e-45)
        elif typ == "gevd":
            assert np.max(np.abs(W)) <= 1e3 * D * EPS64     # every lambda clamps to eps: of order eps
    for k in sorted({0, D - 1}):
        R1 = np.zeros_like(Rnn)
        R1[:, k, k] = 0.75
        for typ, rank, mu in (("gevd", 1, 1.0), ("gevd", 1, 2.5), ("mwf", 1, 1.0)):
            W, T1 = _solve(dev, Rss, R1, typ, rank, mu)
            w, t1 = _truth(Rss, R1, typ, rank, mu)
            assert np.all(np.isfinite(W)) and rel_l2(W, w) <= 2e-6, (k, typ, mu, rel_l2(W, w))


def _all_families(D):
    """Every family above (and a generic rank-one Rnn) in one complex64 batch."""
    rng = np.random.default_rng(600 + D)
    parts = [_cond_family(rng, 8, D, c) for c in (1.0, 1e4, 1e8)]
    if D > 1:
        parts.append(_gap_family(rng, 8, D, 1e-5))
        Rs, Rn = _cond_family(rng, 4, D - 1, 1e2)
        parts.append((_embed(Rs, D, D // 2), _embed(Rn, D, D // 2)))
        parts.append((_embed(Rs, D, 0), _embed(Rn, D, 0)))
        idx = list(range(D - 1)) + [0]
        parts.append((_c64h(Rs)[:, idx][:, :, idx], _c64h(Rn)[:, idx][:, :, idx]))
        diag = np.zeros((1, D, D), complex)
        diag[0] = np.diag(np.r_[2.0, 2.0, np.linspace(1.0, 0.25, D)[2:]])
        parts.append((diag, np.eye(D)[None] * 4.0))
    Rs, Rn = _cond_family(rng, 4, D, 1e2)
    a = rng.standard_normal((4, D, 1)) + 1j * rng.standard_normal((4, D, 1))
    parts += [(Rs, np.zeros_like(Rn)), (np.zeros_like(Rs), Rn), (Rs, a @ a.conj().transpose(0, 2, 1)),
              (np.zeros_like(Rs), np.zeros_like(Rn))]
    return _c64h(np.concatenate([p[0] for p in parts])), _c64h(np.concatenate([p[1] for p in parts]))


@pytest.mark.parametrize("D", DS)
def test_scale(dev, D):
    """Every family times 2^e: finite, and W, t1 bit-identical across e (all three formulas are invariant under a
    common scale, and a power-of-two scale of complex64 input is exact)."""
    from disco_b200 import ops
    Rss, Rnn = _all_families(D)
    Rs0, Rn0 = torch.from_numpy(Rss).to(dev), torch.from_numpy(Rnn).to(dev)
    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        W0, T0 = ops.mwf_solve(Rs0, Rn0, mu, typ, rank)
        for e in (-60, -40, -20, 15, 30, 40, 60):
            s = 2.0 ** e
            assert np.array_equal(_c64(Rss * s) / s, Rss)                  # exact in complex64
            W, T = ops.mwf_solve(Rs0 * s, Rn0 * s, mu, typ, rank)
            assert bool(torch.isfinite(torch.view_as_real(W)).all()), (typ, rank, e)
            assert torch.equal(W, W0) and torch.equal(T, T0), (typ, rank, e)
        assert bool(torch.isfinite(torch.view_as_real(W0)).all()) and bool(torch.isfinite(torch.view_as_real(T0)).all())


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_scale_zero_diagonal(dev, D):
    """An indefinite Rss with an exactly zero diagonal (so the diagonals alone give no scale), with Rnn == 0 and
    Rnn = I, times 2^e: finite and bit-identical across e for the eigenvalue filters.  ('mwf' needs Rnn + Rss
    positive definite and is left out.)"""
    from disco_b200 import ops
    rng = np.random.default_rng(650 + D)
    R = rng.standard_normal((4, D, D)) + 1j * rng.standard_normal((4, D, D))
    R = R + R.conj().transpose(0, 2, 1)
    R[:, np.arange(D), np.arange(D)] = 0
    Rss = _c64(np.concatenate([R, R]))
    Rnn = _c64(np.concatenate([np.zeros_like(R), np.broadcast_to(np.eye(D), R.shape)]))
    Rs0, Rn0 = torch.from_numpy(Rss).to(dev), torch.from_numpy(Rnn).to(dev)
    for typ, rank, mu in FILTERS:
        if typ == "mwf":
            continue
        rank = _rank(rank, D)
        W0, T0 = ops.mwf_solve(Rs0, Rn0, mu, typ, rank)
        assert bool(torch.isfinite(torch.view_as_real(W0)).all()), (typ, rank)
        for e in (-60, -20, 15, 40, 60):
            W, T = ops.mwf_solve(Rs0 * 2.0 ** e, Rn0 * 2.0 ** e, mu, typ, rank)
            assert torch.equal(W, W0) and torch.equal(T, T0), (typ, rank, e)


@pytest.mark.parametrize("D", [d for d in DS if d > 1])
def test_indefinite_rss(dev, D):
    """Rss whose most negative eigenvalue outweighs the largest positive one, and Rss != 0 with an exactly zero
    diagonal: rank-1 GEVD takes the largest SIGNED eigenvalue, so it is the first term of rank 2, and agrees with
    the oracle; compat.intern_filter agrees with the reference's algorithm on complex128 input."""
    from disco_b200.compat.internal_formulas import intern_filter
    from oracle import tango_np
    rng = np.random.default_rng(700 + D)
    n = 16
    lam = np.r_[1.0, -3.0, np.linspace(0.5, 0.1, D - 2)] if D > 2 else np.array([1.0, -3.0])
    V = _unitary(rng, n, D)
    Lc = np.linalg.cholesky(_hpd(rng, n, D, D + 4))
    Rss_a = Lc @ ((V * lam[None, None, :]) @ V.conj().transpose(0, 2, 1)) @ Lc.conj().transpose(0, 2, 1)
    Rnn_a = Lc @ Lc.conj().transpose(0, 2, 1)
    Rss_b = rng.standard_normal((n, D, D)) + 1j * rng.standard_normal((n, D, D))
    Rss_b = Rss_b + Rss_b.conj().transpose(0, 2, 1)
    Rss_b[:, np.arange(D), np.arange(D)] = 0
    Rnn_b = np.broadcast_to(np.diag(2.0 ** np.arange(D) / 2 ** D), (n, D, D)).copy()
    for Rss, Rnn in ((Rss_a, Rnn_a), (Rss_b, Rnn_b)):
        Rss, Rnn = _c64h(Rss), _c64h(Rnn)
        R64s, R64n = Rss.astype(complex), Rnn.astype(complex)
        cond = float(np.max(np.linalg.cond(R64n)))
        Li = np.linalg.inv(np.linalg.cholesky(R64n))
        lam = np.linalg.eigvalsh(Li @ R64s @ Li.conj().transpose(0, 2, 1))[:, ::-1]
        assert np.all(-lam[:, -1] > lam[:, 0]) or np.all(np.trace(Rss, axis1=1, axis2=2) == 0)
        gap = float(np.min((lam[:, 0] - lam[:, 1]) / np.max(np.abs(lam), axis=1)))
        for mu in (1.0, 2.5):
            W1, T1 = _solve(dev, Rss, Rnn, "gevd", 1, mu)
            W2, T2 = _solve(dev, Rss, Rnn, "gevd", 2, mu)
            w1, t1 = _truth(Rss, Rnn, "gevd", 1, mu)
            tol = _err_bound(cond, gap, D)
            assert rel_l2(T1, T2) <= tol, (mu, rel_l2(T1, T2), tol)
            assert rel_l2(W1, w1) <= tol and rel_l2(T1, t1) <= tol, (mu, rel_l2(W1, w1), rel_l2(T1, t1), tol)
        # 'mwf' is left out: Rnn + Rss is indefinite here, which the Cholesky-based solve does not cover
        for b in range(3):
            for typ, rank in (("gevd", 1), ("gevd", 2), ("gevd", "full"), ("r1-mwf", None)):
                kw = {} if rank is None else {"rank": rank}
                W, (t, _) = intern_filter(R64s[b], R64n[b], mu=1.5, type=typ, **kw)
                Wr, (tr, _) = tango_np.intern_filter(R64s[b], R64n[b], mu=1.5, type=typ, **kw)
                assert rel_l2(W, Wr) <= 1e-5, (b, typ, rank, rel_l2(W, Wr))
                if typ == "gevd":
                    assert rel_l2(t, tr) <= 1e-5, (b, typ, rank)


@pytest.mark.parametrize("D", DS)
def test_non_hermitian_input_is_symmetrised(dev, D):
    """R = H + K with K anti-Hermitian and small-integer entries (every sum exact): W(R) == W(H) bit for bit."""
    rng = np.random.default_rng(800 + D)
    n = 24

    def ints(*s):
        return rng.integers(-3, 4, s) + 1j * rng.integers(-3, 4, s)

    Bs, Bn = ints(n, D, 2), ints(n, D, D + 2)
    Hs, Hn = Bs @ Bs.conj().transpose(0, 2, 1), Bn @ Bn.conj().transpose(0, 2, 1) + 4 * np.eye(D)
    Ks, Kn = ints(n, D, D), ints(n, D, D)
    Ks, Kn = Ks - Ks.conj().transpose(0, 2, 1), Kn - Kn.conj().transpose(0, 2, 1)
    for typ, rank, mu in FILTERS:
        rank = _rank(rank, D)
        Wh, Th = _solve(dev, Hs, Hn, typ, rank, mu)
        Wr, Tr = _solve(dev, Hs + Ks, Hn + Kn, typ, rank, mu)
        assert np.array_equal(Wh, Wr) and np.array_equal(Th, Tr), (typ, rank)


@pytest.mark.parametrize("D", DS)
def test_batch_tails(dev, D):
    """disco_mwf_solve with W / T1 longer than n_mat * D and filled with a sentinel: the tail stays untouched,
    n_mat = 0 is a no-op, and the solved part equals the solve of exactly those matrices."""
    from disco_b200 import _lib, ops
    lib = _lib.load()
    mpb_ = mpb(D)
    rng = np.random.default_rng(900 + D)
    many = 3 * mpb_ + 5
    Rss, Rnn = _cond_family(rng, many, D, 1e2)
    Rs, Rn = torch.from_numpy(_c64(Rss)).to(dev), torch.from_numpy(_c64(Rnn)).to(dev)
    ref_W, ref_T = ops.mwf_solve(Rs, Rn, 1.0, "gevd", 1)
    sentinel = torch.view_as_complex(torch.full((many * D + 3 * D, 2), float.fromhex("0x1.5p-7"), device=dev))
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    for n_mat in sorted({0, 1, mpb_ - 1, mpb_, mpb_ + 1, many}):
        if n_mat == 0 and mpb_ == 1:
            continue
        W, T = sentinel.clone(), sentinel.clone()
        assert lib.disco_mwf_solve(ptr(Rs), ptr(Rn), ptr(W), ptr(T), n_mat, D, 0, 1, ctypes.c_double(1.0), stream) == 0
        torch.cuda.synchronize()
        assert torch.equal(W[n_mat * D:], sentinel[n_mat * D:]) and torch.equal(T[n_mat * D:], sentinel[n_mat * D:]), n_mat
        if n_mat:
            assert torch.equal(W[:n_mat * D], ref_W[:n_mat].reshape(-1)), n_mat
            assert torch.equal(T[:n_mat * D], ref_T[:n_mat].reshape(-1)), n_mat
