"""Every instantiation of the per-bin MWF solve against float64, matrix by matrix, in every warp and block slot,
through the C ABI (`disco_mwf_solve`) with W and T1 inside NaN-patterned guard bands.

Dispatch targets (INSTANCES below; tests/test_solver_instances_cpu.py parses the dispatch sets and the geometry out
of the sources and requires this table and `geometry` to match them exactly):
  solve_small  solve_small.cu  mwf_solve_kernel<D, 1, false>, D = 1..4: one thread per matrix, 64-thread CTAs.
               Rank-1 GEVD by repeated squaring (a shifted second pass for indefinite input), ranks > 1 and
               'r1-mwf' by cyclic Jacobi (at most 30 sweeps; squaring at most 40 steps per pass, 2 passes).
  solve        solve.cu        mwf_solve_kernel<D>, D = 5..16: a group of G = 8 (D <= 8) or 16 lanes owns one
               matrix, MPW = 32 / G matrices share a warp, WARPS = 4 (D <= 8) or 2 per CTA, so MPB = 16 or 4
               matrices per CTA.  Rank-1 GEVD by squaring (at most 40 steps), falling back to round-robin Jacobi
               (at most 40 sweeps; a dummy player at odd D) when squaring cannot settle.  Lanes l >= D idle; dead
               groups past n_mat mirror the last matrix and store nothing.
Every iteration loop is capped, so a NaN or inf matrix costs at most its caps and cannot hang its neighbours.

Inputs are built in float64 and rounded to complex64 (exactly Hermitian); the truth is oracle/solve_f64.py on those
complex64 matrices upcast, and kappa and the eigengaps of each matrix are computed in float64 from the same rounded
matrices.  So the rounding of the input is not an error source.

Bound, per matrix m (no batch norm: one wrong matrix or one wrong warp slot cannot hide):
    ||W_m - w_m||_2 <= tol_m ||w_m||_2 + 2^-126 sqrt(2 D)
    tol_m = 2^-24 + r_m kappa_m (10 D eps64 + sqrt(D) 1e-13) / gap_m
  * 2^-24: the kernels compute in float64 and round each real component of the result to float32 once, which moves
    every component by at most 2^-24 of itself, so the vector by at most 2^-24 ||w|| (the floor covers components
    below the float32 normal range).
  * 10 D eps64 / gap: float64 rounding of the D-term sums (Cholesky, whitening, squaring or rotations, back
    substitution), each eigenvector moving by the rounding over its relative eigengap (Davis-Kahan), as in
    test_gpu_solver_edges._err_bound.
  * sqrt(D) 1e-13 / gap: the Jacobi stopping rule.  Sweeps stop no earlier than the off-diagonal energy is below
    1e-26 of the total, i.e. off(A) <= 1e-13 ||A||_F <= 1e-13 sqrt(D) |lambda|_max (the per-pair rule that must hold
    as well only tightens this), which moves each eigenvector by at most that
    over its absolute gap.  (The squaring stops at 1 - ||B||_F^2 <= 1e-14, leaving the other eigenvectors a weight
    below 1e-14 sqrt(D) in the column it takes, which this term covers.)
  * kappa_m = kappa(Rnn) (kappa(Rnn + Rss) for 'mwf'): q = L^-H v amplifies an error of v by at most kappa(L), and
    (Rnn q)[0] = (L v)[0] by kappa(L) again.
  * gap_m: the smallest relative gap (lambda_k - lambda_{k+1}) / |lambda_1| at the boundaries k = 1 .. min(r, D-1)
    of the r eigenpairs the filter sums (every eigenvector it uses is bounded by its two neighbours); for 'r1-mwf'
    the gap of Rss's top eigenvalue; 1 for 'mwf'.  r_m: the number of eigenpairs summed into w (1 for rank 1,
    'r1-mwf', 'mwf' and t1).
The families keep kappa <= 80 and every gap >= 1e-2, so tol_m stays below 1e-7: the float32 rounding of the output
plus a few 1e-8 at D = 16, full rank.  These are bounds, not fits; a neighbour's matrix, a wrong rank, a conjugate or
the second eigenpair are O(1) errors.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import solve_f64
from test_gpu_kernel_instances import GUARD, SENTINEL, Guarded

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
EPS64 = np.finfo(np.float64).eps
INSTANCES = {"solve_small": (1, 2, 3, 4), "solve": tuple(range(5, 17))}
ALL_D = INSTANCES["solve_small"] + INSTANCES["solve"]
SMALL_THREADS = 64                       # solve_small.cu: launch_d's block size, one matrix per thread
TYPES = {"gevd": 0, "r1-mwf": 1, "mwf": 2}
MUS = (0.0, 1.0, 2.5, 1e5)
KAPPA_MAX, GAP_MIN = 80.0, 1e-2


def geometry(D):
    """(G, MPW, WARPS, MPB): lanes per matrix, matrices per warp, warps per CTA, matrices per CTA."""
    if D in INSTANCES["solve_small"]:
        return 1, 32, SMALL_THREADS // 32, SMALL_THREADS
    G = 2 if D <= 2 else (4 if D <= 4 else (8 if D <= 8 else 16))     # solve.cu SolveGeom<D>::G
    warps = 4 if D <= 8 else 2                                        # SolveGeom<D>::WARPS
    return G, 32 // G, warps, (32 // G) * warps


def mpb(D):
    return geometry(D)[3]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


# ---- the C ABI --------------------------------------------------------------------------------------------------

def _launch(Rs, Rn, W, T1, n_mat, D, typ, rank, mu):
    """disco_mwf_solve on device tensors (views: their data pointers are the matrices' starts)."""
    from disco_b200 import _lib, ops
    _lib.check(_lib.load().disco_mwf_solve(ops._ptr(Rs), ops._ptr(Rn), ops._ptr(W), ops._ptr(T1), n_mat, D,
                                           TYPES[typ], rank, float(mu), ops._stream()))


def _solve(dev, Rss, Rnn, typ, rank, mu):
    """W, T1 (complex64 numpy) of the batch, written into guard bands that must come back intact and filled."""
    n, D = Rss.shape[0], Rss.shape[-1]
    g = Guarded(dev)
    W, T1 = g.new((n, D)), g.new((n, D))
    _launch(torch.from_numpy(Rss).to(dev), torch.from_numpy(Rnn).to(dev), W, T1, n, D, typ, rank, mu)
    g.check("%s rank %s mu %g D %d" % (typ, rank, mu, D))
    return W.cpu().numpy(), T1.cpu().numpy()


# ---- inputs -----------------------------------------------------------------------------------------------------

def _c64h(R):
    """Exactly Hermitian complex64 (real diagonal, conjugate mirrors)."""
    return np.ascontiguousarray(0.5 * (R + R.conj().swapaxes(-1, -2)), dtype=np.complex64)


def _up(R):
    return R.astype(np.complex128)


def _unitary(rng, n, D):
    z = rng.standard_normal((n, D, D)) + 1j * rng.standard_normal((n, D, D))
    q, r = np.linalg.qr(z)
    d = np.diagonal(r, axis1=-2, axis2=-1)
    return q * (d / np.abs(d))[:, None, :]


def _herm_from(V, lam):
    return (V * lam[..., None, :]) @ V.conj().swapaxes(-1, -2)


def _geometric(D, top):
    """top, ..., top / 10, geometrically spaced: every relative gap (l_k - l_{k+1}) / l_1 >= 0.1 (10^(1/15) - 1)."""
    return top * 10.0 ** (-np.arange(D) / max(D - 1, 1))


def _scales(rng, n):
    """A factor in [0.5, 1] per matrix, so that no two matrices of a family have the same answer (also at D = 1)."""
    return rng.uniform(0.5, 1.0, (n, 1))


def _rnn(rng, n, D):
    """kappa = 64 as built (log-spaced spectrum 1 .. 1/64 times a per-matrix scale, random eigenvectors)."""
    sig = np.logspace(0, -np.log10(64.0), D) if D > 1 else np.ones(1)
    return _herm_from(_unitary(rng, n, D), _scales(rng, n) * sig)


def fam_spaced(rng, n, D, top=4.0):
    """Whitened pencil with geometric generalised eigenvalues s top .. s top / 10, s in [0.5, 1] per matrix:
    Rss = L V diag(lam) V^H L^H."""
    Rnn = _rnn(rng, n, D)
    L = np.linalg.cholesky(Rnn)
    Rss = L @ _herm_from(_unitary(rng, n, D), _scales(rng, n) * _geometric(D, top)) @ L.conj().swapaxes(-1, -2)
    return _c64h(Rss), _c64h(Rnn)


def fam_clamp(rng, n, D):
    """lambda_1 >= 5e7: every generalised eigenvalue is above the 1e6 clamp, which at mu = 1e5 moves w by ~10 %."""
    return fam_spaced(rng, n, D, top=1e8)


def fam_r1(rng, n, D):
    """Rss = V diag(s 4 .. s 0.4) V^H: its top eigenvalue is separated from the rest by >= 14 %."""
    return _c64h(_herm_from(_unitary(rng, n, D), _scales(rng, n) * _geometric(D, 4.0))), _c64h(_rnn(rng, n, D))


def fam_indefinite(rng, n, D):
    """Rss whose most negative generalised eigenvalue (-3) outweighs the largest positive one (1)."""
    lam = np.r_[1.0, -3.0, np.linspace(0.5, 0.1, max(D - 2, 0))][:D] if D > 1 else np.array([-3.0])
    Rnn = _rnn(rng, n, D)
    L = np.linalg.cholesky(Rnn)
    return _c64h(L @ _herm_from(_unitary(rng, n, D), lam) @ L.conj().swapaxes(-1, -2)), _c64h(Rnn)


def fam_gap(rng, n, D, delta):
    """lambda_1 / lambda_2 = 1 + delta: the squaring runs ~log2(40 / delta) steps (delta = 0: an exact tie, 40)."""
    lam = np.r_[2.0 * (1 + delta), 2.0, np.linspace(1.0, 0.1, max(D - 2, 0))][:D] if D > 1 else np.ones(1)
    return (_c64h(_herm_from(_unitary(rng, n, D), lam)),
            np.ascontiguousarray(np.broadcast_to(4 * np.eye(D), (n, D, D)), dtype=np.complex64))


# ---- per-matrix measures and the bound --------------------------------------------------------------------------

def kappa(R):
    ev = np.linalg.eigvalsh(_up(R))
    return ev[:, -1] / ev[:, 0]


def whitened_eigs(Rss, Rnn):
    """Generalised eigenvalues of the rounded pencil, unclamped, largest signed first."""
    Li = np.linalg.inv(np.linalg.cholesky(_up(Rnn)))
    return np.linalg.eigvalsh(Li @ _up(Rss) @ Li.conj().swapaxes(-1, -2))[:, ::-1]


def rel_gaps(lam, kmax):
    """Smallest (lam_k - lam_{k+1}) / |lam_1| over the boundaries k = 1 .. min(kmax, D - 1); 1 where there is none."""
    D = lam.shape[1]
    kk = min(kmax, D - 1)
    if kk < 1:
        return np.ones(lam.shape[0])
    return np.min(lam[:, :kk] - lam[:, 1:kk + 1], axis=1) / np.max(np.abs(lam), axis=1)


def abi_rank(rank, D):
    """The rank the kernel uses: <= 0 or > D is full."""
    return D if rank <= 0 or rank > D else rank


def tol_of(kap, gap, terms, D):
    return U + terms * kap * (10 * D * EPS64 + math.sqrt(D) * 1e-13) / gap


def floor_of(D):
    return 2.0 ** -126 * math.sqrt(2 * D)


def bound(Rss, Rnn, typ, rank):
    """(tol_m for w, tol_m for t1), one per matrix, from that matrix's own kappa and gaps."""
    D = Rss.shape[-1]
    if typ == "mwf":
        t = tol_of(kappa(_up(Rss) + _up(Rnn)), 1.0, 1, D)
        return t, t
    kap = kappa(Rnn)
    if typ == "r1-mwf":
        t = tol_of(kap, rel_gaps(np.linalg.eigvalsh(_up(Rss))[:, ::-1], 1), 1, D)
        return t, t
    r = abi_rank(rank, D)
    lam = whitened_eigs(Rss, Rnn)
    return tol_of(kap, rel_gaps(lam, r), r, D), tol_of(kap, rel_gaps(lam, 1), 1, D)


def truth(Rss, Rnn, typ, rank, mu):
    D = Rss.shape[-1]
    return solve_f64.solve(_up(Rss), _up(Rnn), mu, typ, abi_rank(rank, D) if typ == "gevd" else 1)


# ---- checkers ---------------------------------------------------------------------------------------------------

def check_forward(W, w, tol, what):
    """Per matrix: ||W_m - w_m|| <= tol_m ||w_m|| + floor.  Returns the largest error as a fraction of its bar."""
    D = w.shape[-1]
    err = np.linalg.norm(W.astype(np.complex128) - w, axis=-1)
    bar = tol * np.linalg.norm(w, axis=-1) + floor_of(D)
    bad = np.flatnonzero(~(err <= bar))
    assert bad.size == 0, "%s: matrices %s: error / bar %s" % (what, bad[:8].tolist(), (err / bar)[bad[:8]].tolist())
    return float(np.max(err / bar))


def check_bits(A, B, what, skip=()):
    """The complex64 arrays (n, D) are identical bit for bit, matrix by matrix, except the matrices in `skip`."""
    a = np.ascontiguousarray(A).view(np.uint32).reshape(A.shape[0], -1)
    b = np.ascontiguousarray(B).view(np.uint32).reshape(B.shape[0], -1)
    diff = np.any(a != b, axis=1)
    diff[list(skip)] = False
    bad = np.flatnonzero(diff)
    assert bad.size == 0, "%s: matrices %s differ" % (what, bad[:8].tolist())


def e0(n, D):
    t = np.zeros((n, D), np.complex64)
    t[:, 0] = 1.0
    return t


def gevd_ranks(D):
    """1, 2, ceil(D / 2), D - 1, D, and 0, D + 3, -1 (full by the ABI), without repeats."""
    return list(dict.fromkeys([1, 2, (D + 1) // 2, D - 1, D, 0, D + 3, -1]))


# ---- a. accuracy of each matrix ---------------------------------------------------------------------------------

@pytest.mark.parametrize("D", ALL_D)
def test_accuracy(dev, D):
    """gevd at every rank class, r1-mwf and mwf, mu in {0, 1, 2.5, 1e5}, on families whose answer is well
    determined, each matrix against float64 within its own bound (module docstring)."""
    rng = np.random.default_rng(1100 + D)
    n = max(40, mpb(D) + 3)
    fams = {"spaced": fam_spaced(rng, n, D), "clamp": fam_clamp(rng, n, D), "r1": fam_r1(rng, n, D)}
    for name, (Rs, Rn) in fams.items():                  # the families are what they claim, after rounding
        assert np.all(kappa(Rn) <= KAPPA_MAX), name
        if name != "r1":
            assert np.all(rel_gaps(whitened_eigs(Rs, Rn), D) >= GAP_MIN), name
        else:
            assert np.all(rel_gaps(np.linalg.eigvalsh(_up(Rs))[:, ::-1], 1) >= GAP_MIN)
    Rs, Rn = fams["clamp"]                               # the clamp is visible at mu = 1e5
    w_clamped = truth(Rs, Rn, "gevd", 1, 1e5)[0]
    eta, solve_f64.ETA = solve_f64.ETA, np.inf
    try:
        w_free = truth(Rs, Rn, "gevd", 1, 1e5)[0]
    finally:
        solve_f64.ETA = eta
    shift = np.linalg.norm(w_clamped - w_free, axis=1) / np.linalg.norm(w_free, axis=1)
    assert np.all(shift > 0.05), float(np.min(shift))
    worst = 0.0
    plan = [("gevd", r, ("spaced", "clamp")) for r in gevd_ranks(D)] + \
           [("r1-mwf", 1, ("r1",)), ("mwf", 1, ("spaced", "clamp", "r1"))]
    for typ, rank, names in plan:
        Rs = np.concatenate([fams[k][0] for k in names])
        Rn = np.concatenate([fams[k][1] for k in names])
        tol_w, tol_t = bound(Rs, Rn, typ, rank)
        assert np.max(tol_w) <= 1e-7 and np.max(tol_t) <= 1e-7, (typ, rank, np.max(tol_w))
        for mu in MUS:
            W, T1 = _solve(dev, Rs, Rn, typ, rank, mu)
            w, t1 = truth(Rs, Rn, typ, rank, mu)
            what = "D %d %s rank %d mu %g" % (D, typ, rank, mu)
            worst = max(worst, check_forward(W, w, tol_w, what))
            if typ == "gevd":
                worst = max(worst, check_forward(T1, t1, tol_t, what + " t1"))
            else:
                check_bits(T1, e0(len(T1), D), what + " t1 = e0")
    print("solver accuracy D=%d: largest per-matrix error / bound = %.3f" % (D, worst))


# ---- b. checks that need no oracle ------------------------------------------------------------------------------

@pytest.mark.parametrize("D", ALL_D)
def test_identities(dev, D):
    """gevd at full rank with mu = 0 is e_0 (Q Q^H Rnn = I, and lambda / lambda = 1 whatever the clamp); 'mwf'
    solves (Rnn + Rss) w = Rss e_0 to the float32 rounding of w; rank-1 gevd passes the backward check: t1 is a
    generalised eigenvector of the largest signed eigenvalue and w / t1 = lambda / (lambda + mu)."""
    from test_gpu_solver_edges import _backward_check
    rng = np.random.default_rng(1200 + D)
    n = max(40, mpb(D) + 3)
    Rs, Rn = fam_spaced(rng, n, D)
    Ri, Rni = fam_indefinite(rng, n, D)
    for rank in (0, D, -1):
        W, _ = _solve(dev, Rs, Rn, "gevd", rank, 0.0)
        check_forward(W, e0(n, D).astype(np.complex128), tol_of(kappa(Rn), 1.0, D, D), "D %d full, mu 0" % D)
    # ||(Rnn + Rss) W - Rss e_0|| <= ||M|| (||W - w~|| + ||E|| ||w~||): 2^-24 (1 + 2^-20) for the output rounding,
    # 10 D eps64 for the float64 Cholesky solve's backward error E, 10 D eps64 for evaluating the residual here
    c = U * (1 + 2.0 ** -20) + 20 * D * EPS64
    for Rss, Rnn in ((Rs, Rn), fam_r1(rng, n, D)):
        M = _up(Rss) + _up(Rnn)
        W, _ = _solve(dev, Rss, Rnn, "mwf", 1, 1.0)
        res = np.linalg.norm(np.einsum("nij,nj->ni", M, _up(W)) - _up(Rss)[:, :, 0], axis=1)
        bar = c * np.linalg.norm(M, axis=(1, 2)) * np.linalg.norm(_up(W), axis=1)
        assert np.all(res <= bar), (D, float(np.max(res / bar)))
    # D = 1 has no positive generalised eigenvalue in the indefinite family: lambda clamps to eps there
    pairs = ((Rs, Rn), (Ri, Rni)) if D > 1 else ((Rs, Rn),)
    for mu in (1.0, 2.5):
        for Rss, Rnn in pairs:
            W, T1 = _solve(dev, Rss, Rnn, "gevd", 1, mu)
            _backward_check(Rss, Rnn, W, T1, mu, 2e-6 * (1 + 4.0 / mu) * D)


# ---- c. each matrix's result depends only on that matrix -------------------------------------------------------

MIX_FILTERS = (("gevd", 1, 1.0), ("gevd", 2, 2.5), ("gevd", 0, 1.0), ("r1-mwf", 1, 2.5), ("mwf", 1, 1.0))


def mixed_batch(rng, D):
    """3 MPB + 5 matrices cycling through seven kinds that take different branches -- generic PSD (squaring),
    indefinite Rss dominated by its negative eigenvalue (the Jacobi fallback / the shifted pass), Rss == 0,
    Rnn == 0, both == 0, a 1e-5 gap (a long squaring), an exact tie (the squaring's 40-step cap) -- with one NaN
    and one inf matrix.  Returns Rss, Rnn, the kind of each matrix and the indices of the non-finite ones."""
    n = 3 * mpb(D) + 5
    kinds = [fam_spaced(rng, n, D), fam_indefinite(rng, n, D), None, None, None,
             fam_gap(rng, n, D, 1e-5), fam_gap(rng, n, D, 0.0)]
    base_s, base_n = fam_r1(rng, n, D)
    Rss, Rnn = base_s.copy(), base_n.copy()
    for m in range(n):
        k = m % len(kinds)
        if kinds[k] is not None:
            Rss[m], Rnn[m] = kinds[k][0][m], kinds[k][1][m]
        elif k == 2:
            Rss[m] = 0
        elif k == 3:
            Rnn[m] = 0
        else:
            Rss[m], Rnn[m] = 0, 0
    bad = (n // 2, n // 2 + 3)
    Rss[bad[0]] = np.nan
    Rnn[bad[1], 0, 0] = np.inf
    return Rss, Rnn, np.arange(n) % len(kinds), bad


@pytest.mark.parametrize("D", ALL_D)
def test_slot_independence(dev, D):
    """The mixed batch under every shift 0 .. MPB - 1 (filler matrices prepended) and each matrix alone
    (n_mat = 1): every finite matrix's W and T1 are the same bits in all these runs."""
    rng = np.random.default_rng(1300 + D)
    P = mpb(D)
    Rss, Rnn, kind, bad = mixed_batch(rng, D)
    n = Rss.shape[0]
    fill_s, fill_n = fam_r1(rng, P - 1, D)
    Rs_all = torch.from_numpy(np.concatenate([fill_s, Rss])).to(dev)
    Rn_all = torch.from_numpy(np.concatenate([fill_n, Rnn])).to(dev)
    Rs, Rn = Rs_all[P - 1:], Rn_all[P - 1:]
    for typ, rank, mu in MIX_FILTERS:
        what = "D %d %s rank %d" % (D, typ, rank)
        W0 = torch.empty((n, D), dtype=torch.complex64, device=dev)
        T0 = torch.empty_like(W0)
        _launch(Rs, Rn, W0, T0, n, D, typ, rank, mu)
        runs = []
        for s in range(P):
            W = torch.empty((s + n, D), dtype=torch.complex64, device=dev)
            T = torch.empty_like(W)
            _launch(Rs_all[P - 1 - s:], Rn_all[P - 1 - s:], W, T, s + n, D, typ, rank, mu)
            runs.append(("shift %d" % s, W[s:], T[s:]))
        Wa, Ta = torch.empty_like(W0), torch.empty_like(T0)
        for m in range(n):
            _launch(Rs[m:], Rn[m:], Wa[m:], Ta[m:], 1, D, typ, rank, mu)
        runs.append(("alone", Wa, Ta))
        torch.cuda.synchronize()
        W0, T0 = W0.cpu().numpy(), T0.cpu().numpy()
        ok = np.ones(n, bool)
        ok[list(bad)] = False
        if typ == "mwf":
            ok &= kind != 1          # Rnn + Rss indefinite: outside what the Cholesky-based 'mwf' covers
        assert np.all(np.isfinite(W0[ok])) and np.all(np.isfinite(T0[ok])), what
        for name, W, T in runs:
            check_bits(W.cpu().numpy(), W0, what + " " + name + " W", skip=bad)
            check_bits(T.cpu().numpy(), T0, what + " " + name + " T1", skip=bad)


# ---- d. tails, guards and reads past the end --------------------------------------------------------------------

def tail_counts(D):
    G, mpw, _, P = geometry(D)
    return sorted({1, max(1, mpw - 1), mpw, mpw + 1, P - 1, P, P + 1, 3 * P + 1})


@pytest.mark.parametrize("D", ALL_D)
def test_tails(dev, D):
    """n_mat at the warp and CTA edges: every word of W and T1 is written and no guard word changes; T1 = nullptr
    gives the same W; NaN matrices past n_mat in the input allocations change nothing."""
    rng = np.random.default_rng(1400 + D)
    P = mpb(D)
    Rss, Rnn = fam_r1(rng, 3 * P + 1, D)
    pad = np.full((P + 3, D, D), np.nan, np.complex64)
    for n_mat in tail_counts(D):
        Rs = torch.from_numpy(np.ascontiguousarray(Rss[:n_mat])).to(dev)
        Rn = torch.from_numpy(np.ascontiguousarray(Rnn[:n_mat])).to(dev)
        Rs_p = torch.from_numpy(np.concatenate([Rss[:n_mat], pad])).to(dev)
        Rn_p = torch.from_numpy(np.concatenate([Rnn[:n_mat], pad])).to(dev)
        for typ, rank, mu in MIX_FILTERS:
            what = "D %d n_mat %d %s rank %d" % (D, n_mat, typ, rank)
            g = Guarded(dev)
            W, T = g.new((n_mat, D)), g.new((n_mat, D))
            _launch(Rs, Rn, W, T, n_mat, D, typ, rank, mu)
            g.check(what)
            W, T = W.cpu().numpy(), T.cpu().numpy()
            assert np.all(np.isfinite(W)) and np.all(np.isfinite(T)), what
            g = Guarded(dev)
            Wn = g.new((n_mat, D))
            _launch(Rs, Rn, Wn, None, n_mat, D, typ, rank, mu)
            g.check(what + " T1 = nullptr")
            check_bits(Wn.cpu().numpy(), W, what + " T1 = nullptr")
            g = Guarded(dev)
            Wp, Tp = g.new((n_mat, D)), g.new((n_mat, D))
            _launch(Rs_p, Rn_p, Wp, Tp, n_mat, D, typ, rank, mu)
            g.check(what + " NaN past n_mat")
            check_bits(Wp.cpu().numpy(), W, what + " NaN past n_mat W")
            check_bits(Tp.cpu().numpy(), T, what + " NaN past n_mat T1")


# ---- e. each checker rejects a result that is only slightly wrong -----------------------------------------------

def _rejects(fn, *args):
    with pytest.raises(AssertionError):
        fn(*args)


@pytest.mark.parametrize("D", ALL_D)
def test_checkers_reject_near_misses(dev, D):
    """A neighbour's W in one slot, the rank r - 1 answer at rank r, conj(W), t1 from the second eigenpair, one
    entry moved by 1e-6 ||w||, one stray word in a guard band, one ulp in the slot check: each is caught."""
    rng = np.random.default_rng(1500 + D)
    n = max(8, mpb(D) + 1)
    Rs, Rn = fam_spaced(rng, n, D)
    r = min(2, D)
    tol_w, tol_t = bound(Rs, Rn, "gevd", r)
    W, T1 = _solve(dev, Rs, Rn, "gevd", r, 1.0)
    w, t1, _, Q = solve_f64.gevd(_up(Rs), _up(Rn), 1.0, r)
    check_forward(W, w, tol_w, "right answer")
    check_forward(T1, t1, tol_t, "right t1")
    k = n - 1 if D < 5 else geometry(D)[1] - 1              # the last group of the first warp
    nb = W.copy()
    nb[k] = W[k - 1]
    _rejects(check_forward, nb, w, tol_w, "neighbour")
    if D > 1:
        Wr, _ = _solve(dev, Rs, Rn, "gevd", r - 1, 1.0)
        _rejects(check_forward, Wr, w, tol_w, "rank r - 1")
        Rs2, Rn2 = solve_f64.prepare(_up(Rs), _up(Rn))
        c1 = np.conj(np.einsum("nj,nj->n", Rn2[:, 0, :], Q[:, :, 1]))
        _rejects(check_forward, (Q[:, :, 1] * c1[:, None]).astype(np.complex64), t1, tol_t, "second eigenpair")
        _rejects(check_forward, np.conj(W), w, tol_w, "conj")
    moved = W.astype(np.complex128)
    moved[k, D - 1] += 1e-6 * np.linalg.norm(w[k])
    _rejects(check_forward, moved.astype(np.complex64), w, tol_w, "one entry by 1e-6")
    g = Guarded(dev)
    out = g.new((n, D))
    out.copy_(torch.from_numpy(W).to(dev))
    g.bufs[0][0].view(torch.int32)[GUARD + 2 * n * D] = SENTINEL + 1    # the first word past the end
    _rejects(g.check, "stray word")
    one_ulp = W.copy()
    one_ulp.view(np.uint32).reshape(n, -1)[k, 0] ^= 1
    _rejects(check_bits, one_ulp, W, "one ulp")
