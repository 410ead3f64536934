"""oracle/solve_f64.py, the float64 statement of the per-bin solver's policy, anchored on the reference's own
answers, on the loaded float64 oracle where its diagonal loading cannot matter, and on hand-checkable cases."""
import numpy as np
import pytest

from conftest import load_golden, rel_l2
from oracle import solve_f64, tango_f64


def _hpd(rng, n, D, r):
    a = rng.standard_normal((n, D, r)) + 1j * rng.standard_normal((n, D, r))
    return a @ a.conj().transpose(0, 2, 1) / r


def test_reference_kats():
    """intern_filter_kat.npz, at the tolerances the GPU solver is held to on the same answers."""
    g = load_golden("intern_filter_kat")
    for i in range(int(g["count"])):
        typ, rank, mu = str(g["cfg_%d" % i]).split("|")
        rank = 1 if rank == "None" else (rank if rank == "full" else int(rank))
        Rxx, Rnn = g["Rxx_%d" % i], g["Rnn_%d" % i]
        w, t1 = solve_f64.solve(Rxx[None], Rnn[None], float(mu), typ, rank)
        tol = 5e-4 if Rxx.dtype == np.complex64 else 1e-5
        assert rel_l2(w[0], g["W_%d" % i]) < tol, (i, typ, rank)
        assert rel_l2(t1[0], g["t1_%d" % i]) < tol, (i, typ, rank)


@pytest.mark.parametrize("D", [1, 2, 4, 7, 16])
def test_matches_loaded_oracle_when_well_conditioned(D):
    """cond(Rnn) ~ 10: the 1e-12 * tr / D loading of tango_f64 moves the answer by ~1e-11."""
    rng = np.random.default_rng(D)
    Rss = 0.1 * _hpd(rng, 50, D, D + 2) + 3 * _hpd(rng, 50, D, 1)
    Rnn = _hpd(rng, 50, D, D + 4)
    for rank, mu in ((1, 1.0), (min(2, D), 2.5), ("full", 1.0)):
        w, t1, lam, _ = solve_f64.gevd(Rss, Rnn, mu, rank)
        wr, tr, lr = tango_f64.gevd_filter(Rss, Rnn, mu, rank)
        assert rel_l2(w, wr) < 1e-9 and rel_l2(t1, tr) < 1e-9 and rel_l2(lam, lr) < 1e-9, rank
    assert rel_l2(solve_f64.mwf(Rss, Rnn), tango_f64.mwf_filter(Rss, Rnn)) < 1e-9
    assert rel_l2(solve_f64.r1_mwf(Rss, Rnn, 1.5), tango_f64.r1_mwf_filter(Rss, Rnn, 1.5)) < 1e-9


def test_d1_closed_form():
    """D = 1: lambda = s / n, w = lambda / (lambda + mu), t1 = 1; mwf = s / (s + n); r1-mwf = s / (mu n + s)."""
    s, n = np.array([[[3.0]], [[0.5]]]), np.array([[[2.0]], [[4.0]]])
    w, t1, lam, _ = solve_f64.gevd(s, n, 2.5, 1)
    lam_x = (s / n)[:, 0, 0]
    assert np.allclose(lam[:, 0], lam_x, rtol=1e-15)
    assert np.allclose(w[:, 0], lam_x / (lam_x + 2.5), rtol=1e-15) and np.allclose(t1, 1.0, rtol=1e-15)
    assert np.allclose(solve_f64.mwf(s, n)[:, 0], (s / (s + n))[:, 0, 0], rtol=1e-15)
    assert np.allclose(solve_f64.r1_mwf(s, n, 2.5)[:, 0], (s / (2.5 * n + s))[:, 0, 0], rtol=1e-15)


def test_identity_noise_is_plain_eigenproblem():
    """Rnn = I: q_i are the eigenvectors of Rss, w = sum g_i q_i conj(q_i[0])."""
    rng = np.random.default_rng(3)
    D = 4
    Rss = _hpd(rng, 1, D, 2)
    lam, V = np.linalg.eigh(Rss[0])
    lam, V = lam[::-1], V[:, ::-1]
    g = np.clip(lam, solve_f64.EPS, solve_f64.ETA)
    g = g / (g + 1.0)
    for rank in (1, 2, "full"):
        r = D if rank == "full" else rank
        want = V[:, :r] @ (g[:r] * np.conj(V[0, :r]))
        w, t1, _, _ = solve_f64.gevd(Rss, np.eye(D)[None], 1.0, rank)
        assert rel_l2(w[0], want) < 1e-13, rank
        assert rel_l2(t1[0], V[:, 0] * np.conj(V[0, 0])) < 1e-13


def test_dead_channel_is_a_zero_tap():
    """Row and column d of both matrices zero: the taps of the other channels are the D - 1 solve, tap d is 0;
    d = 0 (the reference channel) gives w = 0."""
    rng = np.random.default_rng(4)
    D = 5
    Rss = 0.1 * _hpd(rng, 8, D - 1, D + 2) + 3 * _hpd(rng, 8, D - 1, 1)
    Rnn = _hpd(rng, 8, D - 1, D + 4)
    for d in (0, 2, D - 1):
        keep = [i for i in range(D) if i != d]
        Es, En = np.zeros((8, D, D), complex), np.zeros((8, D, D), complex)
        Es[:, np.ix_(keep, keep)[0], np.ix_(keep, keep)[1]] = Rss
        En[:, np.ix_(keep, keep)[0], np.ix_(keep, keep)[1]] = Rnn
        # r1-mwf solves with the singular Rnn itself (u = Rnn^-1 v), so it is only required to stay finite
        assert np.all(np.isfinite(solve_f64.r1_mwf(Es, En, 1.5)))
        for typ, rank in (("gevd", 1), ("gevd", 2), ("gevd", "full"), ("mwf", 1)):
            w, _ = solve_f64.solve(Es, En, 1.5, typ, rank)
            # LAPACK's eigenvectors mix the null direction in at rounding level, eps64, and q = L^-H v amplifies
            # that by 1 / sqrt(floor) ~ 3e6 (the kernels keep the direction exactly 0): 1e-8 is the bound
            assert np.max(np.abs(w[:, d])) <= 1e-8 * np.max(np.abs(w)) or np.all(w == 0), (d, typ, rank)
            if d == 0:
                assert np.all(w == 0), (typ, rank)
            else:
                w_small, _ = solve_f64.solve(Rss, Rnn, 1.5, typ, rank)
                assert rel_l2(w[:, keep], w_small) < 1e-8, (d, typ, rank)


def test_singular_statistics():
    """Rnn == 0 (mask 1 in every frame): w = t1 = 0 exactly.  Rss == 0 (mask 0 in every frame): every eigenvalue
    clamps to eps, so w = eps / (eps + mu) times the rank-1 / full-rank projector, of order eps."""
    rng = np.random.default_rng(5)
    D = 4
    Rss, Rnn = _hpd(rng, 6, D, 3), _hpd(rng, 6, D, D + 2)
    for rank in (1, 2, "full"):
        w, t1, _, _ = solve_f64.gevd(Rss, np.zeros_like(Rnn), 1.0, rank)
        assert np.all(w == 0) and np.all(t1 == 0)
        w, t1, lam, _ = solve_f64.gevd(np.zeros_like(Rss), Rnn, 1.0, rank)
        assert np.all(lam == solve_f64.EPS)
        assert np.all(np.isfinite(w)) and np.max(np.abs(w)) < 10 * solve_f64.EPS * (1 + np.max(np.abs(t1)))
    w, _, _, _ = solve_f64.gevd(np.zeros_like(Rss), Rnn, 1.0, "full")
    assert np.allclose(w, solve_f64.EPS / (1 + solve_f64.EPS) * np.eye(D)[0], atol=1e-25)   # Q Q^H Rnn = I
    assert np.all(np.isfinite(solve_f64.mwf(Rss, np.zeros_like(Rnn))))
    assert np.all(np.isfinite(solve_f64.r1_mwf(Rss, np.zeros_like(Rnn))))


@pytest.mark.parametrize("e", [-60, -20, 0, 30, 60])
def test_scale_invariance(e):
    """A common power-of-two scale changes nothing, bit for bit, singular bins included."""
    rng = np.random.default_rng(6)
    D = 3
    Rss, Rnn = _hpd(rng, 4, D, 1), _hpd(rng, 4, D, D + 1)
    Rnn[0] = 0
    Rss[1] = 0
    for typ, rank in (("gevd", 1), ("gevd", "full"), ("mwf", 1), ("r1-mwf", 1)):
        w0, t0 = solve_f64.solve(Rss, Rnn, 1.0, typ, rank)
        w1, t1 = solve_f64.solve(Rss * 2.0 ** e, Rnn * 2.0 ** e, 1.0, typ, rank)
        assert np.array_equal(w0, w1) and np.array_equal(t0, t1), (typ, rank)


def test_indefinite_takes_largest_signed_eigenvalue():
    """Rss = diag(1, -3), Rnn = I: the rank-1 filter is built on lambda = 1 (e_0), not on the larger |-3|."""
    Rss = np.diag([1.0, -3.0]).astype(complex)[None]
    w, t1, lam, _ = solve_f64.gevd(Rss, np.eye(2)[None], 1.0, 1)
    assert np.allclose(lam[0], [1.0, solve_f64.EPS])
    assert np.allclose(w[0], [0.5, 0.0]) and np.allclose(t1[0], [1.0, 0.0])
