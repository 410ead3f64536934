"""Degenerate bins through the whole pipeline: binary masks (bins whose mask is 1 or 0 in every frame), a dead
microphone, a silent utterance in a batch, and the workspace solve against the matrix solve on such inputs."""
import numpy as np
import pytest
import torch

from conftest import record_parity, rel_l2, rel_l2_mag

pytestmark = pytest.mark.gpu

L = 16000
ONES = (3, 40, 128)        # bins whose step-1 / step-2 mask is 1 in every frame (Rnn == 0 there)
ZEROS = (7, 41, 200)       # ... 0 in every frame (Rss == 0 there)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _inputs(dev, B, K, C, seed):
    """Synthetic utterances with speech pauses and ibm masks of the reference microphone's clean components, with
    some bins forced to 1 or 0 in every frame.  The pauses give every other bin noise-only frames, so Rnn has
    full rank there: a binary mask with fewer noise frames than channels gives a rank-deficient Rnn, which the
    float32 statistics turn into rounding noise the float64 reference does not have (a bin no tolerance can
    compare).  The masks stay informative (Rss is not a multiple of Rnn)."""
    from disco_b200 import ops
    from disco_b200.synth import make_utterance
    y, s, n = (np.stack(a) for a in zip(*[make_utterance(seed + b, K, C, L, gate_period=2048) for b in range(B)]))
    S = ops.stft(torch.from_numpy(s[:, :, 0].copy()).to(dev))
    N = ops.stft(torch.from_numpy(n[:, :, 0].copy()).to(dev))
    mz = ops.tf_mask(S, N, "ibm1").contiguous()
    mw = ops.tf_mask(S, 0.5 * N, "ibm1").contiguous()
    for m, flip in ((mz, False), (mw, True)):
        m[..., list(ONES)] = 0.0 if flip else 1.0
        m[..., list(ZEROS)] = 1.0 if flip else 0.0
    assert set(np.unique(mz.cpu().numpy())) <= {0.0, 1.0}
    return torch.from_numpy(y).to(dev), mz, mw


def _run(y, mz, mw):
    from disco_b200.tango import tango_batched
    out = tango_batched(y, masks=(mz, mw), out_layout="FT")
    torch.cuda.synchronize()
    return {k: out[k] for k in ("yf", "z_y", "zn")}


def _finite(out):
    return all(bool(torch.isfinite(torch.view_as_real(v)).all()) for v in out.values())


@pytest.mark.parametrize("K,C", [(1, 4), (2, 4), (1, 8)])
def test_binary_masks(dev, K, C):
    """K = 1, C = 4: two-mask fused route (two-set workspace solve); K = 2, C = 4: fused middle pass and the D = 5
    cooperative solve; K = 1, C = 8: the 5..8-microphone route.  Finite and exactly homogeneous at every scale
    (power-of-two scales of y are exact), and per node within TOL of the float64 Tango with the solver policy."""
    from oracle import solve_f64, tango_f64
    y, mz, mw = _inputs(dev, 2, K, C, seed=10 * K + C)
    base = _run(y, mz, mw)
    assert _finite(base)
    for a in (2.0 ** -20, 2.0 ** 15):
        out = _run(y * a, mz, mw)
        assert _finite(out), a
        for nm in base:
            assert torch.equal(out[nm], base[nm] * a), (a, nm)
    policy = lambda Rss, Rnn, mu, typ, rank: solve_f64.solve(Rss, Rnn, mu, typ, rank)[0]
    yn, mzn, mwn = y.cpu().numpy(), mz.cpu().numpy(), mw.cpu().numpy()
    for b in range(y.shape[0]):
        ref = tango_f64.offline_tango(yn[b], masks=(mzn[b].transpose(0, 2, 1), mwn[b].transpose(0, 2, 1)),
                                      solve=policy)
        for nm in ("yf", "z_y", "zn"):
            got = base[nm][b].cpu().numpy()
            for k in range(K):
                err = rel_l2_mag(got[k], ref[nm][k])
                assert record_parity("binary_masks_k%dc%d_b%d" % (K, C, b), nm, k, err_f64=err,
                                     note="ibm masks with all-1 / all-0 bins; float64 Tango with the solver policy"), \
                    (nm, b, k, err)


def test_dead_microphone(dev):
    """A dead microphone, the reference one or another: every output finite, and both filter sets of the two-mask
    pass equal the float64 policy solve of the statistics that pass accumulated.  The statistics are not exactly
    those of the smaller array: the STFT transforms two real channels per complex FFT, and separating them leaves
    ~1e-7 of the partner channel's level in a silent one, so the dead row and column hold rounding noise (a
    numerically singular direction, which the pivot floor handles) instead of exact zeros.
    End to end, a dead non-reference microphone leaves every output within 5e-2 (relative magnitude) of the run
    on the array without it: the two runs' float32 statistics differ in rounding, which bins with a small eigen-gap
    amplify to ~1e-2, far above TOL, but a mishandled singular direction gives O(1).  A dead reference
    microphone gives z_y at the rounding level of the crosstalk, <= 1e-5 of the input."""
    from disco_b200 import ops
    from oracle import solve_f64
    for d in (2, 0):
        y, mz, mw = _inputs(dev, 2, 1, 4, seed=31)
        y[:, :, d] = 0
        out = _run(y, mz, mw)
        assert _finite(out), d
        if d == 2:
            ref = _run(y[:, :, [0, 1, 3]].contiguous(), mz, mw)
            for nm in out:
                err = rel_l2_mag(out[nm].cpu().numpy(), ref[nm].cpu().numpy())
                assert err <= 5e-2, (nm, err)
        else:
            assert float(torch.linalg.vector_norm(out["z_y"])) <= 1e-5 * float(torch.linalg.vector_norm(y))
        _, ws = ops.stft_scm2(y[:, 0].contiguous(), mz[:, 0].contiguous(), mw[:, 0].contiguous(), want_Y=False)
        W12, _ = ops.mwf_solve_workspace2(ws, 2, 4, L)
        for q in range(2):
            Rss, Rnn = ops.scm_from_workspace(ws, 2, 4, L, n_set=2, set=q)
            w, _ = solve_f64.solve(Rss.cpu().numpy().astype(complex), Rnn.cpu().numpy().astype(complex))
            W = W12[q].cpu().numpy()
            assert np.all(np.isfinite(W)) and rel_l2(W, w) <= 2e-6, (d, q, rel_l2(W, w))


@pytest.mark.parametrize("K,C", [(1, 4), (2, 4), (1, 8)])
def test_silent_utterance_in_batch(dev, K, C):
    """An all-zero utterance gives exactly zero outputs, and every other utterance is bit-identical to the run
    where that slot holds its original content (the tiling depends only on shapes)."""
    y, mz, mw = _inputs(dev, 3, K, C, seed=40 + K + C)
    full = _run(y, mz, mw)
    y0 = y.clone()
    y0[1] = 0
    out = _run(y0, mz, mw)
    assert _finite(out)
    for nm in out:
        assert bool((out[nm][1] == 0).all()), nm
        assert torch.equal(out[nm][0], full[nm][0]) and torch.equal(out[nm][2], full[nm][2]), nm


@pytest.mark.parametrize("C", [1, 2, 3, 4])
def test_workspace_solve_equals_matrix_solve(dev, C):
    """On binary-mask inputs: mwf_solve_workspace (one set) and mwf_solve_workspace2 (two sets) are bit-identical
    to mwf_solve on the matrices scm_from_workspace rebuilds."""
    from disco_b200 import ops
    y, mz, mw = _inputs(dev, 3, 1, C, seed=50 + C)
    x = y[:, 0].contiguous()
    for typ, rank, mu in (("gevd", 1, 1.0), ("gevd", "full", 2.5), ("mwf", 1, 1.0), ("r1-mwf", 1, 1.0)):
        _, ws = ops.stft_scm(x, mz[:, 0].contiguous(), keep_partials=True)
        W, T1 = ops.mwf_solve_workspace(ws, 3, C, L, mu=mu, type=typ, rank=rank)
        Rss, Rnn = ops.scm_from_workspace(ws, 3, C, L)
        W2, T2 = ops.mwf_solve(Rss, Rnn, mu, typ, rank)
        assert torch.equal(W, W2) and torch.equal(T1, T2), (typ, rank)
        _, ws = ops.stft_scm2(x, mz[:, 0].contiguous(), mw[:, 0].contiguous(), want_Y=False)
        W12, T12 = ops.mwf_solve_workspace2(ws, 3, C, L, mu=mu, type=typ, rank=rank)
        for q in range(2):
            Rss, Rnn = ops.scm_from_workspace(ws, 3, C, L, n_set=2, set=q)
            W2, T2 = ops.mwf_solve(Rss, Rnn, mu, typ, rank)
            assert torch.equal(W12[q], W2) and torch.equal(T12[q], T2), (typ, rank, q)
