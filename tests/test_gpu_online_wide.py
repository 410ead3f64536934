"""The online (recursive) kernels at D = C + K - 1 from 9 to 16: scm_recursive_wide_kernel<D> (online_wide.cu) and
filter_sum_blocks_kernel<D> (online.cu, instantiated for 9..16), against float64 through the C ABI with every output
inside a NaN-filled guard band, plus the exactness that their value contract promises and online_tango end to end.

Value contract (DESIGN §4.5): every (group, block, bin) matrix is the two-level definition of online.cu evaluated in
the same operation order, A_j the sequential float32 sum over the block's frames in frame order and
R_j = fmaf(lambda_j, R_(j-1), A_j).  So the bound of tests/test_gpu_kernel_instances.py ("online"),
sqrt(2) (P + J + 6) u, applies unchanged, and the results do not depend on launch geometry, batch position or where
a caller cuts the frames at a block boundary: those are checked bit for bit here.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_gpu_kernel_instances import (N_FFTS, ONLINE_CASES, U, Guarded, Step2, _call, _p, _sel_arg, check_filter,
                                       check_recursive, cplx, node_subset, splits)

pytestmark = pytest.mark.gpu

# the D of online_wide.cu launch_scm_recursive_wide and of online.cu launch_filter_sum_blocks_wide
# (tests/test_online_wide_cpu.py parses both switches and requires this set)
WIDE_D = tuple(range(9, 17))
TS, NS = 4, 4     # online_wide.cu launch_recursive_wide_d: frames per ring stage, stages in the ring
LAM = 0.93
# (T, block, lag, power, R0, mask) at the ring's edges: one stage of frames -1 / +1, the ring's length +- 1, and
# blocks of 5 / 3 frames straddling the wrap of the ring at frame NS * TS
ENGINE_CASES = [(TS - 1, 2, 1, 2, True, True), (TS + 1, 3, 0, 1, False, True), (NS * TS - 1, 5, 1, 2, False, False),
                (NS * TS + 1, 5, 2, 2, True, True), (NS * TS + 4, 3, 1, 1, True, False),
                (3 * NS * TS + 1, 64, 1, 2, False, True)]


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def hermitian_r0(rng, G, F, D):
    """(Rs0, Rn0) [G, F, D, D] complex64, exactly Hermitian with real diagonals, as the recursion keeps them."""
    out = []
    for _ in range(2):
        a = cplx(rng, G, F, D, D).astype(np.complex128)
        r = np.triu((a @ a.conj().transpose(0, 1, 3, 2) / D).astype(np.complex64))
        r = r + np.triu(r, 1).conj().transpose(0, 1, 3, 2)
        r.imag[..., np.arange(D), np.arange(D)] = 0
        out.append(r)
    return out


def run_recursive(dev, Yd, Zd, md, R0, n_utt, K, C, T, P, power, n_fft, sel=None, lam=LAM):
    """disco_scm_recursive into guarded outputs -> Rss, Rnn [n_grp, J, F, D, D]."""
    D, F, J = C + K - 1, n_fft // 2 + 1, (T + P - 1) // P
    n_grp = n_utt * (K if sel is None else len(sel)) if K > 1 else n_utt
    o = Guarded(dev)
    Rss, Rnn = o.new((n_grp, J, F, D, D)), o.new((n_grp, J, F, D, D))
    r0d = [None, None] if R0 is None else [r if isinstance(r, torch.Tensor) else torch.from_numpy(r).to(dev) for r in R0]
    s, n_sel = _sel_arg(sel)
    _call("disco_scm_recursive", _p(Yd), _p(Zd), _p(md), _p(r0d[0]), _p(r0d[1]), _p(Rss), _p(Rnn), ctypes.c_double(lam),
          P, power, n_utt, K, C, T, n_fft, s, n_sel)
    o.check("scm_recursive D=%d T=%d block=%d" % (D, T, P))
    return Rss, Rnn


def run_case(dev, D, n_fft, i, case, seed):
    T, P, lag, power, with_r0, with_mask = case
    F = n_fft // 2 + 1
    rng = np.random.default_rng(seed)
    sp = splits(D)
    C, K = sp[i % len(sp)]
    prob = Step2(rng, dev, 2 if K <= 4 and T < 64 else 1, C, K, T, F, sel=node_subset(K, i),
                 mask="TF" if with_mask else None)
    J = (T + P - 1) // P
    R0 = hermitian_r0(rng, prob.n_grp, F, D) if with_r0 else None
    what = "D=%d C=%d K=%d T=%d block=%d power=%d R0=%d mask=%d" % (D, C, K, T, P, power, with_r0, with_mask)
    Rss, Rnn = run_recursive(dev, prob.Yd, prob.Zd, prob.md, R0, prob.n_utt, K, C, T, P, power, n_fft, prob.sel)
    assert torch.equal(Rss, Rss.conj().transpose(-1, -2)) and torch.equal(Rnn, Rnn.conj().transpose(-1, -2)), what
    Rs, Rn = Rss.cpu().numpy(), Rnn.cpu().numpy()
    if not with_mask and not with_r0:
        assert not np.any(Rn), what + ": Rnn not exactly 0 without a mask"
    check_recursive(Rs, Rn, np.stack([prob.X(g) for g in range(prob.n_grp)]), prob.m, LAM, P, power, R0,
                    math.sqrt(2) * (P + J + 6) * U, what)

    conj = i % 2 == 0
    ref = (D - 1) if (K > 1 and i % 3 == 0) else (i % C)
    W = cplx(rng, prob.n_grp, J, F, D)
    o = Guarded(dev)
    out, resid = o.new((prob.n_grp, T, F)), o.new((prob.n_grp, T, F))
    sel, n_sel = _sel_arg(prob.sel)
    _call("disco_filter_sum_blocks", _p(torch.from_numpy(W).to(dev)), int(conj), _p(prob.Yd), _p(prob.Zd), _p(out),
          _p(resid), ref, P, lag, prob.n_utt, K, C, T, n_fft, sel, n_sel)
    o.check("filter_sum_blocks " + what)
    out, resid = out.cpu().numpy(), resid.cpu().numpy()
    t_first = min(T, lag * P)                              # frames before the first filter pass channel `ref`
    for g in range(prob.n_grp):
        X = prob.X(g)
        assert np.array_equal(out[g, :t_first], X[ref, :t_first]), what
        assert not np.any(resid[g, :t_first]), what
        for j in range(lag, J):
            t0, t1 = j * P, min(T, (j + 1) * P)
            check_filter(out[g, t0:t1], resid[g, t0:t1], W[g, j - lag], X[:, t0:t1], conj, ref,
                         "%s lag=%d group %d block %d" % (what, lag, g, j))


@pytest.mark.parametrize("n_fft", N_FFTS)
@pytest.mark.parametrize("D", WIDE_D)
def test_online_wide_every_instance(dev, D, n_fft):
    """scm_recursive against the per-frame float64 recursion at every block end and filter_sum_blocks against float64,
    over the (C, K) splits of D, node subsets, every row of the D <= 8 table and the ring's edges."""
    for i, case in enumerate(ONLINE_CASES + ENGINE_CASES):
        run_case(dev, D, n_fft, i, case, 7000 * D + 10 * i + n_fft)


@pytest.mark.parametrize("D,C,K,n_fft", [(9, 2, 8, 512), (12, 12, 1, 256), (16, 4, 13, 1024), (16, 16, 1, 512)])
def test_online_wide_split_at_block_boundary(dev, D, C, K, n_fft):
    """Frames [jP, T) run with R0 = the matrices after block j - 1 give the full run's blocks j .. bit for bit, with
    and without a mask, at a boundary inside the ring and at one past it."""
    F = n_fft // 2 + 1
    for i, (T, P, jcut, power, mask) in enumerate([(37, 4, 3, 2, "TF"), (61, 7, 1, 1, None), (70, 8, 5, 2, "TF")]):
        rng = np.random.default_rng(8000 + 100 * D + i)
        prob = Step2(rng, dev, 1, C, K, T, F, mask=mask)
        R0 = hermitian_r0(rng, prob.n_grp, F, D) if i % 2 == 0 else None
        full = run_recursive(dev, prob.Yd, prob.Zd, prob.md, R0, prob.n_utt, K, C, T, P, power, n_fft)
        t0 = jcut * P
        tail = lambda x: None if x is None else x[..., t0:, :].contiguous()
        R0b = (full[0][:, jcut - 1].contiguous(), full[1][:, jcut - 1].contiguous())
        part = run_recursive(dev, tail(prob.Yd), tail(prob.Zd), tail(prob.md), R0b, prob.n_utt, K, C, T - t0, P, power,
                             n_fft)
        for a, b in zip(full, part):
            assert torch.equal(a[:, jcut:], b), "D=%d T=%d block=%d cut at block %d" % (D, T, P, jcut)


@pytest.mark.parametrize("D,C,K", [(9, 2, 8), (11, 4, 8), (16, 1, 16)])
def test_online_wide_batch_independent(dev, D, C, K):
    """A group's matrices are equal whether it runs inside a batch of utterances and nodes or alone (node_sel, one
    utterance)."""
    n_fft, T, P = 256, 45, 6
    F = n_fft // 2 + 1
    rng = np.random.default_rng(8500 + D)
    prob = Step2(rng, dev, 3, C, K, T, F, mask="TF")
    R0 = hermitian_r0(rng, prob.n_grp, F, D)
    Rss, Rnn = run_recursive(dev, prob.Yd, prob.Zd, prob.md, R0, prob.n_utt, K, C, T, P, 2, n_fft)
    for g in (0, prob.n_grp // 2, prob.n_grp - 1):
        b, k = divmod(g, K)
        one = run_recursive(dev, prob.Yd[g:g + 1].contiguous(), prob.Zd[b:b + 1].contiguous(),
                            prob.md[g:g + 1].contiguous(), [r[g:g + 1] for r in R0], 1, K, C, T, P, 2, n_fft, sel=[k])
        assert torch.equal(Rss[g], one[0][0]) and torch.equal(Rnn[g], one[1][0]), "group %d" % g


@pytest.mark.parametrize("D,C,K", [(9, 9, 1), (13, 2, 12), (16, 3, 14)])
def test_online_wide_r0_reads_upper_triangle(dev, D, C, K):
    """R0 entries the header lists as not read (strict lower triangle, imaginary part of the diagonal) set to NaN
    change nothing."""
    n_fft, T, P = 512, 23, 4
    F = n_fft // 2 + 1
    rng = np.random.default_rng(8700 + D)
    prob = Step2(rng, dev, 2, C, K, T, F, mask="TF")
    R0 = hermitian_r0(rng, prob.n_grp, F, D)
    clean = run_recursive(dev, prob.Yd, prob.Zd, prob.md, R0, prob.n_utt, K, C, T, P, 2, n_fft)
    poisoned = []
    for r in R0:
        r = r.copy()
        low = np.tril(np.ones((D, D), bool), -1)
        r[..., low] = np.complex64(complex(np.nan, np.nan))
        r.imag[..., np.arange(D), np.arange(D)] = np.nan
        poisoned.append(r)
    got = run_recursive(dev, prob.Yd, prob.Zd, prob.md, poisoned, prob.n_utt, K, C, T, P, 2, n_fft)
    for a, b in zip(clean, got):
        assert torch.equal(a, b)


# ---- online_tango end to end ------------------------------------------------------------------------------------

def _oracle_online_tango(y, mz, mw, lam, block, lag, fsel, n_fft):
    """oracle/online_np.online_mwf with the float64 solver, per utterance and node, on the bins fsel -> z_y, yf
    [B, K, len(fsel), T] complex128."""
    from oracle import librosa_np, online_np, solve_f64, tango_np
    B, K, C, _ = y.shape
    solve = lambda Rs, Rn, mu, ft, rank: solve_f64.solve(Rs, Rn, mu, ft, rank)
    fn = (tango_np.spatial_correlation_matrix, solve)
    kw = dict(lambda_cor=lam, block=block, lag=lag)
    Y = [[np.stack([librosa_np.stft(y[b, k, c].astype(np.float64), n_fft=n_fft, hop_length=n_fft // 2)
                    for c in range(C)])[:, fsel] for k in range(K)] for b in range(B)]
    z1 = np.stack([np.stack([online_np.online_mwf(Y[b][k], mz[b, k].T[fsel], *fn, **kw)[0] for k in range(K)])
                   for b in range(B)])
    yf = np.empty_like(z1)
    for b in range(B):
        for k in range(K):
            X = Y[b][k] if K == 1 else np.concatenate([Y[b][k], z1[b, [j for j in range(K) if j != k]]], axis=0)
            yf[b, k] = online_np.online_mwf(X, mw[b, k].T[fsel], *fn, **kw)[0]
    return z1, yf


def _rel_abs(got, want):
    return np.linalg.norm(np.abs(got) - np.abs(want)) / np.linalg.norm(np.abs(want))


def _settled(a, j0, P):
    return a[..., j0 * P:]


@pytest.mark.parametrize("B,K,C", [(2, 8, 2), (2, 4, 6), (1, 1, 12), (2, 4, 2)])
def test_online_tango_wide_matches_oracle(dev, B, K, C):
    """online_tango with step-2 stacks of D = C + K - 1 = 9, 9 (step 1 on the D <= 8 kernel at D = 6) and 12 (both
    steps), and D = 5 on the existing kernels as the comparable baseline, against the float64 composition over bins
    including 0 and F - 1, with irm masks of the clean components (4 s, block 16, lambda 0.98, lag 1).

    The 1e-5 relative rule on |yf| and |z_y| holds on every frame whose filter was solved from at least 4 D frames of
    statistics (blocks j >= ceil(4 D / block)).  Before that the GEVD of a D-channel pair smoothed over few frames is
    ill-conditioned and float32 statistics move the filter: on these inputs the first filtered block of yf is 2.9e-4
    off at D = 9 (K = 8), 1.7e-4 at D = 9 (K = 4), 3.1e-5 at D = 12, and 3.2e-6 at D = 5, so the whole signal is held
    to 1e-5 at D <= 8 and to 2e-4 at D >= 9 (measured: 6.9e-5, 5.1e-5, 6.8e-6 and 7.8e-7).  The matrices themselves
    are bit-identical to the D <= 8 engine's definition (tests above)."""
    from disco_b200 import online, ops
    from disco_b200.synth import make_batch
    n_fft, L, lam, block, lag = 512, 64000, 0.98, 16, 1
    y, s, n = make_batch(B, K, C, L, seed0=900 + 10 * K + C)
    S, N = (ops.stft(torch.from_numpy(a[:, :, 0]).contiguous().to(dev), n_fft) for a in (s, n))
    mz = ops.tf_mask(S, N, "irm1")
    mw = ops.tf_mask(S, N, "irm2")
    on = online.online_tango(torch.from_numpy(y).to(dev), (mz, mw), lambda_cor=lam, block=block, lag=lag, n_fft=n_fft)
    T, F = mz.shape[-2:]
    for key in ("yf", "z_y"):
        assert on[key].shape == (B, K, T, F) and bool(torch.isfinite(torch.view_as_real(on[key])).all()), key
    fsel = [0, 37, 128, F - 1]
    z1, yf = _oracle_online_tango(y, mz.cpu().numpy(), mw.cpu().numpy(), lam, block, lag, fsel, n_fft)
    got_z = on["z_y"].cpu().numpy()[:, :, :, fsel].transpose(0, 1, 3, 2)
    got_y = on["yf"].cpu().numpy()[:, :, :, fsel].transpose(0, 1, 3, 2)
    what = "B=%d K=%d C=%d" % (B, K, C)
    for name, got, want, D in (("z_y", got_z, z1, C), ("yf", got_y, yf, C + K - 1)):
        j0 = -(-4 * D // block)
        e = _rel_abs(_settled(got, j0, block), _settled(want, j0, block))
        assert e < 1e-5, "%s: |%s| from block %d: rel %.3g" % (what, name, j0, e)
        e = _rel_abs(got, want)
        assert e < (1e-5 if D <= 8 else 2e-4), "%s: |%s| whole signal: rel %.3g" % (what, name, e)
