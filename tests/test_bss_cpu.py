"""BSS-eval without a device: the float64 oracle (mir_eval's published algorithm) against the brute-force definition,
the G / D / ‖y‖² identities the kernels rely on, the permutation choice, and argument validation of the compat layer
and of the C ABI."""
import numpy as np
import pytest
from scipy.signal import lfilter

from oracle import bss_np


def _sources(rng, nsrc, L, lowpass=False):
    x = rng.standard_normal((nsrc, L))
    if lowpass:
        x = lfilter([0.2, 0.2], [1.0, -0.6], x, axis=1)
    return x.astype(np.float32).astype(np.float64)


def _mix(rng, refs, snr_db=10.0):
    nsrc, L = refs.shape
    mixing = np.eye(nsrc) + 0.3 * rng.standard_normal((nsrc, nsrc))
    est = np.stack([np.convolve(m, [1.0, 0.4, -0.2])[:L] for m in mixing @ refs])
    return est + 10 ** (-snr_db / 20) * rng.standard_normal(est.shape)


@pytest.mark.parametrize("nsrc", [1, 2, 3])
@pytest.mark.parametrize("flen,L", [(16, 200), (16, 9), (64, 300), (64, 40), (512, 700)])
def test_oracle_equals_brute_force(nsrc, flen, L):
    """Short lengths with L + flen - 1 < nsrc flen make G singular: the delayed references then span every zero-padded
    signal, so P_all e = e (SAR beyond 100 dB, rounding-level artifacts) while SDR and SIR stay well defined."""
    rng = np.random.default_rng(nsrc * 1000 + flen + L)
    refs = _sources(rng, nsrc, L)
    ests = _mix(rng, refs)
    singular = L + flen - 1 < nsrc * flen
    want = bss_np.brute_force(refs, ests, compute_permutation=True, flen=flen)
    got = bss_np.bss_eval_sources(refs, ests, compute_permutation=True, flen=flen, solver="svd")
    for w, g in zip(want[:2], got[:2]):
        np.testing.assert_allclose(g, w, atol=1e-6, rtol=0)
    if singular:
        assert np.all(want[2] > 100) and np.all(got[2] > 100)
    else:
        np.testing.assert_allclose(got[2], want[2], atol=1e-6, rtol=0)
    np.testing.assert_array_equal(want[3], got[3])
    if not singular:
        lu = bss_np.bss_eval_sources(refs, ests, compute_permutation=True, flen=flen, solver="lu")
        for w, g in zip(want[:3], lu[:3]):
            np.testing.assert_allclose(g, w, atol=1e-6, rtol=0)


@pytest.mark.parametrize("nsrc,flen,L", [(1, 16, 100), (2, 16, 150), (2, 64, 400), (3, 16, 20), (2, 64, 50)])
def test_gram_identities_equal_explicit_projections(nsrc, flen, L):
    """‖P_S e‖² = ‖y_S‖² with L y = D, ‖e - Pe‖² = ‖e‖² - ‖y‖², the single factor of reference 0 = the leading
    block of the full factor; also when G is singular (dependent columns dropped)."""
    rng = np.random.default_rng(7 + nsrc + L)
    refs = _sources(rng, nsrc, L, lowpass=True)
    ests = _mix(rng, refs, snr_db=20.0)
    for j in range(nsrc):
        norms = bss_np.gram_norms(refs, ests[j], flen)
        e = np.hstack((ests[j], np.zeros(flen - 1)))
        A = bss_np.delay_matrix(refs, flen)
        p_all = A @ np.linalg.lstsq(A, e, rcond=None)[0]
        np.testing.assert_allclose(norms[0], e @ e, rtol=1e-12)
        np.testing.assert_allclose(norms[1:1 + nsrc].sum(), p_all @ p_all, rtol=1e-8)
        np.testing.assert_allclose(norms[1 + nsrc], norms[1], rtol=1e-12)   # block 0 of the full factor
        for k in range(nsrc):
            Ak = bss_np.delay_matrix(refs, flen, [k])
            pk = Ak @ np.linalg.lstsq(Ak, e, rcond=None)[0]
            np.testing.assert_allclose(norms[1 + nsrc + k], pk @ pk, rtol=1e-8)
        sdr, sir, sar = bss_np.scores_from_norms(norms, nsrc)
        bf = bss_np.brute_force(refs, ests, compute_permutation=False, flen=flen)
        np.testing.assert_allclose(sdr[j], bf[0][j], atol=1e-6)
        if bf[2][j] > 100:      # singular G: P_all e = e up to rounding, ‖e‖² - ‖y‖² may round to <= 0 (+inf)
            assert sar > 100
        else:
            np.testing.assert_allclose(sar, bf[2][j], atol=1e-6)
        if nsrc > 1:
            np.testing.assert_allclose(sir[j], bf[1][j], atol=1e-6)


def test_permutation_choice_on_swapped_estimates():
    rng = np.random.default_rng(3)
    refs = _sources(rng, 3, 600)
    ests = _mix(rng, refs, snr_db=25.0)
    order = [2, 0, 1]
    sdr, sir, sar, perm = bss_np.bss_eval_sources(refs, ests[order], compute_permutation=True, flen=16)
    ref_sdr, ref_sir, ref_sar, ref_perm = bss_np.bss_eval_sources(refs, ests, compute_permutation=True, flen=16)
    np.testing.assert_array_equal(ref_perm, [0, 1, 2])
    np.testing.assert_array_equal(np.asarray(order)[perm], [0, 1, 2])
    np.testing.assert_allclose(sdr, ref_sdr, atol=1e-9)
    np.testing.assert_allclose(sir, ref_sir, atol=1e-9)


def test_compat_validation_without_device():
    from disco_b200.compat import separation
    x = np.ones((2, 100))
    with pytest.raises(ValueError):
        separation.bss_eval_sources(x, np.ones((2, 99)))
    with pytest.raises(ValueError):
        separation.bss_eval_sources(np.vstack((x[0], np.zeros(100))), x)
    with pytest.raises(ValueError):
        separation.bss_eval_sources(x, np.vstack((x[0], np.zeros(100))))
    with pytest.raises(ValueError):
        separation.bss_eval_sources(np.ones((2, 2, 2, 2)), np.ones((2, 2, 2, 2)))
    with pytest.warns(UserWarning):
        out = separation.bss_eval_sources(np.zeros((0, 10)), np.zeros((0, 10)))
    assert all(o.size == 0 for o in out)


def test_ops_rejects_cpu_tensors():
    import torch
    from disco_b200 import bss_eval
    with pytest.raises(TypeError):
        bss_eval.bss_eval_sources(torch.ones(2, 100), torch.ones(2, 100))


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_abi_validation_and_workspace(lib):
    assert lib.disco_bss_eval(None, None, None, 1, 5, 1, 1000, 512, None, 0, None) == -2     # nsrc > 4
    assert b"4" in lib.disco_last_error()
    assert lib.disco_bss_eval(None, None, None, 1, 2, 1, 1000, 513, None, 0, None) == -1     # flen > 512
    assert lib.disco_bss_eval(None, None, None, 1, 2, 0, 1000, 512, None, 0, None) == -1     # no estimate rows
    assert lib.disco_bss_eval(None, None, None, 1, 2, 1, 0, 512, None, 0, None) == -1        # empty signals
    assert lib.disco_bss_eval(None, None, None, 1, 2, 1, 1000, 512, None, 0, None) == -1     # null pointers
    assert lib.disco_bss_eval_workspace(1, 5, 1, 1000, 512) == 0
    # part sums [nsrc][M][n_seg][flen] + corr [nsrc][M][flen] + [G; D^T] + the single-reference blocks, in doubles
    nsrc, R, L, flen = 2, 3, 144000, 512
    M, n_seg, NF = nsrc + R, -(-L // 4096), nsrc * flen
    want = 8 * (nsrc * M * flen * (n_seg + 1) + (NF + R) * NF + (nsrc - 1) * (flen + R) * flen)
    assert lib.disco_bss_eval_workspace(1, nsrc, R, L, flen) == want
    assert lib.disco_bss_eval_workspace(5, nsrc, R, L, flen) == 5 * want
    # a device pointer is never touched before the size checks: a too-small workspace fails first
    fake = 16
    assert lib.disco_bss_eval(fake, fake, fake, 1, nsrc, R, L, flen, fake, want - 8, None) == -3
