"""Network (DNN) masks through offline_tango on uniform and ragged arrays, next to oracle and 'ivad' masks, and the
concatenated-channel ops refusing a Z that does not match Y."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

L = 8192                     # 33 frames at n_fft 512


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _crnn(n_ch, seed):
    from disco_b200 import dnn_mask
    torch.manual_seed(seed)
    return dnn_mask.CRNN(n_ch, cnn_filters=(4, 6, 6), rnn_units=(8,)).cuda().eval()


def _mods(vads, K, z_sigs="zs_hat"):
    """Small random networks: step 1 hears its own mixture, step 2 also the compressed signals of the K - 1 others
    (one per node for 'zs_hat' / 'zn_hat', z_y and zn of each otherwise)."""
    n2 = 1 + (K - 1) * (1 if z_sigs in ("zs_hat", "zn_hat") else 2)
    return [_crnn(1, 0) if vads[0] == "crnn" else None, _crnn(n2, 1) if vads[1] == "crnn" else None]


# the reference's dtypes: 'ivad' masks are float64, 'ibmX' masks bool, network and ratio masks float32
DTYPES = {"ivad": np.float64, "ibm1": np.bool_, "crnn": np.float32}


@pytest.mark.parametrize("vads", [("ivad", "crnn"), ("crnn", "ivad"), ("crnn", "ibm1")])
def test_dnn_next_to_oracle_masks(dev, vads):
    from disco_b200.tango import offline_tango
    from oracle.make_golden import case_inputs
    for chans in ([2, 2, 2], [2, 3, 2]):
        y, s, n = case_inputs(40, chans, L, vads)
        mods = _mods(vads, len(chans))
        out = offline_tango(y, s, n, list(vads), mods, "local")
        mz, mw = out[7], out[8]
        for k in range(len(chans)):
            assert mz[k].dtype == DTYPES[vads[0]] and mw[k].dtype == DTYPES[vads[1]], (chans, k)
            assert mz[k].shape == mw[k].shape == (257, 33)
            assert 0.0 <= mz[k].min() and mz[k].max() <= 1.0 and 0.0 <= mw[k].min() and mw[k].max() <= 1.0
        again = offline_tango(y, s, n, ["irm1", "irm1"], [None, None], "local", masks=(mz, mw))
        for k in range(len(chans)):
            # step 1 runs on the same mask in both calls.  (An untrained network's masks are nearly constant, so the
            # step-2 GEVD is degenerate and yf is only required to be finite.)
            assert np.array_equal(out[3][k], again[3][k]) and np.array_equal(out[6][k], again[6][k]), (chans, k)
            assert np.all(np.isfinite(out[0][k]))


@pytest.mark.parametrize("z_sigs", ["zs_hat", "interleaved"])
def test_ragged_dnn_masks(dev, z_sigs):
    from disco_b200.tango import offline_tango
    from oracle.make_golden import case_inputs
    chans = [2, 3, 2]
    y, s, n = case_inputs(41, chans, L)
    out = offline_tango(y, s, n, ["crnn", "crnn"], _mods(("crnn", "crnn"), 3, z_sigs), "local", z_sigs)
    mz, mw = out[7], out[8]
    assert all(m.dtype == np.float32 and m.shape == (257, 33) and 0.0 <= m.min() and m.max() <= 1.0 for m in mz + mw)
    again = offline_tango(y, s, n, ["irm1", "irm1"], [None, None], "local", masks=(mz, mw))
    for k in range(3):
        assert np.array_equal(out[3][k], again[3][k]) and np.array_equal(out[6][k], again[6][k])
        assert np.all(np.isfinite(out[0][k]))


def test_get_z_signals_dnn_equals_offline_tango(dev):
    from disco_b200.compat.get_z_signals import offline_tango as step1_only
    from disco_b200.tango import offline_tango
    from oracle.make_golden import case_inputs
    y, s, n = case_inputs(42, [2, 2, 2], L)
    m1 = _crnn(1, 0)
    full = offline_tango(y, s, n, ["crnn", "crnn"], [m1, None], "local")
    z_y, _, _, zn, mz = step1_only(y, s, n, "crnn", [m1], "local")
    for k in range(3):
        assert np.array_equal(z_y[k], full[3][k]) and np.array_equal(zn[k], full[6][k])
        assert np.array_equal(mz[k], full[7][k])


def test_cat_ops_reject_a_z_one_frame_short(dev):
    from disco_b200 import ops
    B, K, C, T, F = 1, 2, 2, 20, 257
    cplx = lambda *shape: torch.zeros(shape, dtype=torch.complex64, device=dev)
    Y, Z = cplx(B, K, C, T, F), cplx(B, K, T - 1, F)
    mask = torch.zeros((B, K, T, F), dtype=torch.float32, device=dev)
    D, J = C + K - 1, (T + 7) // 8
    with pytest.raises(ValueError):
        ops.masked_scm(Y, mask, Z)
    with pytest.raises(ValueError):
        ops.filter_sum(cplx(B, K, F, D), Y, Z)
    with pytest.raises(ValueError):
        ops.scm_recursive(Y, mask, Z, block=8)
    with pytest.raises(ValueError):
        ops.filter_sum_blocks(cplx(B, K, J, F, D), Y, Z, block=8)
