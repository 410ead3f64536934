"""Argument errors of ragged.tango_ragged / ragged.online_tango_ragged without a device: every rejection raises its
type before any device work (every `ops` operator that reaches the library or the device is replaced by one that
fails the test, and CUDA stays uninitialised)."""
import numpy as np
import pytest
import torch

from disco_b200 import ops, ragged

B, L, N_FFT = 2, 2000, 256
T, F = 1 + L // (N_FFT // 2), N_FFT // 2 + 1
HOST_ONLY = {"n_frames", "signal_lengths", "stft_scm_supported", "tango_mid_supported", "max_stream_length"}


@pytest.fixture
def no_device(monkeypatch):
    """Every device-facing ops operator fails the test if called."""
    for name in dir(ops):
        fn = getattr(ops, name)
        if name.startswith("_") or name in HOST_ONLY or not callable(fn) or getattr(fn, "__module__", "") != ops.__name__:
            continue

        def boom(*a, _name=name, **kw):
            raise AssertionError("ops.%s ran before the argument error" % _name)
        monkeypatch.setattr(ops, name, boom)
    yield
    assert not torch.cuda.is_initialized()


def _packed(chans):
    M = sum(chans)
    z = lambda: torch.zeros((B, M, L), dtype=torch.float32)
    return z(), z(), z()


def _masks(K):
    return torch.zeros((B, K, T, F)), torch.zeros((B, K, T, F))


FNS = {"offline": ragged.tango_ragged, "online": ragged.online_tango_ragged}


def _call(which, y, chans, **kw):
    kw.setdefault("n_fft", N_FFT)
    return FNS[which](y, chans, **kw)


@pytest.mark.parametrize("which", sorted(FNS))
@pytest.mark.parametrize("chans,exc", [
    ([2, 3, 0], ValueError),               # a node without microphones
    ([2, -1, 4], ValueError),
    ([2.0, 3, 1], TypeError),              # not integers
    ([True, 3, 2], TypeError),
    ("232", TypeError),
    ([], TypeError),
])
def test_bad_channel_counts(no_device, which, chans, exc):
    y, s, n = _packed([2, 3, 1])
    with pytest.raises(exc):
        _call(which, y, chans, s=s, n=n)


@pytest.mark.parametrize("which", sorted(FNS))
def test_channels_must_sum_to_the_rows(no_device, which):
    y, s, n = _packed([2, 3, 2])
    for chans in ([2, 3, 1], [2, 3, 3], [8]):
        with pytest.raises(ValueError):
            _call(which, y, chans, s=s, n=n)


@pytest.mark.parametrize("which", sorted(FNS))
@pytest.mark.parametrize("chans", [[15, 1, 1], [10] + [2] * 7, [1] * 17, [2] * 16, [14, 1, 2, 1]])
def test_more_than_16_stacked_channels(no_device, which, chans):
    """C_k + K - 1 > 16 for some node, or K > 16: NotImplementedError, as the uniform kernels refuse it."""
    y, s, n = _packed(chans)
    with pytest.raises(NotImplementedError):
        _call(which, y, chans, s=s, n=n)


@pytest.mark.parametrize("which", sorted(FNS))
@pytest.mark.parametrize("ref_mic,exc", [(1, ValueError), (3, ValueError), (-1, ValueError), (0.0, TypeError)])
def test_ref_mic_must_be_a_microphone_of_every_node(no_device, which, ref_mic, exc):
    chans = [2, 1, 3]
    y, s, n = _packed(chans)
    with pytest.raises(exc):
        _call(which, y, chans, s=s, n=n, ref_mic=ref_mic)


@pytest.mark.parametrize("which", sorted(FNS))
@pytest.mark.parametrize("kw,exc", [
    (dict(mask_for_z=None), TypeError),                                      # reference tango.py:343
    (dict(s=None), ValueError),                                              # no masks and no clean components
    (dict(vads=("foo1", "irm1")), ValueError),                               # reference tango.py:223
    (dict(vads=("crnn", "irm1")), ValueError),                               # network masks come in through masks=
    (dict(mask_for_z="use_oracle_sigs"), NotImplementedError),
    (dict(filter_type="lcmv"), AttributeError),                              # internal_formulas.py:79
])
def test_option_errors_of_the_uniform_entry_points(no_device, which, kw, exc):
    chans = [2, 3, 1]
    y, s, n = _packed(chans)
    args = dict(s=s, n=n)
    args.update(kw)
    with pytest.raises(exc):
        _call(which, y, chans, **args)


@pytest.mark.parametrize("which", sorted(FNS))
@pytest.mark.parametrize("mode", ["compressed", "use_oracle_refs", "use_oracle_zs"])
def test_exchange_modes_that_need_the_clean_components(no_device, which, mode):
    chans = [2, 3, 1]
    y, _, _ = _packed(chans)
    with pytest.raises(ValueError):
        _call(which, y, chans, masks=_masks(3), mask_for_z=mode)


@pytest.mark.parametrize("which", sorted(FNS))
def test_shapes(no_device, which):
    chans = [2, 3, 1]
    y, s, n = _packed(chans)
    with pytest.raises(ValueError):
        _call(which, y.view(B, 1, 6, L), chans, s=s, n=n)                   # not packed
    with pytest.raises(ValueError):
        _call(which, y, chans, s=s[:, :5], n=n)                             # s not shaped like y
    with pytest.raises(ValueError):
        _call(which, y.double(), chans, s=s, n=n)
    mz, mw = _masks(3)
    with pytest.raises(ValueError):
        _call(which, y, chans, masks=(mz[:, :2], mw))                       # masks of 2 nodes for 3
    with pytest.raises(ValueError):
        _call(which, y, chans, masks=(mz, mw), n_fft=512)                   # masks of another frame grid
    with pytest.raises(ValueError):
        _call(which, y, chans, s=s, n=n, lengths=[L, N_FFT // 2])           # a length at or below n_fft / 2
    with pytest.raises(ValueError):
        _call(which, y, chans, s=s, n=n, lengths=[L + 1, L])
    with pytest.raises(ValueError):
        _call(which, y, chans, s=s, n=n, lengths=[L])                       # one length for two utterances
    if which == "offline":
        with pytest.raises(ValueError):
            _call(which, y, chans, s=s, n=n, out_layout="XY")


def test_online_R0_is_one_pair_per_node(no_device):
    chans = [2, 3, 1]
    y, s, n = _packed(chans)
    good = [tuple(torch.zeros((B, F, c, c), dtype=torch.complex64) for _ in range(2)) for c in chans]
    bad = [good[:2], good[:2] + [good[0]], good[:2] + [(good[2][0], good[2][1].to(torch.complex128))],
           (good[0][0], good[0][1])]
    for R0 in bad:
        with pytest.raises(ValueError):
            ragged.online_tango_ragged(y, chans, n_fft=N_FFT, s=s, n=n, R0=R0)


def test_layout_groups_nodes_by_count():
    lay = ragged._Layout([2, 4, 2, 1, 4], 13, 0)
    assert lay.K == 5 and list(lay.offsets) == [0, 2, 6, 8, 9]
    assert lay.groups == [(1, [3]), (2, [0, 2]), (4, [1, 4])]
    x = torch.arange(13, dtype=torch.float32).view(1, 13, 1).expand(2, 13, 3).contiguous()
    g = lay.gather(x, 2)
    assert g.shape == (2, 2, 2, 3) and g[0, :, :, 0].tolist() == [[0, 1], [6, 7]]
    g = lay.gather(x, 4)
    assert g[1, :, :, 2].tolist() == [[2, 3, 4, 5], [9, 10, 11, 12]]
    assert lay.mic_rows(0, torch.device("cpu")).tolist() == [0, 2, 6, 8, 9]
