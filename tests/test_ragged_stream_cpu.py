"""Argument errors of the online Tango stream and pool on ragged arrays (disco_b200/stream.py with per-node channel
counts), without a device.  Every rejection raises its type before any device work: every `ops` operator that reaches
the library is replaced by one that fails the test, the stream and pool are built on PyTorch's meta device (their
state allocates nowhere), and CUDA stays uninitialised."""
import numpy as np
import pytest
import torch

from disco_b200 import ops, stream
from disco_b200.stream import OnlineTangoPool, OnlineTangoStream

HOST_ONLY = {"n_frames", "signal_lengths", "stft_scm_supported", "tango_mid_supported", "max_stream_length"}
META = torch.device("meta")
CH = [2, 4, 6, 4]                       # K = 4, M = 16, D = 5..9
F = 257


@pytest.fixture(autouse=True)
def no_device(monkeypatch):
    """No ops operator may run, and the streams and pools live on the meta device."""
    for name in dir(ops):
        fn = getattr(ops, name)
        if name.startswith("_") or name in HOST_ONLY or not callable(fn) \
                or getattr(fn, "__module__", "") != ops.__name__:
            continue

        def boom(*a, _name=name, **kw):
            raise AssertionError("ops.%s ran before the argument error" % _name)
        monkeypatch.setattr(ops, name, boom)
    monkeypatch.setattr(stream, "_cuda_device", lambda device, what: META)
    yield
    assert not torch.cuda.is_initialized()


class _OnDevice(torch.Tensor):
    """A host tensor that passes for one on the stream's device, so that the checks after that one run."""

    @property
    def is_cuda(self):
        return True

    @property
    def device(self):
        return META


def _t(*shape, dtype=torch.float32):
    return torch.zeros(shape, dtype=dtype).as_subclass(_OnDevice)


def _stream(B=2, channels=CH, **kw):
    kw.setdefault("wide", True)
    return OnlineTangoStream(B, len(channels), channels, **kw)


# ------------------------------------------------------------------------------------------------ construction
@pytest.mark.parametrize("K,channels,exc,msg", [
    (3, [2, 3, 0], ValueError, "at least one"),           # a node without microphones
    (3, [2, -1, 4], ValueError, "at least one"),
    (3, [2.0, 3, 1], TypeError, "integers"),              # not integers
    (3, [True, 3, 2], TypeError, "integers"),
    (3, [2, None, 2], TypeError, "integers"),
    (1, [], TypeError, "non-empty"),
    (3, [2, 3], ValueError, "K = 3"),                     # one count per node
    (2, [2, 3, 1], ValueError, "K = 2"),
    (17, [1] * 17, NotImplementedError, "at most 16"),     # K > 16
    (2, [16, 1], NotImplementedError, "<= 16"),            # D = 17
    (15, [1] * 14 + [3], NotImplementedError, "<= 16"),
])
def test_bad_channel_counts(K, channels, exc, msg):
    with pytest.raises(exc, match=msg):
        OnlineTangoStream(1, K, channels, wide=True)
    with pytest.raises(exc, match=msg):
        OnlineTangoPool(3, K, channels)


def test_ref_mic_on_every_node():
    for cls in (OnlineTangoStream, OnlineTangoPool):
        with pytest.raises(ValueError, match="every node"):
            cls(1, 3, [1, 3, 2], ref_mic=1)
        with pytest.raises(ValueError, match="every node"):
            cls(1, 4, CH, ref_mic=2, **(dict(wide=True) if cls is OnlineTangoStream else {}))
        with pytest.raises(TypeError, match="integer"):
            cls(1, 3, [1, 3, 2], ref_mic=0.0)
    assert _stream(ref_mic=1).ref_mic == 1


def test_wide_at_nine_or_more():
    """The stream needs wide=True once any count's C_k + K - 1 exceeds 8; the pool takes up to 16 either way."""
    for channels in ([2, 4, 6, 4], [8, 2], [1] * 8 + [2], [15, 1]):
        with pytest.raises(NotImplementedError, match="wide=True"):
            OnlineTangoStream(1, len(channels), channels)
        st = OnlineTangoStream(1, len(channels), channels, wide=True)
        assert st.D == max(channels) + len(channels) - 1
        assert OnlineTangoPool(2, len(channels), channels).D == st.D
    st = OnlineTangoStream(1, 3, [1, 2, 3])                     # D = 5: no opt-in needed
    assert (st.channels, st.C, st.M, st.nodes) == ([1, 2, 3], (1, 2, 3), 6, {1: [0], 2: [1], 3: [2]})
    st = OnlineTangoStream(1, 4, [4, 4, 4, 4])                  # equal counts: one group
    assert st.nodes == {4: [0, 1, 2, 3]} and st.M == 16
    assert OnlineTangoStream(1, 3, np.array([1, 2, 1])).nodes == {1: [0, 2], 2: [1]}


def test_options_as_the_int_stream():
    """The option errors of the int-C stream reach the ragged one unchanged."""
    for kw, exc in ((dict(mask_for_z="compressed"), ValueError), (dict(filter_type="wiener"), AttributeError),
                    (dict(vads=("ivad", "irm1")), ValueError), (dict(block=0), ValueError),
                    (dict(mask_for_z="use_oracle_sigs"), NotImplementedError), (dict(lag=0), NotImplementedError),
                    (dict(n_fft=300), ValueError)):
        with pytest.raises(exc):
            _stream(**kw)
    with pytest.raises(ValueError):
        OnlineTangoPool(2, 4, CH, mask_for_z="use_oracle_zs")
    with pytest.raises(ValueError, match="positive"):
        OnlineTangoStream(0, 4, CH, wide=True)


# ------------------------------------------------------------------------------------------------ R0
def _r0(B=2, channels=CH, dtype=torch.complex64):
    return [(_t(B, F, c, c, dtype=dtype), _t(B, F, c, c, dtype=dtype)) for c in channels]


@pytest.mark.parametrize("bad,exc", [
    (lambda: _r0()[0], ValueError),                                   # one pair, not K
    (lambda: _r0()[:3], ValueError),                                  # K - 1 pairs
    (lambda: _r0() + _r0()[:1], ValueError),
    (lambda: [p[:1] for p in _r0()], ValueError),                     # a pair of one
    (lambda: [(torch.zeros(2, F, c, c, dtype=torch.complex64),) * 2 for c in CH], TypeError),   # host tensors
    (lambda: [("a", "b")] * 4, TypeError),
    (lambda: _r0(channels=[2, 4, 4, 4]), ValueError),                # node 2 holds 6 microphones
    (lambda: _r0(B=1), ValueError),
    (lambda: _r0(dtype=torch.complex128), ValueError),
    (lambda: [(_t(2, 4, F, c, c, dtype=torch.complex64),) * 2 for c in CH], ValueError),        # the int layout
])
def test_bad_r0(bad, exc):
    with pytest.raises(exc):
        _stream(R0=bad())
    pool = OnlineTangoPool(3, 4, CH)
    r0 = bad()
    with pytest.raises(exc):
        pool.open([0, 1], R0=r0)                          # two slots: B = 2 matrices
    assert not pool.is_open(0) and not pool.is_open(1)


# ------------------------------------------------------------------------------------------------ chunks and masks
def test_chunk_shapes():
    st = _stream()
    ok = lambda *a: None
    for x in (_t(2, 15, 100), _t(2, 17, 100), _t(2, 4, 4, 100), _t(1, 16, 100), _t(2, 16), _t(2, 16, 1, 100)):
        with pytest.raises(ValueError, match="expected"):
            st.push(x, ok)
    with pytest.raises(TypeError):
        st.push(torch.zeros(2, 16, 100), ok)                         # a host tensor
    with pytest.raises(TypeError):
        st.push(_t(2, 16, 100, dtype=torch.float64), ok)
    assert st.samples_in == 0 and not st.closed
    cl = _stream(clean=True)
    y = _t(2, 16, 300)
    for s, n in ((y, _t(2, 16, 299)), (_t(2, 15, 300), y), (y, _t(2, 4, 4, 300))):
        with pytest.raises(ValueError):
            cl.push(y, ok, s_chunk=s, n_chunk=n)
    with pytest.raises(ValueError, match="s_chunk and n_chunk"):
        cl.push(y, ok, s_chunk=y)
    with pytest.raises(ValueError, match="clean=True"):
        st.push(y, ok, s_chunk=y, n_chunk=y)
    assert cl.samples_in == 0 and not cl.closed


def test_mask_sources():
    y = _t(2, 16, 600)                                               # completes frames at n_fft 512
    st = _stream()
    with pytest.raises(ValueError, match="mask_fn"):
        st.push(y)
    with pytest.raises(ValueError, match="n_fft / 2"):
        st.flush(lambda *a: None)                                    # no samples yet
    v = _stream(vads=("irm1", "irm2"))
    assert v.clean
    with pytest.raises(ValueError, match="vads"):
        v.push(y, lambda *a: None, s_chunk=y, n_chunk=y)
    with pytest.raises(ValueError, match="s_chunk and n_chunk"):
        v.push(y)
    assert not st.closed and not v.closed and st.samples_in == v.samples_in == 0


def test_pool_y_shapes():
    pool = OnlineTangoPool(3, 4, CH)
    pool._open[1], pool._L[1] = True, 300          # host state of an open slot: the checks read nothing else
    ok = lambda *a: None
    for y in (torch.zeros(3, 15, 10), torch.zeros(3, 4, 4, 10), torch.zeros(2, 16, 10), torch.zeros(3, 16)):
        with pytest.raises(ValueError, match="expected"):
            pool.push(y, [0, 5, 0], ok)
    with pytest.raises(ValueError):
        pool.push(torch.zeros(3, 16, 10), [0, 5, 5], ok)              # samples to free slot 2
    with pytest.raises(TypeError):
        pool.push(torch.zeros(3, 16, 10), [0, 5, 0], ok)              # a valid call on a host tensor
    assert pool._L[1] == 300 and list(pool._open) == [False, True, False]
    assert pool.filters(1) is None
