"""CPU checks of the options of the online Tango stream and pool (disco_b200/stream.py): the wide=True opt-in to
D = 9..16, and every rejected filter type, exchange mode and mask source, raised before any CUDA work (without a
device, a call that got past its checks fails on the device instead)."""
import pytest

from disco_b200.tango import _ORACLE_SIGS


def test_stream_wide_validation_without_gpu():
    """Stacks of 9..16 channels are an opt-in: without wide=True the stream refuses them as it always has, with it
    they pass every check and the device ("cpu" is not CUDA) is the first thing to refuse the call; 17 is refused
    either way."""
    from disco_b200.stream import OnlineTangoStream
    for K, C in ((2, 8), (8, 2), (1, 9), (1, 16)):
        with pytest.raises(NotImplementedError, match="wide=True"):
            OnlineTangoStream(1, K, C)
        with pytest.raises(NotImplementedError, match="wide=True"):
            OnlineTangoStream(1, K, C, mask_for_z="distant", vads=("irm1", "irm1"))
    for K, C in ((2, 16), (1, 17)):
        with pytest.raises(NotImplementedError, match="<= 16"):
            OnlineTangoStream(1, K, C, wide=True)
    with pytest.raises(TypeError, match="CUDA device"):
        OnlineTangoStream(1, 4, 4, device="cpu", wide=True)            # D = 7: wide=True is only a limit


@pytest.mark.parametrize("K,C", [(2, 8), (8, 2), (1, 9), (2, 15), (1, 16), (4, 6)])
def test_stream_takes_wide_stacks(K, C):
    """With wide=True, D = 9..16 passes every check: the first thing to refuse the call is the device ("cpu" is not
    CUDA)."""
    from disco_b200.stream import OnlineTangoStream
    with pytest.raises(TypeError, match="CUDA device"):
        OnlineTangoStream(1, K, C, device="cpu", wide=True)
    with pytest.raises(TypeError, match="CUDA device"):
        OnlineTangoStream(1, K, C, device="cpu", mask_for_z="distant", filter_type="mwf", vads=("irm1", "ibm2"),
                          wide=True)


# (keyword arguments, exception, message fragment): each is refused by the stream before any device work
STREAM_ERRORS = [
    (dict(mask_for_z=None), TypeError, "NoneType"),
    (dict(mask_for_z=3), TypeError, "string"),
    (dict(mask_for_z="use_oracle_sigs"), NotImplementedError, "ill-formed"),
    (dict(mask_for_z="use_oracle_sigs", clean=True), NotImplementedError, "ill-formed"),
    (dict(mask_for_z="compressed"), ValueError, "clean components"),
    (dict(mask_for_z="use_oracle_refs"), ValueError, "clean components"),
    (dict(mask_for_z="use_oracle_zs"), ValueError, "clean components"),
    (dict(filter_type="wiener"), AttributeError, "Unknown filter"),
    (dict(filter_type="gevd", rank="two"), ValueError, "int"),
    (dict(vads=("ivad", "irm1")), ValueError, "whole signal"),
    (dict(vads=("irm1", "ivad")), ValueError, "whole signal"),
    (dict(vads=("crnn", "irm1")), ValueError, "mask_fn"),
    (dict(vads=("irm1", "rnn")), ValueError, "mask_fn"),
    (dict(vads=("xyz1", "irm1")), ValueError, "Unknown value"),
    (dict(vads="irm1"), ValueError, "pair"),
    (dict(vads=("irm1",)), ValueError, "pair"),
]


@pytest.mark.parametrize("kw,exc,msg", STREAM_ERRORS, ids=[str(i) for i in range(len(STREAM_ERRORS))])
def test_stream_option_errors(kw, exc, msg):
    from disco_b200.stream import OnlineTangoStream
    for K, C in ((1, 4), (8, 2)):
        with pytest.raises(exc, match=msg):
            OnlineTangoStream(1, K, C, device="cuda:0", wide=True, **kw)


def test_stream_option_errors_match_online_tango():
    """The stream raises what online_tango raises for the same option (tango._check_sources, the solver)."""
    from disco_b200.stream import _check_options
    with pytest.raises(TypeError, match="argument of type 'NoneType' is not iterable"):
        _check_options("gevd", 1, None, True, None)
    with pytest.raises(NotImplementedError) as e:
        _check_options("gevd", 1, "use_oracle_sigs", True, None)
    assert str(e.value) == _ORACLE_SIGS
    with pytest.raises(AttributeError, match="Unknown filter reference"):
        _check_options("bad", 1, "local", False, None)
    for mode in ("local", "distant", "previous", "anything else"):
        _check_options("gevd", 1, mode, False, None)
        _check_options("r1-mwf", "full", mode, False, None)
    for mode in ("compressed", "use_oracle_refs", "use_oracle_zs"):
        _check_options("mwf", 1, mode, True, ("irm2", "iam1"))


POOL_ERRORS = [
    (dict(mask_for_z=None), TypeError),
    (dict(mask_for_z="use_oracle_sigs"), NotImplementedError),
    (dict(mask_for_z="compressed"), ValueError),              # a pool takes no clean components
    (dict(mask_for_z="use_oracle_refs"), ValueError),
    (dict(mask_for_z="use_oracle_zs"), ValueError),
    (dict(filter_type="wiener"), AttributeError),
]


@pytest.mark.parametrize("kw,exc", POOL_ERRORS, ids=[str(i) for i in range(len(POOL_ERRORS))])
def test_pool_option_errors(kw, exc):
    from disco_b200.stream import OnlineTangoPool
    with pytest.raises(exc):
        OnlineTangoPool(3, 8, 2, device="cuda:0", **kw)


def test_pool_options_without_gpu():
    """A pool allocates on its first open, so the accepted options construct here and keep their values."""
    from disco_b200.stream import OnlineTangoPool
    for mode in ("local", "distant", "previous"):
        for ft in ("gevd", "r1-mwf", "mwf"):
            p = OnlineTangoPool(2, 8, 2, device="cuda:0", filter_type=ft, mask_for_z=mode)
            assert (p.filter_type, p.mask_for_z, p.D) == (ft, mode, 9)
    p = OnlineTangoPool(2, 1, 16, device="cuda:0", mask_for_z="distant")
    assert p.D == 16
