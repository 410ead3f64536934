"""Session states of the online Tango stream and pool (disco_b200/stream_state.py), without a device.

States are built on the host.  The stream and pool run on the host device here (their state is plain tensors, and
saving and restoring a session launches no kernel): every `ops` operator that reaches the library is replaced by one
that fails the test, and CUDA stays uninitialised.  Checked: every rejection raises ValueError and leaves its target as
it was; a state survives torch.save -> torch.load(weights_only=True); the mapping of each class's layout to the
format and back keeps every bit (NaN payloads and -0 included), through the stream, the pool's ring of filters and
double-buffered history, and "no carried matrix yet"."""
import io
import re

import numpy as np
import pytest
import torch

from disco_b200 import ops, stream, stream_state
from disco_b200.stream import OnlineTangoPool, OnlineTangoStream, emission

HOST_ONLY = {"n_frames", "signal_lengths", "stft_scm_supported", "tango_mid_supported", "max_stream_length"}
CPU = torch.device("cpu")


@pytest.fixture(autouse=True)
def no_device(monkeypatch):
    for name in dir(ops):
        fn = getattr(ops, name)
        if name.startswith("_") or name in HOST_ONLY or not callable(fn) \
                or getattr(fn, "__module__", "") != ops.__name__:
            continue

        def boom(*a, _name=name, **kw):
            raise AssertionError("ops.%s ran" % _name)
        monkeypatch.setattr(ops, name, boom)
    monkeypatch.setattr(stream, "_cuda_device", lambda device, what: CPU)
    yield
    assert not torch.cuda.is_initialized()


def _rand(gen, shape, dtype):
    """Random values with -0.0 and a NaN payload in them, so that a copy that is not bit-exact shows."""
    x = torch.randn(shape, generator=gen, dtype=torch.float32 if dtype == torch.float32 else torch.complex64)
    flat = (torch.view_as_real(x) if x.is_complex() else x).view(-1)
    if flat.numel() > 2:
        flat[0] = -0.0
        flat[1] = float("nan")
        flat.view(torch.int32)[1] |= 0x1234
    return x


def _synthetic(B=2, K=4, C=None, channels=(2, 4, 6, 4), L=5000, seed=0, *, n_fft=512, block=8, lag=2,
               mask_for_z="local", clean=False, vads=None, seeded=True, **opts):
    """A valid state of the given geometry and options, with random tensors."""
    gen = torch.Generator().manual_seed(seed)
    f32, c64 = torch.float32, torch.complex64
    counts = [C] * K if channels is None else list(channels)
    clean = clean or vads is not None
    T, S = emission(L, n_fft)
    J, F, H, P = T // block, n_fft // 2 + 1, n_fft // 2, block
    nw = min(J, lag)
    groups = []
    for c in sorted(set(counts)):
        nodes = [k for k, x in enumerate(counts) if x == c]
        n, D = len(nodes), c + K - 1
        R = lambda d: None if (J == 0 and not seeded) else [_rand(gen, (B, n, F, d, d), c64) for _ in range(2)]
        groups.append({"C": c, "nodes": nodes, "hist": _rand(gen, (B, n, c, n_fft), f32),
                       "hist_s": _rand(gen, (B, n, c, n_fft), f32) if clean else None,
                       "hist_n": _rand(gen, (B, n, c, n_fft), f32) if clean else None,
                       "Yblk": _rand(gen, (B, n, c, P, F), c64),
                       "Sblk": _rand(gen, (B, n, c, P, F), c64) if "use_oracle_" in mask_for_z else None,
                       "Nblk": _rand(gen, (B, n, c, P, F), c64) if "use_oracle_" in mask_for_z else None,
                       "R1": R(c), "R2": R(D) if (J > 0 or K == 1) else None,
                       "W1": _rand(gen, (B, nw, n, F, c), c64), "W2": _rand(gen, (B, nw, n, F, D), c64)})
    zsn = K > 1 and mask_for_z in ("compressed", "use_oracle_zs")
    st = {"version": 1, "kind": "clean" if clean else "plain", "n_fft": n_fft, "lambda_cor": 0.95, "block": block,
          "lag": lag, "mu": 1.0, "rank": 1, "ref_mic": 0, "filter_type": "gevd", "mask_for_z": mask_for_z,
          "clean": clean, "vads": vads, "wide": max(counts) + K - 1 > 8, "K": K, "C": C,
          "channels": None if channels is None else list(channels), "B": B, "samples_in": L, "frames_out": T,
          "samples_out": S, "closed": J, "groups": groups, "m1": _rand(gen, (B, K, P, F), f32),
          "m2": _rand(gen, (B, K, P, F), f32), "zblk": _rand(gen, (B, K, P, F), c64) if K > 1 else None,
          "zsblk": _rand(gen, (B, K, P, F), c64) if zsn else None,
          "znblk": _rand(gen, (B, K, P, F), c64) if zsn else None,
          "carry": _rand(gen, (B, 6 if clean else 1, K, H), f32)}
    st.update(opts)
    return stream_state.check(st)


def _bits(x):
    return (torch.view_as_real(x) if x.is_complex() else x).contiguous().view(torch.int32)


def _same(a, b, path="state"):
    """Equal structure and bit-identical tensors."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, path
        assert torch.equal(_bits(a), _bits(b)), path
    elif isinstance(a, dict):
        assert isinstance(b, dict) and a.keys() == b.keys(), path
        for k in a:
            _same(a[k], b[k], "%s.%s" % (path, k))
    elif isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (path, i))
    else:
        assert a == b and type(a) is type(b), (path, a, b)


def _slice(state, i):
    """Stream i of a state as a B = 1 state (what OnlineTangoStream.state(i) gives)."""
    def walk(x):
        if isinstance(x, torch.Tensor):
            return x[i:i + 1].clone()
        if isinstance(x, dict):
            return {k: walk(v) for k, v in x.items()}
        if isinstance(x, list):
            return [walk(v) for v in x]
        return x
    out = walk(state)
    out["B"] = 1
    for g, g0 in zip(out["groups"], state["groups"]):
        g["nodes"] = list(g0["nodes"])
    return out


GEOMETRIES = [dict(C=2, channels=None, K=3), dict(C=None, channels=[2, 4, 6, 4], K=4),
              dict(C=None, channels=[15, 1], K=2), dict(C=4, channels=None, K=1)]


# ------------------------------------------------------------------------------------------------ format
@pytest.mark.parametrize("geo", GEOMETRIES)
@pytest.mark.parametrize("L", [0, 200, 256, 257, 5000, 2 ** 31 + 12345])
def test_save_load_round_trip(geo, L):
    st = _synthetic(L=L, **geo)
    buf = io.BytesIO()
    torch.save(st, buf)
    buf.seek(0)
    back = torch.load(buf, weights_only=True)
    _same(st, back)
    stream_state.check(back)


@pytest.mark.parametrize("geo", GEOMETRIES)
@pytest.mark.parametrize("kw", [dict(), dict(mask_for_z="distant", lag=1), dict(clean=True, mask_for_z="compressed"),
                                dict(vads=("irm1", "ibm1"), mask_for_z="use_oracle_zs", block=1),
                                dict(clean=True, mask_for_z="use_oracle_refs", block=64, n_fft=256)])
@pytest.mark.parametrize("L", [0, 300, 8 * 256 + 256, 40 * 256 + 17])
def test_stream_maps_every_bit(geo, kw, L):
    """from_state followed by state() gives the state back, bit for bit, for all streams and for each one."""
    st = _synthetic(L=L, **geo, **kw)
    s = OnlineTangoStream.from_state(st)
    assert (s.samples_in, s.frames_out, s.samples_out, s.closed) == (L,) + emission(L, st["n_fft"]) + (False,)
    _same(s.state(), st)
    for i in range(st["B"]):
        _same(s.state(i), _slice(st, i))
    # B = 1 states joined in order make the same stream
    _same(OnlineTangoStream.from_state([_slice(st, i) for i in range(st["B"])]).state(), st)


@pytest.mark.parametrize("geo", GEOMETRIES)
@pytest.mark.parametrize("lag", [1, 2, 3])
@pytest.mark.parametrize("L", [0, 300, 7 * 256, 9 * 256 + 3, 33 * 256 + 255])
@pytest.mark.parametrize("seeded", [False, True])
def test_pool_maps_every_bit(geo, lag, L, seeded):
    """restore followed by export gives the state back bit for bit, at any slot, next to busy slots, through the
    ring of filters (whose pre-first-block entries are the pass-through (e_ref, -0)) and the history pair."""
    st = _slice(_synthetic(L=L, lag=lag, block=4, mask_for_z="previous", seeded=seeded, **geo), 1)
    counts = st["channels"] or st["C"]
    pool = OnlineTangoPool(5, st["K"], counts, block=4, lag=lag, mask_for_z="previous")
    pool.restore(3, st)
    other = _slice(_synthetic(L=L + 999, lag=lag, block=4, mask_for_z="previous", seed=1, **geo), 0)
    pool.restore(0, other)
    pool._par[3] = 1 - pool._par[3]                  # the live history in the other buffer
    for g in pool._groups:
        g.hist[:, 3] = g.hist[:, 3].flip(0)
    _same(pool.export(3), st)
    _same(pool.export(0), other)
    J = st["closed"]
    for g in pool._groups:
        for j in range(J - lag, 0):                  # blocks before the first read the stored pass-through
            w = g.W1[3, j % (lag + 1)]
            assert torch.equal(_bits(w), _bits(g.pass_[0]))
            assert torch.signbit(w.imag).all()
    if J:
        W1, W2 = pool.filters(3)
        want = {g["C"]: g["W1"][0, -1] for g in st["groups"]}
        if st["channels"] is None:
            assert torch.equal(_bits(W1), _bits(want[st["C"]]))
        else:
            assert all(torch.equal(_bits(W1[c]), _bits(w)) for c, w in want.items())
    # stream <-> pool: the formats are one
    s = OnlineTangoStream.from_state(pool.export(3, release=True), device=None)
    assert not pool.is_open(3) and pool.is_open(0)
    _same(s.state(0), st)
    pool.restore(4, s.state())
    _same(pool.export(4), st)


def test_stream_state_leaves_stream_alone():
    st = _synthetic(L=9 * 256 + 5)
    s = OnlineTangoStream.from_state(st)
    before = [t.clone() for g in s._groups for t in (g.hist[0], g.Yblk)] + [s._carry.clone(), s._m1.clone()]
    a, b = s.state(), s.state(1)
    after = [t for g in s._groups for t in (g.hist[0], g.Yblk)] + [s._carry, s._m1]
    assert all(torch.equal(_bits(x), _bits(y)) for x, y in zip(before, after))
    _same(a, s.state())
    _same(b, s.state(1))


# ------------------------------------------------------------------------------------------------ rejections
def _del(k):
    def f(st):
        del st[k]
    return f


def _set(k, v):
    def f(st):
        st[k] = v
    return f


def _grp(k, v):
    def f(st):
        st["groups"][0][k] = v(st["groups"][0][k]) if callable(v) else v
    return f


BAD = [
    ("version", _set("version", 2)),
    ("version", _set("version", None)),
    ("carry", _del("carry")),
    ("samples_in", _del("samples_in")),
    ("groups", _del("groups")),
    ("groups[0].W2", lambda st: st["groups"][0].pop("W2")),
    ("kind", _set("kind", "clean")),
    ("options", _set("n_fft", 300)),
    ("options", _set("lambda_cor", 1.0)),
    ("options", _set("filter_type", "wiener")),
    ("options", _set("mask_for_z", "compressed")),           # needs clean components
    ("options", _set("lag", 0)),
    ("mask_for_z", _set("mask_for_z", None)),
    ("wide", _set("wide", False)),
    ("channels", _set("channels", [2, 4, 6])),
    ("channels", _set("channels", [2, 4, 6, 0])),
    ("channels", _set("channels", [16, 1, 1, 1])),
    ("C", _set("C", 4)),
    ("groups[0].hist", _set("B", 3)),
    ("B", _set("B", 0)),
    ("samples_in", _set("samples_in", -1)),
    ("samples_in", _set("samples_in", 5000.0)),
    ("frames_out", _set("frames_out", 18)),
    ("frames_out", _set("samples_out", 0)),
    ("closed", _set("closed", 1)),
    ("m1", _set("m1", torch.zeros(2, 4, 8, 257, dtype=torch.float64))),
    ("m2", _set("m2", torch.zeros(2, 4, 7, 257))),
    ("zblk", _set("zblk", None)),
    ("zsblk", _set("zsblk", torch.zeros(2, 4, 8, 257, dtype=torch.complex64))),
    ("carry", _set("carry", torch.zeros(2, 6, 4, 256))),
    ("groups", _set("groups", [])),
    ("groups[0].C", _grp("C", 4)),
    ("groups[0].hist", _grp("hist", lambda h: h[..., :256])),
    ("groups[0].hist_s", _grp("hist_s", torch.zeros(2, 1, 2, 512))),
    ("groups[0].Yblk", _grp("Yblk", lambda y: y.to(torch.complex128))),
    ("groups[0].R1", _grp("R1", None)),                        # carried matrices missing after a block
    ("groups[0].R2[1]", _grp("R2", lambda r: [r[0], r[1][..., :4]])),
    ("groups[0].W1", _grp("W1", lambda w: w[:, :1])),          # lag 2 keeps two filters
    ("groups[0].W2", _grp("W2", "W")),
]


@pytest.mark.parametrize("field,edit", BAD)
def test_rejections(field, edit):
    st = _synthetic()
    edit(st)
    with pytest.raises(ValueError, match=r"\b" + re.escape(field)):
        stream_state.check(st)
    with pytest.raises(ValueError):
        OnlineTangoStream.from_state(st)
    pool = OnlineTangoPool(3, 4, [2, 4, 6, 4], lag=2)
    with pytest.raises(ValueError):
        pool.restore(1, st)
    assert not pool.is_open(1) and not pool._bufs


def test_not_a_state():
    for bad in (None, [], "state", [{"version": 1}]):
        with pytest.raises(ValueError):
            OnlineTangoStream.from_state(bad)
    with pytest.raises(ValueError):
        stream_state.check(None)


@pytest.mark.parametrize("field,value", [("samples_in", 5300), ("n_fft", 1024), ("lambda_cor", 0.9), ("lag", 1),
                                         ("mask_for_z", "previous"), ("channels", [4, 2, 6, 4]), ("block", 4)])
def test_join_needs_equal_settings(field, value):
    a = _synthetic(B=1)
    b = _synthetic(B=2, seed=3, **({"L": value} if field == "samples_in" else {field: value}))
    with pytest.raises(ValueError, match=field):
        OnlineTangoStream.from_state([a, b])
    with pytest.raises(ValueError, match=field):
        stream_state.concat([b, a])


def test_join_fills_missing_matrices_with_zeros():
    """A state still without carried matrices (closed = 0, no R0) joins one that has them as zeros, the scan's
    start either way."""
    a, b = _synthetic(B=1, L=600, seeded=False), _synthetic(B=2, L=600, seeded=True, seed=5)
    j = stream_state.concat([a, b])
    for g, gb in zip(j["groups"], b["groups"]):
        assert torch.equal(g["R1"][0][:1], torch.zeros_like(g["R1"][0][:1]))
        assert torch.equal(_bits(g["R1"][1][1:]), _bits(gb["R1"][1]))
    _same(stream_state.concat([a])["groups"], a["groups"])


def test_pool_restore_rejections():
    pool = OnlineTangoPool(4, 4, [2, 4, 6, 4], lag=2)
    good = _slice(_synthetic(), 0)
    for kw, match in ((dict(B=2), "B = 2"), (dict(clean=True), "clean"), (dict(lag=1), "lag"),
                      (dict(mask_for_z="distant"), "mask_for_z"), (dict(channels=[4, 2, 6, 4]), "channels"),
                      (dict(n_fft=256), "n_fft"), (dict(block=4), "block")):
        st = _synthetic(**kw) if "B" in kw else _slice(_synthetic(**kw), 0)
        with pytest.raises(ValueError, match=match):
            pool.restore(2, st)
    other = dict(good, mu=0.5)
    with pytest.raises(ValueError, match="mu"):
        pool.restore(2, other)
    assert not pool._bufs and not pool._open.any()
    pool.restore(2, good)
    with pytest.raises(ValueError, match="already open"):
        pool.restore(2, good)
    with pytest.raises(ValueError, match="not open"):
        pool.export(1)
    with pytest.raises(ValueError):
        pool.export(7)
    equal_counts = OnlineTangoPool(2, 4, [4, 4, 4, 4], lag=2)     # packed inputs: not the int-C layout
    with pytest.raises(ValueError, match="C"):
        equal_counts.restore(0, _slice(_synthetic(C=4, channels=None), 0))
    assert not equal_counts._bufs


def test_stream_state_rejections():
    s = OnlineTangoStream.from_state(_synthetic())
    for bad in (2, -1, 1.0, True):
        with pytest.raises(ValueError, match="index"):
            s.state(bad)
    s._closed = True
    with pytest.raises(ValueError, match="closed"):
        s.state()
