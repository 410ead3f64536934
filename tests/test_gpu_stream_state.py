"""Saving, restoring and moving live online Tango sessions (OnlineTangoStream.state / from_state, OnlineTangoPool.export
/ restore).  The yardstick is always the same session run without interruption: the outputs emitted before the
export followed by those emitted after the restore equal its outputs bit for bit (equal values, or equal bits where an
ill-conditioned first filter gives NaN), z_y, zn, yf and every time signal.

Routes: stream -> file -> stream; one index of a B = 3 stream -> a pool slot among busy ones; pool slot -> stream;
every open slot of a pool -> a larger pool (released from the old one); B = 1 states -> one lockstep stream.  Splitting
or joining lockstep streams keeps the bits when every stream's signals pair among themselves (n_C * C even for every
group, K even), which the geometries of those routes satisfy.  Export points: before the first frame, inside the
first hop, mid-block, at a block close, with a lag-2 filter pending, after R2 first exists."""

import numpy as np
import pytest
import torch

from test_gpu_ragged_stream import _r0_nodes, _same
from test_gpu_stream import _r0

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _sizes(rng, a, b):
    """Chunk sizes that cover samples [a, b): empty chunks, chunks under a hop, chunks over several blocks."""
    out, pos = [], a
    while pos < b:
        k = min(b - pos, int(rng.choice([0, 1, 37, 128, 255, 256, 700, 2100, 5000])))
        out.append(k)
        pos += k
    return out


def _cat(outs):
    keys = [k for k in outs[0] if k != "t0"]
    return {k: torch.cat([o[k] for o in outs], dim=2) for k in keys}


def _feed(st, x, sizes, pos, fn):
    """Push x = (y, s, n) (s, n None without clean components) from sample pos in chunks of `sizes`."""
    y, s, n = x
    outs = []
    for k in sizes:
        sn = {} if s is None else dict(s_chunk=s[..., pos:pos + k], n_chunk=n[..., pos:pos + k])
        outs.append(st.push(y[..., pos:pos + k], fn, **sn))
        pos += k
    return outs


def _inputs(rng, lead, L, clean, dev):
    y = torch.from_numpy(rng.standard_normal(lead + (L,)).astype(np.float32)).to(dev)
    if not clean:
        return y, None, None
    n = torch.from_numpy(0.5 * rng.standard_normal(lead + (L,)).astype(np.float32)).to(dev)
    return y + n, y, n


def _mask_table(rng, B, K, T, F, dev):
    return [torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev) for _ in range(2)]


def _stream_fn(mz, mw):
    return lambda t0, Y, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]])


def _check(got, want):
    assert got.keys() == want.keys()
    for k in want:
        assert _same(got[k], want[k]), k


def _stream_kw(case, dev, B):
    """OnlineTangoStream arguments of a case, with R0 on the device when asked."""
    kw = dict(case)
    C, K = kw.pop("C"), kw.pop("K")
    F = kw["n_fft"] // 2 + 1
    if kw.pop("R0", False):
        if isinstance(C, int):
            kw["R0"] = _r0(B, K, C, F, 7, dev)
        else:
            kw["R0"] = _r0_nodes(B, C, F, 7, dev, every=1)
    return (B, K, C), kw


def _lead(B, K, C):
    return (B, K, C) if isinstance(C, int) else (B, sum(C))


# export points in samples, as functions of (H, P): (name, samples in at the export)
POINTS = {
    "start": lambda H, P: 0,
    "first_hop": lambda H, P: H // 2,
    "mid_block": lambda H, P: (P + P // 2 + 1) * H + 17,
    "block_close": lambda H, P: 2 * P * H,                  # frames_out = 2 P: a block has just closed
    "lag_pending": lambda H, P: (3 * P + 1) * H + 5,        # with lag 2 the filters of two blocks are pending
}

# the options grid: int C and ragged, D <= 8 and wide, modes x filter types, clean components and vads, R0, n_fft,
# block and lag
CASES = [
    dict(K=4, C=2, n_fft=512, block=8, lag=1),
    dict(K=4, C=[2, 4, 6, 4], n_fft=256, block=8, lag=2, mask_for_z="distant", filter_type="mwf", R0=True,
         wide=True),
    dict(K=2, C=[15, 1], n_fft=512, block=1, lag=1, mask_for_z="previous", filter_type="r1-mwf", wide=True),
    dict(K=8, C=2, n_fft=256, block=8, lag=2, mask_for_z="compressed", clean=True, wide=True),
    dict(K=1, C=4, n_fft=1024, block=8, lag=1, R0=True, filter_type="gevd", rank=2),
    dict(K=3, C=3, n_fft=512, block=64, lag=1, mask_for_z="use_oracle_refs", vads=("irm1", "ibm1")),
    dict(K=2, C=[3, 5], n_fft=256, block=8, lag=2, mask_for_z="use_oracle_zs", vads=("irm2", "irm1"), R0=True),
    dict(K=4, C=[4, 4, 4, 4], n_fft=512, block=8, lag=1, mask_for_z="distant", filter_type="gevd"),
    dict(K=2, C=4, n_fft=256, block=8, lag=1, mask_for_z="local", filter_type="r1-mwf"),
]


def _stream_session(case, dev, point, seed, tmp_path, B=2):
    """One session uninterrupted and the same session saved at `point` (a function of H and P: the samples in at the
    export) through a file and resumed in a new stream."""
    from disco_b200.stream import OnlineTangoStream
    (B, K, C), kw = _stream_kw(case, dev, B)
    clean = kw.get("clean", False) or kw.get("vads") is not None
    rng = np.random.default_rng(seed)
    H, P = kw["n_fft"] // 2, kw["block"]
    L = (5 * P + 3) * H + 77
    cut = point(H, P)
    x = _inputs(rng, _lead(B, K, C), L, clean, dev)
    fn = None if kw.get("vads") else _stream_fn(*_mask_table(rng, B, K, L // H + 1, H + 1, dev))
    first, rest = _sizes(rng, 0, cut), _sizes(rng, cut, L)

    whole = OnlineTangoStream(B, K, C, device=dev, **kw)
    outs = _feed(whole, x, first + rest, 0, fn) + [whole.flush(fn)]

    st = OnlineTangoStream(B, K, C, device=dev, **kw)
    pre = _feed(st, x, first, 0, fn)
    state = st.state()
    path = tmp_path / "session.pt"
    torch.save(state, path)
    state = torch.load(path, weights_only=True)
    resumed = OnlineTangoStream.from_state(state, device=dev)
    assert resumed.samples_in == cut and resumed.frames_out == st.frames_out
    post = _feed(resumed, x, rest, cut, fn) + [resumed.flush(fn)]
    _check(_cat(pre + post), _cat(outs))
    # the exporting stream continues unaffected
    post2 = _feed(st, x, rest, cut, fn) + [st.flush(fn)]
    _check(_cat(pre + post2), _cat(outs))
    return state


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("point", sorted(POINTS))
def test_stream_to_file_to_stream(dev, tmp_path, case, point):
    if point == "lag_pending" and CASES[case]["lag"] != 2:
        pytest.skip("lag 1 keeps one filter")
    state = _stream_session(CASES[case], dev, POINTS[point], 100 + case, tmp_path)
    if point == "block_close":
        assert state["closed"] == 2 and all(g["R1"] is not None for g in state["groups"])
        assert all(g["R2"] is not None for g in state["groups"])      # R2 exists, K > 1 included
        assert state["groups"][0]["W1"].shape[1] == CASES[case]["lag"]
    if point == "start":
        assert state["closed"] == 0 and (CASES[case].get("R0") or state["groups"][0]["R1"] is None)
        if CASES[case]["K"] > 1:
            assert state["groups"][0]["R2"] is None


def test_after_r2_first_exists(dev, tmp_path):
    """K > 1: exported right after the first block closed (R2 was None until then)."""
    case = dict(K=3, C=2, n_fft=256, block=4, lag=1, mask_for_z="distant")
    state = _stream_session(case, dev, lambda H, P: (P + 1) * H, 7, tmp_path, B=1)
    assert state["closed"] == 1 and state["groups"][0]["R2"] is not None


# ------------------------------------------------------------------------------------------------ pools
def _pool_fn(tables):
    """Pool mask_fn over per-slot mask tables {slot: (mz [K, T, F], mw)} (slot -> session)."""
    def fn(t0, n_fr, Y, z, zn):
        S, K, f, F = z.shape
        mz = torch.full((S, K, f, F), float("nan"), device=z.device)
        mw = mz.clone()
        for s in np.nonzero(n_fr)[0]:
            a, b = tables[s]
            mz[s, :, :n_fr[s]] = a[:, t0[s]:t0[s] + n_fr[s]]
            mw[s, :, :n_fr[s]] = b[:, t0[s]:t0[s] + n_fr[s]]
        return mz, mw
    return fn


def _slot_out(out, s):
    f, m = int(out["frames"][s]), int(out["samples"][s])
    return {"z_y": out["z_y"][s:s + 1, :, :f], "zn": out["zn"][s:s + 1, :, :f], "yf": out["yf"][s:s + 1, :, :f],
            "yf_time": out["yf_time"][s:s + 1, :, :m]}


def _pool_push(pool, xs, pos, n, tables):
    """Push n[s] samples of session xs[s] (slot -> [1, ..., L]) at pos[s]; returns per-slot outputs."""
    lead = pool._lead(pool.S)
    y = torch.full(lead + (max(max(n), 1),), float("nan"), device=pool.device)
    for s, k in enumerate(n):
        if k:
            y[s, ..., :k] = xs[s][0, ..., pos[s]:pos[s] + k]
            pos[s] += k
    out = pool.push(y, np.array(n, dtype=np.int64), _pool_fn(tables))
    return {s: _slot_out(out, s) for s in range(pool.S) if pool.is_open(s) or n[s]}


@pytest.mark.parametrize("C,K,point", [(2, 4, "mid_block"), ([2, 4, 6, 4], 4, "lag_pending"),
                                       (4, 2, "block_close"), ([2, 4, 6, 4], 4, "first_hop")])
def test_stream_index_to_pool_slot(dev, C, K, point):
    """Index 1 of a B = 3 stream leaves for slot 5 of a pool of 7 whose other slots are busy, and continues there
    exactly as it would have in the stream."""
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    rng = np.random.default_rng(11)
    n_fft, P, lag = 256, 4, 2
    H, F = n_fft // 2, n_fft // 2 + 1
    L = (6 * P + 2) * H + 31
    cut = POINTS[point](H, P)
    x = _inputs(rng, _lead(3, K, C), L, False, dev)
    mz, mw = _mask_table(rng, 3, K, L // H + 1, F, dev)
    fn = _stream_fn(mz, mw)
    kw = dict(n_fft=n_fft, block=P, lag=lag, mask_for_z="distant", filter_type="mwf")
    st = OnlineTangoStream(3, K, C, device=dev, wide=True, **kw)
    sizes = _sizes(rng, 0, cut)
    pre = _feed(st, x, sizes, 0, fn)
    state = st.state(1)
    rest = _sizes(rng, cut, L)
    post_stream = _feed(st, x, rest, cut, fn) + [st.flush(fn)]

    pool = OnlineTangoPool(7, K, C, device=dev, **kw)
    others = {s: _inputs(rng, _lead(1, K, C), L, False, dev)[0] for s in (0, 2, 6)}
    tables = {s: tuple(t[0] for t in _mask_table(rng, 1, K, L // H + 1, F, dev)) for s in others}
    pool.open([0, 2])
    pos = [0] * 7
    xs = dict(others)
    _pool_push(pool, xs, pos, [900, 0, 1500, 0, 0, 0, 0], tables)
    pool.restore(5, state)
    pool.open([6])
    xs[5], pos[5] = x[0][1:2], cut
    tables[5] = (mz[1], mw[1])
    got = []
    for k in rest:
        n = [int(rng.integers(0, 600)) if s in (0, 2, 6) else 0 for s in range(7)]
        n = [min(v, L - pos[s]) if s in xs else 0 for s, v in enumerate(n)]
        n[5] = k
        got.append(_pool_push(pool, xs, pos, n, tables)[5])
    out = pool.close([5], _pool_fn(tables))
    got.append(_slot_out(out, 5))
    want = _cat(pre + post_stream)
    have = _cat([{k: v[1:2] for k, v in o.items() if k != "t0"} for o in pre] + got)
    _check(have, {k: v[1:2] for k, v in want.items()})


@pytest.mark.parametrize("C,K,lag", [(3, 3, 1), ([2, 4, 6, 4], 4, 2), ([15, 1], 2, 1)])
def test_pool_slot_to_stream_and_larger_pool(dev, C, K, lag):
    """Slots of a pool of 3, exported mid-flight: one into OnlineTangoStream.from_state (its pool keeps running it
    after an export without release, as the yardstick), then every open slot released into a pool of 8 at other
    indices.  Each session's outputs equal the uninterrupted pool's."""
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    rng = np.random.default_rng(21)
    n_fft, P = 512, 8
    H, F = n_fft // 2, n_fft // 2 + 1
    L = (5 * P) * H + 99
    kw = dict(n_fft=n_fft, block=P, lag=lag, mask_for_z="previous", filter_type="gevd")
    xs = {s: _inputs(rng, _lead(1, K, C), L, False, dev)[0] for s in range(3)}
    tables = {s: tuple(t[0] for t in _mask_table(rng, 1, K, L // H + 1, F, dev)) for s in range(3)}
    schedule = [[int(rng.integers(0, 1800)) for _ in range(3)] for _ in range(200)]

    def run(resize_at=None, to_stream_at=None):
        pool = OnlineTangoPool(3, K, C, device=dev, **kw)
        pool.open([0, 1, 2])
        pos, outs, where = [0] * 3, {s: [] for s in range(3)}, {s: s for s in range(3)}
        stream, fn = None, None
        for i, n in enumerate(schedule):
            n = [min(v, L - pos[s]) for s, v in enumerate(n)]
            if not any(n):
                break
            if i == to_stream_at:
                stream = OnlineTangoStream.from_state(pool.export(1), device=dev)
                s_pos, s_outs = pos[1], []
                fn = _stream_fn(tables[1][0][None], tables[1][1][None])
            if i == resize_at:
                big = OnlineTangoPool(8, K, C, device=dev, **kw)
                where = {0: 6, 1: 3, 2: 0}
                for s in range(3):
                    big.restore(where[s], pool.export(s, release=True))
                assert not pool._open.any()
                pool = big
            m = {where[s]: n[s] for s in range(3)}
            xsw = {where[s]: xs[s] for s in range(3)}
            tw = {where[s]: tables[s] for s in range(3)}
            p = {where[s]: pos[s] for s in range(3)}
            pl = [p.get(s, 0) for s in range(pool.S)]
            got = _pool_push(pool, xsw, pl, [m.get(s, 0) for s in range(pool.S)], tw)
            for s in range(3):
                outs[s].append(got[where[s]])
                pos[s] = pl[where[s]]
            if stream is not None:
                k = n[1]
                s_outs.extend(_feed(stream, (xs[1], None, None), [k], s_pos, fn))
                s_pos += k
        tw = {where[s]: tables[s] for s in range(3)}
        out = pool.close([where[s] for s in range(3)], _pool_fn(tw))
        for s in range(3):
            outs[s].append(_slot_out(out, where[s]))
        res = {s: _cat(o) for s, o in outs.items()}
        if stream is not None:
            s_outs.append(stream.flush(fn))
            res["stream"] = _cat(s_outs)
        return res

    whole = run()
    moved = run(resize_at=4, to_stream_at=2)
    for s in range(3):
        _check(moved[s], whole[s])
    # the stream took slot 1 over at push 2: its outputs are the tail of the slot's
    frames = moved["stream"]["yf"].shape[2]
    samples = moved["stream"]["yf_time"].shape[2]
    for k in ("z_y", "zn", "yf"):
        assert _same(moved["stream"][k], whole[1][k][:, :, -frames:]), k
    assert _same(moved["stream"]["yf_time"], whole[1]["yf_time"][:, :, -samples:])


@pytest.mark.parametrize("C,K", [(2, 4), ([2, 4, 6, 4], 4)])
def test_b1_states_join_one_lockstep_stream(dev, C, K):
    """Three B = 1 sessions at the same position join one B = 3 stream, which continues each of them exactly."""
    from disco_b200.stream import OnlineTangoStream
    rng = np.random.default_rng(31)
    kw = dict(n_fft=512, block=8, lag=2, mask_for_z="distant", wide=True)
    H, F = 256, 257
    L, cut = 40 * H + 7, 13 * H + 100
    xs = [_inputs(rng, _lead(1, K, C), L, False, dev)[0] for _ in range(3)]
    tabs = [_mask_table(rng, 1, K, L // H + 1, F, dev) for _ in range(3)]
    first, rest = _sizes(rng, 0, cut), _sizes(rng, cut, L)
    states, wants = [], []
    for x, (mz, mw) in zip(xs, tabs):
        fn = _stream_fn(mz, mw)
        st = OnlineTangoStream(1, K, C, device=dev, **kw)
        pre = _feed(st, (x, None, None), first, 0, fn)
        states.append(st.state())
        wants.append(_cat(pre + _feed(st, (x, None, None), rest, cut, fn) + [st.flush(fn)]))
        wants[-1]["pre"] = _cat(pre)
    joined = OnlineTangoStream.from_state(states, device=dev)
    assert joined.B == 3
    fn = _stream_fn(torch.cat([t[0] for t in tabs]), torch.cat([t[1] for t in tabs]))
    post = _cat(_feed(joined, (torch.cat(xs), None, None), rest, cut, fn) + [joined.flush(fn)])
    for b, want in enumerate(wants):
        pre = want.pop("pre")
        _check({k: torch.cat([pre[k], post[k][b:b + 1]], 2) for k in post}, want)


# ------------------------------------------------------------------------------------------------ extra checks
def test_resume_past_2_31_samples(dev):
    """A session that has passed 2^31 samples resumes exactly.  A stream fed Z zeros (no R0) holds the same device
    state for every Z of one residue mod P H once Z spans lag + 2 blocks (tests/test_gpu_stream_positions.py), so a
    state saved after Z_TWIN zeros, with its counters moved on by 2^31 + 3 P H - Z_TWIN samples, is the state of a
    stream fed 2^31 + 3 P H zeros.  Resumed, it must give what the twin gives, and save itself again unchanged."""
    from disco_b200 import stream_state
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    rng = np.random.default_rng(41)
    n_fft, P, lag, K, C = 1024, 64, 1, 2, 2
    H = n_fft // 2
    twin_zeros = (lag + 2) * P * H
    shift = 2 ** 31 + 3 * P * H - twin_zeros
    L = 3 * P * H + 501
    kw = dict(n_fft=n_fft, block=P, lag=lag, device=dev)
    x = _inputs(rng, (1, K, C), L, False, dev)[0]
    mz, mw = _mask_table(rng, 1, K, (twin_zeros + L) // H + 1, H + 1, dev)
    zeros_fn = lambda t0, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), torch.full(z.shape, 0.5, device=dev))
    twin = OnlineTangoStream(1, K, C, **kw)
    _feed(twin, (torch.zeros((1, K, C, twin_zeros), device=dev), None, None), [twin_zeros], 0, zeros_fn)
    state = twin.state()
    far = dict(state, samples_in=state["samples_in"] + shift, frames_out=state["frames_out"] + shift // H,
               samples_out=state["samples_out"] + shift // H * H, closed=state["closed"] + shift // (P * H))
    stream_state.check(far)
    sizes = _sizes(rng, 0, L)
    T0 = twin.frames_out
    fn = lambda t0, Y, z, zn, off=0: (mz[:, :, t0 - off - T0:t0 - off - T0 + z.shape[2]],
                                      mw[:, :, t0 - off - T0:t0 - off - T0 + z.shape[2]])
    want = _cat(_feed(twin, (x, None, None), sizes, 0, fn) + [twin.flush(fn)])
    long = OnlineTangoStream.from_state(far)
    assert long.samples_in > 2 ** 31
    lfn = lambda t0, Y, z, zn: fn(t0, Y, z, zn, off=shift // H)
    got = _feed(long, (x, None, None), sizes[:len(sizes) // 2], 0, lfn)
    again = long.state()
    assert again["samples_in"] > 2 ** 31 and stream_state.check(again)
    long = OnlineTangoStream.from_state(again)                          # save and resume past 2^31
    pos = sum(sizes[:len(sizes) // 2])
    got += _feed(long, (x, None, None), sizes[len(sizes) // 2:], pos, lfn) + [long.flush(lfn)]
    _check(_cat(got), want)
    # and through a pool slot
    pool = OnlineTangoPool(2, K, C, n_fft=n_fft, block=P, lag=lag, device=dev)
    pool.restore(1, far)
    assert pool.samples_in[1] > 2 ** 31
    back = pool.export(1)
    for k in stream_state.COUNTERS:
        assert back[k] == far[k]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs a second GPU")
def test_restore_on_second_gpu(dev):
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    rng = np.random.default_rng(51)
    d1 = torch.device("cuda:1")
    K, C, n_fft, P = 2, 4, 512, 8
    H = n_fft // 2
    L, cut = 20 * H + 3, 9 * H + 11
    x = _inputs(rng, (1, K, C), L, False, dev)[0]
    mz, mw = _mask_table(rng, 1, K, L // H + 1, H + 1, dev)
    fn = _stream_fn(mz, mw)
    st = OnlineTangoStream(1, K, C, n_fft=n_fft, block=P, device=dev)
    first, rest = _sizes(rng, 0, cut), _sizes(rng, cut, L)
    pre = _feed(st, (x, None, None), first, 0, fn)
    state = st.state()
    want = _cat(pre + _feed(st, (x, None, None), rest, cut, fn) + [st.flush(fn)])
    fn1 = _stream_fn(mz.to(d1), mw.to(d1))
    other = OnlineTangoStream.from_state(state, device=d1)
    post = _feed(other, (x.to(d1), None, None), rest, cut, fn1) + [other.flush(fn1)]
    got = _cat(pre)
    post = _cat(post)
    _check({k: torch.cat([got[k], post[k].to(dev)], 2) for k in got}, want)
    pool = OnlineTangoPool(2, K, C, n_fft=n_fft, block=P, device=d1)
    pool.restore(0, state)
    assert pool._carry.device == d1
