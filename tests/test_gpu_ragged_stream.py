"""The online Tango stream and pool (disco_b200/stream.py) on ragged arrays: nodes with different microphone counts,
packed as ragged.py packs them.

- Stream = whole signal: whatever the chunking, a ragged stream's outputs concatenated equal online_tango_ragged on
  the whole signal with the masks mask_fn returned (or the stream's oracle masks) and the same options, and its time
  samples ops.istft / post.to_time of that run, bit for bit.
- Pool slot = lone ragged stream: every slot equals OnlineTangoStream(1, K, channels) fed the same samples.
- Equal counts = the int-C stream: channels = [C] * K with packed chunks equals OnlineTangoStream(B, K, C).
- The int-C stream makes the ops calls it made before ragged arrays were added (tests/golden/stream_int_c_calls.json,
  recorded from the short runs of _int_c_runs)."""
import inspect
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "stream_int_c_calls.json")


# ------------------------------------------------------------------------------------------------ the ops spy
def _describe(v):
    """A value of an ops call as the spy records it: tensors by dtype and shape, host arrays by their values."""
    if isinstance(v, torch.Tensor):
        return "%s%s" % (str(v.dtype).replace("torch.", ""), list(v.shape))
    if isinstance(v, np.ndarray):
        return "array%s" % (v.tolist(),)
    if isinstance(v, (list, tuple)):
        return "(%s)" % ", ".join(_describe(x) for x in v)
    if isinstance(v, (bool, np.bool_)):
        return repr(bool(v))
    if isinstance(v, (int, np.integer)):
        return repr(int(v))
    return repr(v)


class _Spy:
    """Records every public ops call (name and arguments, defaults filled in) while installed."""

    def __init__(self):
        from disco_b200 import ops
        self.ops, self.calls, self.saved = ops, [], {}

    def __enter__(self):
        for name, fn in vars(self.ops).items():
            if name.startswith("_") or not inspect.isfunction(fn) or fn.__module__ != self.ops.__name__:
                continue
            sig = inspect.signature(fn)

            def spy(*a, _fn=fn, _name=name, _sig=sig, **kw):
                bound = _sig.bind(*a, **kw)
                bound.apply_defaults()
                self.calls.append("%s(%s)" % (_name, ", ".join("%s=%s" % (k, _describe(v))
                                                                for k, v in bound.arguments.items())))
                return _fn(*a, **kw)
            self.saved[name] = fn
            setattr(self.ops, name, spy)
        return self

    def __exit__(self, *exc):
        for name, fn in self.saved.items():
            setattr(self.ops, name, fn)


def _int_c_runs(dev):
    """Short int-C runs that reach every stage of the stream and the pool: masks from mask_fn under 'local'; clean
    components, oracle masks and R0 under 'distant' on a wide stack; a pool with a slot opening late."""
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *shape: torch.randn(shape, generator=g, device=dev)
    fn = lambda t0, Y, z, zn: (torch.full(z.shape, 0.7, device=dev), torch.full(z.shape, 0.4, device=dev))
    st = OnlineTangoStream(2, 3, 2, n_fft=256, block=2, lag=1, device=dev)
    for n in (0, 100, 300, 700, 5):
        st.push(rnd(2, 3, 2, n), fn)
    st.flush(fn)
    F = 129
    eye = torch.eye(8, dtype=torch.complex64, device=dev).expand(1, 2, F, 8, 8).contiguous()
    st = OnlineTangoStream(1, 2, 8, n_fft=256, block=2, lag=2, ref_mic=1, R0=(eye, 2 * eye), device=dev,
                           mask_for_z="distant", vads=("irm1", "irm2"), wide=True)
    for n in (200, 0, 900):
        s, nn = rnd(1, 2, 8, n), rnd(1, 2, 8, n)
        st.push(s + nn, s_chunk=s, n_chunk=nn)
    st.flush()
    pool = OnlineTangoPool(3, 2, 2, n_fft=256, block=2, lag=1, device=dev, mask_for_z="previous")
    pfn = lambda t0, n_fr, Y, z, zn: fn(t0, Y, z, zn)
    pool.open([0, 2])
    for step, n in enumerate(([300, 0, 129], [500, 700, 1], [0, 40, 600])):
        pool.push(rnd(3, 2, 2, max(n)), np.array(n, dtype=np.int64), pfn)
        if step == 0:
            pool.open([1])
    pool.close([0, 1, 2], pfn)
    torch.cuda.synchronize()


def test_int_c_stream_makes_the_parent_calls():
    """An int-C stream or pool is the one-group case of the ragged code: same ops calls, same order, same arguments
    (node_sel=None) as before per-node counts were added."""
    with open(GOLDEN) as f:
        want = json.load(f)
    with _Spy() as spy:
        _int_c_runs(torch.device("cuda:0"))
    assert len(spy.calls) == len(want)
    for i, (a, b) in enumerate(zip(spy.calls, want)):
        assert a == b, (i, a, b)


# ------------------------------------------------------------------------------------------------ helpers
@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _same(a, b):
    """Equal values, or equal bits (a NaN of an ill-conditioned first filter compares equal to itself)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if torch.equal(a, b):
        return True
    bits = lambda x: (torch.view_as_real(x) if x.is_complex() else x).contiguous().view(torch.int32)
    return torch.equal(bits(a), bits(b))


def _same_dict(a, b):
    return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)


def _r0_nodes(B, channels, F, seed, dev, every=2):
    """R0 as online_tango_ragged takes it: K pairs [B, F, C_k, C_k]; Hermitian on every `every`-th node, zeros (the
    scan's own start) on the others."""
    from test_gpu_stream import _r0
    out = []
    for k, C in enumerate(channels):
        Rs, Rn = _r0(B, 1, C, F, seed + k, dev)
        if k % every:
            Rs, Rn = torch.zeros_like(Rs), torch.zeros_like(Rn)
        out.append((Rs[:, 0].contiguous(), Rn[:, 0].contiguous()))
    return out


def _packed_stft(y, channels, n_fft):
    """Packed [B, M, T, F] spectra of y [B, M, L] from the per-group transforms of the whole signal."""
    from disco_b200 import ops
    from disco_b200.ragged import _Layout
    lay = _Layout(channels, y.shape[1], 0)
    out = None
    for C, nodes in lay.groups:
        Y = ops.stft(lay.gather(y, C), n_fft)
        Y = Y.reshape(Y.shape[0], len(nodes) * C, *Y.shape[3:])
        if out is None:
            out = torch.empty((y.shape[0], y.shape[1]) + tuple(Y.shape[2:]), dtype=Y.dtype, device=Y.device)
        out.index_copy_(1, lay.rows(C, y.device), Y)
    return out


def _clone_W(W):
    return None if W is None else ({C: w.clone() for C, w in W.items()} if isinstance(W, dict) else W.clone())


def _run(y, s, n, C, sizes, mask_fn, **kw):
    """Push y (and s, n) in chunks of `sizes`, then flush; returns the concatenated outputs, the Y and masks of
    mask_fn, and the filters after every call.  C: an int (y [B, K, C, L]) or per-node counts (y packed)."""
    from disco_b200.stream import OnlineTangoStream
    B, L = y.shape[0], y.shape[-1]
    K = y.shape[1] if isinstance(C, int) else len(C)
    st = OnlineTangoStream(B, K, C, device=y.device, clean=s is not None, wide=True, **kw)
    got, seen, Ws = {}, {"Y": [], "mz": [], "mw": []}, []

    def fn(t0, Y, z, zn):
        assert t0 == sum(m.shape[2] for m in seen["mz"])
        mz, mw = mask_fn(t0, Y, z, zn)
        seen["Y"].append(Y.clone())
        seen["mz"].append(mz.clone())
        seen["mw"].append((mz if mw is None else mw).clone())
        return mz, mw

    fn = fn if mask_fn is not None else None
    pos = 0
    for k in sizes + [None]:
        if k is None:
            out = st.flush(fn)
        else:
            sn = {} if s is None else dict(s_chunk=s[..., pos:pos + k], n_chunk=n[..., pos:pos + k])
            out = st.push(y[..., pos:pos + k], fn, **sn)
            pos += k
        assert out["t0"] == sum(v.shape[2] for v in got.get("yf", []))
        for key, v in out.items():
            if key != "t0":
                got.setdefault(key, []).append(v)
        Ws.append((st.frames_out, _clone_W(st.W1), _clone_W(st.W2)))
    assert st.samples_in == L and st.samples_out == L and st.closed
    cat = {k: torch.cat(v, dim=2) for k, v in got.items()}
    for k, v in seen.items():
        if v:
            cat[k] = torch.cat(v, dim=-2)                       # frames: second to last in Y and the masks
    return cat, Ws, st


def _inputs(rng, B, M, L, clean, dev):
    if not clean:
        return torch.from_numpy(rng.standard_normal((B, M, L)).astype(np.float32)).to(dev), None, None
    s = torch.from_numpy(rng.standard_normal((B, M, L)).astype(np.float32)).to(dev)
    n = torch.from_numpy(0.5 * rng.standard_normal((B, M, L)).astype(np.float32)).to(dev)
    return s + n, s, n


def _masks(rng, B, K, T, F, two, dev):
    mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
    mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
    return lambda t0, Y, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]] if two else None)


def _check_whole(y, s, n, channels, got, Ws, st, block, n_fft, vads, kw):
    """The stream's outputs against online_tango_ragged on the whole signal (and ops.istft / post.to_time of it)."""
    from disco_b200 import ops, post
    from disco_b200.ragged import online_tango_ragged
    L = y.shape[-1]
    clean = s is not None
    extra = dict(s=s, n=n) if clean else {}
    if vads is not None:
        ref = online_tango_ragged(y, channels, None, block=block, n_fft=n_fft, vads=vads, **extra, **kw)
        assert _same(got["masks_z"], ref["masks_z"]) and _same(got["mask_w"], ref["mask_w"])
    else:
        ref = online_tango_ragged(y, channels, (got["mz"], got["mw"]), block=block, n_fft=n_fft, **extra, **kw)
        assert torch.equal(got["Y"], _packed_stft(y, channels, n_fft))     # what mask_fn saw
    assert got["yf"].shape[2] == ops.n_frames(L, n_fft)
    for k in ("z_y", "zn", "yf") + (("z_s", "z_n", "sf", "nf") if clean else ()):
        assert _same(got[k], ref[k]), k
    if clean:
        want = post.to_time(ref, L, n_fft, layout="TF")
        for k in ("yf", "z_y", "sf", "nf", "z_s", "z_n"):
            assert _same(got[k + "_time"], want[k]), k + "_time"
    else:
        assert _same(got["yf_time"], ops.istft(ref["yf"], L, n_fft))
    assert st.nodes == ref["nodes"]
    J = ref["W1"][channels[0]].shape[2]
    for i, (frames, W1, W2) in enumerate(Ws):
        closed = frames // block if i + 1 < len(Ws) else J
        if closed == 0:
            assert W1 is None and W2 is None
        else:
            assert _same_dict(W1, {C: w[:, :, closed - 1] for C, w in ref["W1"].items()}), i
            assert _same_dict(W2, {C: w[:, :, closed - 1] for C, w in ref["W2"].items()}), i
    return ref


# ------------------------------------------------------------------------------------------------ stream = whole signal
# (n_fft, B, channels, block, lag, mask_for_z, filter_type, rank, clean, vads, R0, hops)
CASES = [
    (512, 2, [2, 4, 6, 4], 8, 1, "local", "gevd", 1, False, None, True, 40),
    (256, 1, [1, 2, 3], 1, 2, "distant", "mwf", 1, True, ("irm1", "irm1"), False, 14),
    (1024, 1, [8, 2], 8, 1, "previous", "r1-mwf", 1, False, None, True, 30),
    (256, 1, [15, 1], 8, 2, "use_oracle_refs", "gevd", 1, True, ("irm1", "ibm1"), True, 30),
    (512, 1, [1] * 14 + [2], 64, 1, "compressed", "gevd", 1, True, None, False, 140),
    (256, 2, [5], 8, 2, "local", "gevd", 2, True, ("iam1", "irm1"), True, 41),
    (512, 1, [4, 4, 4, 4], 8, 1, "use_oracle_zs", "mwf", 1, True, ("irm2", "irm1"), False, 30),
    (256, 1, [2, 4, 6, 4], 64, 2, "compressed", "r1-mwf", 1, True, ("irm1", "irm1"), True, 140),
    (1024, 1, [1, 2, 3], 8, 1, "use_oracle_zs", "gevd", 1, True, None, True, 26),
    (512, 1, [8, 2], 1, 2, "distant", "gevd", 1, False, None, False, 12),
    (256, 3, [1, 2, 3], 8, 1, "local", "mwf", 1, False, None, False, 33),
    (512, 1, [15, 1], 8, 1, "previous", "gevd", 1, True, ("ibm1", "irm1"), False, 25),
]


def _ids(c):
    return "%d-B%d-%s-P%d-lag%d-%s-%s%d-%s-R0%d" % (c[0], c[1], "x".join(map(str, c[2])), c[3], c[4], c[5], c[6], c[7],
                                                   "clean" if c[8] else "masks", int(c[10]))


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_ragged_stream_equals_whole_signal(dev, case):
    from test_gpu_stream import _schedule
    n_fft, B, channels, P, lag, mode, ftype, rank, clean, vads, with_r0, hops = case
    i = CASES.index(case)
    H, F, K, M = n_fft // 2, n_fft // 2 + 1, len(channels), sum(channels)
    rng = np.random.default_rng(700 + i)
    L = hops * H + int(rng.integers(0, H))
    y, s, n = _inputs(rng, B, M, L, clean, dev)
    mask_fn = None if vads is not None else _masks(rng, B, K, 1 + L // H, F, i % 2 == 0, dev)
    R0 = _r0_nodes(B, channels, F, 40 + i, dev) if with_r0 else None
    ref_mic = min(channels) - 1 if lag == 2 else 0
    kw = dict(lambda_cor=0.95 if i % 3 else 0.5, lag=lag, mu=1.0, rank=rank, ref_mic=ref_mic, R0=R0,
              mask_for_z=mode, filter_type=ftype)
    got, Ws, st = _run(y, s, n, channels, _schedule("random", L, H, P, rng), mask_fn, n_fft=n_fft, block=P, vads=vads,
                       **kw)
    _check_whole(y, s, n, channels, got, Ws, st, P, n_fft, vads, kw)


@pytest.mark.parametrize("mode", ["local", "distant", "previous", "compressed", "use_oracle_refs", "use_oracle_zs"])
def test_ragged_stream_every_mode_and_filter(dev, mode):
    """Every exchange mode x filter type on [1, 2, 3] with clean components: half with the stream's oracle masks,
    half with mask_fn, each against online_tango_ragged."""
    from test_gpu_stream import _schedule
    n_fft, P, channels = 256, 4, [1, 2, 3]
    H, F, K, M = 128, 129, 3, 6
    for j, ftype in enumerate(("gevd", "mwf", "r1-mwf")):
        rng = np.random.default_rng(900 + 10 * j + len(mode))
        L = 18 * H + 5
        y, s, n = _inputs(rng, 1, M, L, True, dev)
        vads = ("irm1", "irm2") if j % 2 == 0 else None
        mask_fn = None if vads is not None else _masks(rng, 1, K, 1 + L // H, F, True, dev)
        kw = dict(lag=1, mask_for_z=mode, filter_type=ftype)
        got, Ws, st = _run(y, s, n, channels, _schedule("random", L, H, P, rng), mask_fn, n_fft=n_fft, block=P,
                           vads=vads, **kw)
        _check_whole(y, s, n, channels, got, Ws, st, P, n_fft, vads, kw)


@pytest.mark.parametrize("C,K,lag,clean", [(4, 4, 1, False), (2, 3, 2, True), (3, 1, 1, True)])
def test_equal_counts_equal_the_int_c_stream(dev, C, K, lag, clean):
    """channels = [C] * K with packed chunks is the int-C stream bit for bit: outputs, mask_fn's Y (a view of the
    int stream's), filters ({C: W}) and nodes."""
    from test_gpu_stream import _schedule
    n_fft, P, B = 512, 8, 2
    H, F = 256, 257
    rng = np.random.default_rng(C * 10 + K)
    L = 35 * H + 17
    y, s, n = _inputs(rng, B, K * C, L, clean, dev)
    mask_fn = _masks(rng, B, K, 1 + L // H, F, True, dev)
    sizes = _schedule("random", L, H, P, rng)
    kw = dict(n_fft=n_fft, block=P, lag=lag, mask_for_z="distant" if K > 1 else "local")
    a, Wa, _ = _run(y, s, n, [C] * K, sizes, mask_fn, **kw)
    four = lambda x: None if x is None else x.view(B, K, C, L)
    b, Wb, st = _run(four(y), four(s), four(n), C, sizes, mask_fn, **kw)
    assert st.nodes == {C: list(range(K))}
    assert a.keys() == b.keys()
    for k in a:
        want = b[k].reshape(a[k].shape) if k == "Y" else b[k]
        assert torch.equal(a[k], want), k
    for (fa, W1a, W2a), (fb, W1b, W2b) in zip(Wa, Wb):
        assert fa == fb
        if W1b is None:
            assert W1a is None and W2a is None
        else:
            assert torch.equal(W1a[C], W1b) and torch.equal(W2a[C], W2b)


# ---------------------------------------------------------------------------------------------- pool slot = lone stream
NAN = float("nan")


class _Slots:
    """Drives a pool of per-node counts through a plan (opens, samples per slot and step, closes) and records, per
    opened stream, its samples, outputs, masks and filters.  Padding, free rows and masks past each run are NaN."""

    def __init__(self, pool, dev, seed, r0_every=0):
        self.pool, self.dev, self.rng = pool, dev, np.random.default_rng(seed)
        self.r0_every, self.cur, self.done, self.count = r0_every, {}, [], 0

    def mask_fn(self, t0, n_fr, Y, z, zn):
        p = self.pool
        S, K, f, F = z.shape
        assert Y.shape == (S, p.M, f, F)
        mz, mw = torch.rand((S, K, f, F), device=self.dev), torch.rand((S, K, f, F), device=self.dev)
        for s in range(S):
            mz[s, :, n_fr[s]:] = NAN
            mw[s, :, n_fr[s]:] = NAN
            if n_fr[s]:
                rec = self.cur[s]
                assert t0[s] == rec["t_next"]
                rec["t_next"] += int(n_fr[s])
                rec["Y"].append(Y[s, :, :n_fr[s]].clone())
                rec["mz"].append(mz[s, :, :n_fr[s]].clone())
                rec["mw"].append(mw[s, :, :n_fr[s]].clone())
        return mz, mw

    def _take(self, out, slots):
        p = self.pool
        for s in slots:
            rec = self.cur[s]
            f, m = int(out["frames"][s]), int(out["samples"][s])
            for k in ("z_y", "zn", "yf"):
                rec[k].append(out[k][s, :, :f].clone())
                assert not out[k][s, :, f:].any()
            rec["yf_time"].append(out["yf_time"][s, :, :m].clone())
            assert not out["yf_time"][s, :, m:].any()
            W = p.filters(s)
            rec["W"].append((int(p.frames_out[s]), None if W is None else (_clone_W(W[0]), _clone_W(W[1]))))

    def open(self, slots):
        if not slots:
            return
        p = self.pool
        R0 = None
        if self.r0_every and self.count % self.r0_every == 0:
            R0 = _r0_nodes(len(slots), p.channels, p.F, self.count, self.dev)
        p.open(slots, R0)
        for i, s in enumerate(slots):
            assert p.is_open(s) and p.filters(s) is None
            r0 = None if R0 is None else [(a[i:i + 1].clone(), b[i:i + 1].clone()) for a, b in R0]
            self.cur[s] = {"y": [], "z_y": [], "zn": [], "yf": [], "yf_time": [], "Y": [], "mz": [], "mw": [],
                           "W": [], "t_next": 0, "R0": r0}
        self.count += 1

    def push(self, n):
        p = self.pool
        y = torch.full((p.S, p.M, max(int(n.max()), 1)), NAN, device=self.dev)
        for s, rec in self.cur.items():
            if n[s]:
                seg = torch.from_numpy(self.rng.standard_normal((p.M, int(n[s]))).astype(np.float32)).to(self.dev)
                y[s, :, :n[s]] = seg
                rec["y"].append(seg)
        self._take(p.push(y, n, self.mask_fn), list(self.cur))

    def close(self, slots):
        if slots:
            self._take(self.pool.close(slots, self.mask_fn), slots)
            for s in slots:
                assert not self.pool.is_open(s)
                self.done.append(self.cur.pop(s))

    def run(self, opens, n, closes):
        for t in range(len(opens)):
            self.open(opens[t])
            self.push(n[t])
            self.close(closes[t])
        assert not self.cur
        return self.done


def _plan(S, P, H, steps, rng):
    """Slot s opens at step s % 3, takes s % block hops and one sample first (every offset within a block), idles
    now and then, and closes; slots that close early reopen two steps later."""
    opens, closes = [[] for _ in range(steps)], [[] for _ in range(steps)]
    nn = np.zeros((steps, S), dtype=np.int64)
    for s in range(S):
        first = s % 3
        while first < steps - 1:
            last = min(steps - 1, first + 1 + s % 3)
            opens[first].append(s)
            nn[first, s] = (s % P) * H + 1 + H
            for t in range(first + 1, last + 1):
                nn[t, s] = int(rng.choice([0, 1, H - 1, P * H, int(rng.integers(1, 3 * P * H))]))
            closes[last].append(s)
            first = last + 2
    return opens, nn, closes


def _check_slot(rec, pool, dev):
    """One closed slot against OnlineTangoStream(1, K, channels) with the pool's options (one push and a flush), and
    against online_tango_ragged on its whole signal."""
    from disco_b200 import ops
    from disco_b200.ragged import online_tango_ragged
    from disco_b200.stream import OnlineTangoStream
    K, P, n_fft, channels = pool.K, pool.block, pool.n_fft, pool.channels
    y = torch.cat(rec["y"], dim=-1)[None]
    L = y.shape[-1]
    mz, mw = torch.cat(rec["mz"], dim=1)[None], torch.cat(rec["mw"], dim=1)[None]
    kw = dict(lambda_cor=pool.lambda_cor, lag=pool.lag, mu=pool.mu, rank=pool.rank, ref_mic=pool.ref_mic,
              filter_type=pool.filter_type, mask_for_z=pool.mask_for_z)
    got = {k: torch.cat(rec[k], dim=1) for k in ("z_y", "zn", "yf", "yf_time", "Y")}
    st = OnlineTangoStream(1, K, channels, n_fft=n_fft, block=P, R0=rec["R0"], device=dev, wide=True, **kw)
    fn = lambda t0, Yv, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]])
    a, b = st.push(y, fn), st.flush(fn)
    for k in ("z_y", "zn", "yf", "yf_time"):
        assert _same(torch.cat((a[k], b[k]), dim=2)[0], got[k]), k
    assert torch.equal(got["Y"], _packed_stft(y, channels, n_fft)[0])
    ref = online_tango_ragged(y, channels, (mz, mw), block=P, n_fft=n_fft, R0=rec["R0"], **kw)
    for k in ("z_y", "zn", "yf"):
        assert _same(got[k], ref[k][0]), k
    assert _same(got["yf_time"], ops.istft(ref["yf"], L, n_fft)[0])
    J = ref["W1"][channels[0]].shape[2]
    for i, (frames, W) in enumerate(rec["W"]):
        closed = frames // P if i + 1 < len(rec["W"]) else J
        if closed == 0:
            assert W is None, i
        else:
            assert _same_dict(W[0], {C: w[0, :, closed - 1] for C, w in ref["W1"].items()}), i
            assert _same_dict(W[1], {C: w[0, :, closed - 1] for C, w in ref["W2"].items()}), i


# (n_fft, channels, block, lag, mask_for_z, filter_type, slots, steps)
POOL_CASES = [
    (256, [2, 4, 6, 4], 4, 1, "distant", "gevd", 5, 7),
    (512, [1, 2, 3], 8, 2, "local", "mwf", 4, 7),
    (256, [8, 2], 8, 1, "previous", "r1-mwf", 4, 6),
    (256, [15, 1], 4, 2, "local", "gevd", 3, 6),
    (256, [1] * 14 + [2], 8, 1, "distant", "gevd", 3, 5),
    (1024, [5], 8, 1, "local", "gevd", 4, 6),
    (512, [4, 4, 4, 4], 1, 1, "previous", "mwf", 3, 6),
]


@pytest.mark.parametrize("case", POOL_CASES, ids=["%d-%s-P%d-lag%d-%s-%s-S%d" % ((c[0], "x".join(map(str, c[1])))
                                                                              + c[2:7]) for c in POOL_CASES])
def test_ragged_pool_slots_equal_lone_streams(dev, case):
    from disco_b200.stream import OnlineTangoPool
    n_fft, channels, P, lag, mode, ftype, S, steps = case
    i = POOL_CASES.index(case)
    pool = OnlineTangoPool(S, len(channels), channels, n_fft=n_fft, lambda_cor=0.9, block=P, lag=lag,
                           ref_mic=min(channels) - 1 if lag == 2 else 0, device=dev, filter_type=ftype,
                           mask_for_z=mode)
    assert pool.nodes == {C: [k for k, c in enumerate(channels) if c == C] for C in sorted(set(channels))}
    rng = np.random.default_rng(60 + i)
    done = _Slots(pool, dev, seed=80 + i, r0_every=2).run(*_plan(S, P, n_fft // 2, steps, rng))
    assert len(done) >= S
    for rec in done:
        _check_slot(rec, pool, dev)


def test_equal_counts_pool_equals_int_c_pool(dev):
    """A pool of channels [3, 3] with packed y equals the int-C pool (K = 2, C = 3) bit for bit."""
    from disco_b200.stream import OnlineTangoPool
    n_fft, P, S, K, C = 256, 4, 3, 2, 3
    H = n_fft // 2
    kw = dict(n_fft=n_fft, block=P, lag=1, device=dev, mask_for_z="distant")
    a, b = OnlineTangoPool(S, K, [C] * K, **kw), OnlineTangoPool(S, K, C, **kw)
    rng = np.random.default_rng(5)
    for p in (a, b):
        p.open([0, 2])
    for step in range(5):
        n = np.array([int(rng.integers(H + 1, 3 * P * H)) for _ in range(S)], dtype=np.int64)
        if step == 0:
            n[1] = 0
        if step == 1:
            for p in (a, b):
                p.open([1])
        y = torch.from_numpy(rng.standard_normal((S, K * C, int(n.max()))).astype(np.float32)).to(dev)
        rounds = []

        def fa(t0, n_fr, Y, z, zn):
            m = (torch.rand(z.shape, device=dev), torch.rand(z.shape, device=dev))
            rounds.append((Y.clone(), m))
            return m

        def fb(t0, n_fr, Y, z, zn):
            Ya, m = rounds.pop(0)
            Y = Y.reshape(Ya.shape)
            for s in range(S):                                  # rows past n_fr[s] are not defined
                assert torch.equal(Ya[s, :, :n_fr[s]], Y[s, :, :n_fr[s]])
            return m
        oa = a.push(y, n, fa) if step < 4 else a.close([0, 1, 2], fa)
        ob = b.push(y.view(S, K, C, -1), n, fb) if step < 4 else b.close([0, 1, 2], fb)
        assert not rounds
        for k in ("z_y", "zn", "yf", "yf_time"):
            assert torch.equal(oa[k], ob[k]), (step, k)
        for s in range(S):
            Wa, Wb = a.filters(s), b.filters(s)
            assert (Wa is None) == (Wb is None)
            if Wb is not None:
                assert torch.equal(Wa[0][C], Wb[0]) and torch.equal(Wa[1][C], Wb[1])


def test_ragged_errors_on_the_device(dev):
    """Rejected calls leave the stream and pool as they were; an exception inside push closes the stream, and the
    pool closes only the slots the call advanced."""
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    ch = [1, 2, 3]
    F = 257
    ok = lambda t0, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), None)
    st = OnlineTangoStream(2, 3, ch, device=dev)
    y = torch.zeros(2, 6, 700, device=dev)
    with pytest.raises(ValueError, match="expected"):
        st.push(torch.zeros(2, 3, 2, 700, device=dev), ok)          # the int layout
    with pytest.raises(ValueError, match="expected"):
        st.push(torch.zeros(2, 5, 700, device=dev), ok)             # M = 6
    assert not st.closed and st.samples_in == 0
    out = st.push(y, ok)
    assert out["yf"].shape == (2, 3, 2, F) and out["yf_time"].shape == (2, 3, 256)
    with pytest.raises(ValueError, match="shape"):
        st.push(y, lambda t0, Y, z, zn: (torch.zeros(2, 3, 1, F, device=dev), None))
    assert st.closed
    pool = OnlineTangoPool(3, 3, ch, device=dev)
    pool.open([0, 1])
    pfn = lambda t0, n_fr, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), None)
    pool.push(torch.zeros(3, 6, 600, device=dev), np.array([600, 600, 0]), pfn)
    with pytest.raises(ValueError):
        pool.push(torch.zeros(3, 2, 3, 600, device=dev), np.array([600, 0, 0]), pfn)
    assert pool.is_open(0) and pool.is_open(1)
    bad = lambda t0, n_fr, Y, z, zn: (torch.zeros(1, device=dev), None)
    with pytest.raises(ValueError, match="shape"):
        pool.push(torch.zeros(3, 6, 600, device=dev), np.array([600, 0, 0]), bad)
    assert not pool.is_open(0) and pool.is_open(1)
    pool.close([1], pfn)
