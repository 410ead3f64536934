"""The options of the online Tango stream and pool (disco_b200/stream.py) against the whole-signal run: channel stacks
D = 9..16, the exchange modes (mask_for_z), the filter types, and (stream only) the clean components with the oracle
masks and the diagnostic outputs.  Whatever the chunking, the stream's outputs concatenated equal online_tango on the
whole signal with the same options, and its time samples ops.istft / post.to_time of that run, bit for bit; the pool's
slots equal lone streams with the same options."""
import numpy as np
import pytest
import torch

from test_gpu_stream import _r0, _schedule
from test_gpu_stream_pool import _Streams

pytestmark = pytest.mark.gpu

CLEAN_NAMES = ("z_s", "z_n", "sf", "nf")
TIME_NAMES = ("yf", "z_y", "sf", "nf", "z_s", "z_n")


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


def _hermitian(R):
    """The carried matrices: Hermitian (the mirror of the upper triangle) with a real diagonal, all the wide scan
    reads of R0."""
    return torch.equal(R, R.conj().transpose(-1, -2)) and not R.diagonal(dim1=-2, dim2=-1).imag.any()


def _run(y, s, n, sizes, mask_fn, **kw):
    """Push y (and s, n) in chunks of `sizes`, then flush; returns the concatenated outputs, the masks mask_fn
    returned, the filters after every call, and whether the carried matrices stayed Hermitian."""
    from disco_b200.stream import OnlineTangoStream
    B, K, C, L = y.shape
    st = OnlineTangoStream(B, K, C, device=y.device, clean=s is not None, wide=True, **kw)
    got, masks, Ws = {}, {"mz": [], "mw": []}, []
    herm = []

    def fn(t0, Y, z, zn):
        assert t0 == sum(m.shape[2] for m in masks["mz"])
        mz, mw = mask_fn(t0, Y, z, zn)
        masks["mz"].append(mz.clone())
        masks["mw"].append((mz if mw is None else mw).clone())
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
        Ws.append((st.frames_out, None if st.W1 is None else st.W1.clone(), None if st.W2 is None else st.W2.clone()))
        for R in (st._R1, st._R2) if st.W1 is not None else ():    # carried from a closed block, not the given R0
            if R[0].shape[-1] >= 9:
                herm.append(_hermitian(R[0]) and _hermitian(R[1]))
    assert st.samples_in == L and st.samples_out == L and st.closed
    cat = {k: torch.cat(v, dim=2) for k, v in got.items()}
    if masks["mz"]:
        cat["mz"], cat["mw"] = torch.cat(masks["mz"], dim=2), torch.cat(masks["mw"], dim=2)
    return cat, Ws, herm


def _check(y, s, n, got, Ws, block, n_fft, vads, kw):
    from disco_b200 import ops, post
    from disco_b200.online import online_tango
    L = y.shape[-1]
    clean = s is not None
    extra = dict(s=s, n=n) if clean else {}
    if vads is not None:
        ref = online_tango(y, None, block=block, n_fft=n_fft, vads=vads, **extra, **kw)
        assert _same(got["masks_z"], ref["masks_z"]) and _same(got["mask_w"], ref["mask_w"])
    else:
        ref = online_tango(y, (got["mz"], got["mw"]), block=block, n_fft=n_fft, **extra, **kw)
    T = ops.n_frames(L, n_fft)
    assert got["yf"].shape[2] == T
    for k in ("z_y", "zn", "yf") + (CLEAN_NAMES if clean else ()):
        assert _same(got[k], ref[k]), k
    if clean:
        want = post.to_time(ref, L, n_fft, layout="TF")
        for k in TIME_NAMES:
            assert got[k + "_time"].shape[-1] == L
            assert _same(got[k + "_time"], want[k]), k + "_time"
    else:
        assert _same(got["yf_time"], ops.istft(ref["yf"], L, n_fft))
    J = ref["W1"].shape[2]
    for i, (frames, W1, W2) in enumerate(Ws):
        closed = frames // block if i + 1 < len(Ws) else J
        if closed == 0:
            assert W1 is None and W2 is None
        else:
            assert _same(W1, ref["W1"][:, :, closed - 1]) and _same(W2, ref["W2"][:, :, closed - 1]), i
    return ref


# (n_fft, B, K, C, block, lag, mask_for_z, filter_type, rank, clean, vads, R0, hops, schedule)
CASES = [
    (256, 1, 8, 2, 8, 1, "local", "gevd", 1, False, None, False, 40, "random"),
    (512, 1, 8, 2, 1, 2, "distant", "mwf", 1, True, ("irm1", "irm1"), False, 14, "random"),
    (1024, 1, 4, 6, 8, 1, "previous", "r1-mwf", 1, False, None, False, 30, "H-1"),
    (256, 2, 1, 9, 64, 2, "local", "gevd", 2, False, None, True, 150, "random"),
    (512, 1, 2, 15, 8, 1, "compressed", "gevd", 1, True, None, False, 36, "random"),
    (256, 1, 1, 16, 8, 2, "use_oracle_refs", "mwf", 1, True, ("irm1", "ibm1"), True, 30, "H+1"),
    (512, 1, 4, 4, 64, 1, "use_oracle_zs", "gevd", 1, True, ("irm2", "irm1"), False, 140, "3PH+7"),
    (1024, 1, 4, 4, 1, 1, "distant", "r1-mwf", 1, True, None, False, 12, "random"),
    (256, 1, 4, 4, 8, 2, "local", "gevd", 1, True, ("iam1", "irm1"), False, 41, "random"),
    (512, 1, 1, 9, 8, 1, "distant", "gevd", 1, False, None, True, 33, "PH"),
    (256, 1, 8, 2, 64, 1, "use_oracle_zs", "r1-mwf", 1, True, ("irm1", "irm1"), False, 140, "random"),
    (512, 1, 2, 15, 1, 2, "previous", "mwf", 1, True, ("ibm1", "irm1"), False, 10, "random"),
    (1024, 1, 1, 16, 8, 2, "compressed", "gevd", 2, True, ("irm1", "irm1"), True, 26, "random"),
    (256, 1, 4, 6, 8, 1, "use_oracle_refs", "gevd", 1, True, None, False, 30, "random"),
    (512, 2, 4, 4, 8, 1, "local", "mwf", 1, False, None, False, 25, "random"),
    (256, 1, 1, 4, 8, 2, "distant", "gevd", 1, True, ("irm1", "irm1"), True, 27, "random"),
    (512, 1, 8, 2, 8, 2, "previous", "gevd", 1, True, ("irm1", "irm1"), False, 30, "random"),
    (1024, 1, 2, 15, 64, 1, "local", "gevd", 1, False, None, False, 70, "random"),
]


def _ids(c):
    return "%d-%dx%dx%d-P%d-lag%d-%s-%s%s-%s-R0%d-%s" % (c[0], c[1], c[2], c[3], c[4], c[5], c[6], c[7], c[8],
                                                         "clean" if c[9] else "masks", int(c[11]), c[13])


@pytest.mark.parametrize("case", CASES, ids=[_ids(c) for c in CASES])
def test_stream_options_equal_whole_signal(dev, case):
    n_fft, B, K, C, P, lag, mode, ftype, rank, clean, vads, with_r0, hops, sched = case
    i = CASES.index(case)
    H, F = n_fft // 2, n_fft // 2 + 1
    rng = np.random.default_rng(300 + i)
    L = hops * H + int(rng.integers(0, H))
    T = 1 + L // H
    s = n = None
    if clean:
        s = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
        n = torch.from_numpy(0.5 * rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
        y = s + n
    else:
        y = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
    mask_fn = None
    if vads is None:
        mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        two = i % 2 == 0
        mask_fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]] if two else None)
    R0 = _r0(B, K, C, F, L, dev) if with_r0 else None
    kw = dict(lambda_cor=0.95 if i % 3 else 0.5, lag=lag, mu=1.0, rank=rank, ref_mic=C - 1 if lag == 2 else 0,
              R0=R0, mask_for_z=mode, filter_type=ftype)
    got, Ws, herm = _run(y, s, n, _schedule(sched, L, H, P, rng), mask_fn, n_fft=n_fft, block=P, vads=vads, **kw)
    assert all(herm)
    if C + K - 1 >= 9:
        assert herm                                      # the carried wide matrices were checked
    _check(y, s, n, got, Ws, P, n_fft, vads, kw)


def test_stream_options_change_the_result(dev):
    """Each option reaches the computation: every exchange mode and filter type moves yf away from the default."""
    n_fft, B, K, C, P = 256, 1, 4, 4, 8
    rng = np.random.default_rng(9)
    L = 40 * 128 + 5
    s = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
    n = torch.from_numpy(0.5 * rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
    y = s + n
    runs = {}
    for mode, ftype in (("local", "gevd"), ("distant", "gevd"), ("previous", "gevd"), ("compressed", "gevd"),
                        ("use_oracle_refs", "gevd"), ("use_oracle_zs", "gevd"), ("local", "mwf"),
                        ("local", "r1-mwf")):
        kw = dict(mask_for_z=mode, filter_type=ftype)
        got, Ws, _ = _run(y, s, n, _schedule("random", L, 128, P, rng), None, n_fft=n_fft, block=P,
                          vads=("irm1", "irm1"), **kw)
        _check(y, s, n, got, Ws, P, n_fft, ("irm1", "irm1"), kw)
        runs[(mode, ftype)] = got["yf"]
    base = runs[("local", "gevd")]
    for key, yf in runs.items():
        if key != ("local", "gevd"):
            assert float((yf - base).abs().max()) > 1e-3 * float(base.abs().max()), key


def _slot_check(rec, pool, dev):
    """One closed slot against OnlineTangoStream(1, K, C) with the pool's options, fed its samples in one push, and
    against online_tango on its whole signal."""
    from disco_b200 import ops
    from disco_b200.online import online_tango
    from disco_b200.stream import OnlineTangoStream
    K, C, P, n_fft = pool.K, pool.C, pool.block, pool.n_fft
    y = torch.cat(rec["y"], dim=-1)[None]
    L = y.shape[-1]
    mz, mw = torch.cat(rec["mz"], dim=1)[None], torch.cat(rec["mw"], dim=1)[None]
    kw = dict(lambda_cor=pool.lambda_cor, lag=pool.lag, mu=pool.mu, rank=pool.rank, ref_mic=pool.ref_mic,
              filter_type=pool.filter_type, mask_for_z=pool.mask_for_z)
    got = {k: torch.cat(rec[k], dim=1) for k in ("z_y", "zn", "yf", "yf_time")}
    st = OnlineTangoStream(1, K, C, n_fft=n_fft, block=P, R0=rec["R0"], device=dev, wide=True, **kw)
    fn = lambda t0, Yv, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]])
    a, b = st.push(y, fn), st.flush(fn)
    for k in ("z_y", "zn", "yf", "yf_time"):
        assert _same(torch.cat((a[k], b[k]), dim=2)[0], got[k]), k
    ref = online_tango(y, (mz, mw), block=P, n_fft=n_fft, R0=rec["R0"], **kw)
    for k in ("z_y", "zn", "yf"):
        assert _same(got[k], ref[k][0]), k
    assert _same(got["yf_time"], ops.istft(ref["yf"], L, n_fft)[0])
    J = ref["W1"].shape[2]
    for i, (frames, W) in enumerate(rec["W"]):
        closed = frames // P if i + 1 < len(rec["W"]) else J
        if closed:
            assert _same(W[0], ref["W1"][0, :, closed - 1]) and _same(W[1], ref["W2"][0, :, closed - 1]), i


# (n_fft, K, C, block, lag, mask_for_z, filter_type)
POOL_CASES = [
    (256, 8, 2, 8, 1, "distant", "gevd"),
    (512, 1, 16, 4, 2, "previous", "mwf"),
    (256, 2, 15, 8, 1, "distant", "r1-mwf"),
    (256, 8, 2, 4, 2, "local", "mwf"),
    (512, 3, 2, 8, 1, "previous", "gevd"),
]


@pytest.mark.parametrize("case", POOL_CASES, ids=["%d-%dx%d-P%d-lag%d-%s-%s" % c for c in POOL_CASES])
def test_pool_options_equal_lone_streams(dev, case):
    """Slot s opens at step s % 2 and first takes s % block hops and one sample, so the slots stand at every offset
    within a block; they close at different steps, R0 on every other open."""
    from disco_b200.stream import OnlineTangoPool
    n_fft, K, C, P, lag, mode, ftype = case
    H, S, steps = n_fft // 2, P, 6
    pool = OnlineTangoPool(S, K, C, n_fft=n_fft, lambda_cor=0.9, block=P, lag=lag, ref_mic=C - 1 if lag == 2 else 0,
                           device=dev, filter_type=ftype, mask_for_z=mode)
    rng = np.random.default_rng(POOL_CASES.index(case))
    opens, closes = [[] for _ in range(steps)], [[] for _ in range(steps)]
    nn = np.zeros((steps, S), dtype=np.int64)
    for s in range(S):
        first, last = s % 2, min(steps - 1, 2 + s % 2 + s % 3)
        opens[first].append(s)
        nn[first, s] = (s % P) * H + 1 + H
        for t in range(first + 1, last + 1):
            nn[t, s] = int(rng.choice([0, 1, H - 1, P * H, int(rng.integers(1, 3 * P * H))]))
        closes[last].append(s)
    done = _Streams(pool, dev, seed=50 + POOL_CASES.index(case), r0_every=2).run((opens, nn, closes))
    assert len(done) == S
    for rec in done:
        _slot_check(rec, pool, dev)


def test_stream_wide_and_push_errors(dev):
    """D = 9..16 only with wide=True, 17 never; the mask-source and clean-component checks of a push are raised before
    any device work, and the stream stays open."""
    from disco_b200.stream import OnlineTangoStream
    F = 257
    with pytest.raises(NotImplementedError, match="wide=True"):
        OnlineTangoStream(1, 2, 8, device=dev)                     # D = 9 without the opt-in
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(1, 2, 16, device=dev, wide=True)         # D = 17
    OnlineTangoStream(1, 2, 8, device=dev, wide=True)              # D = 9 and
    OnlineTangoStream(1, 1, 16, device=dev, wide=True)             # D = 16 run
    ok = lambda t0, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), None)
    # the mask source and the clean components
    y = torch.zeros(1, 8, 2, 600, device=dev)
    s = OnlineTangoStream(1, 8, 2, device=dev, wide=True)
    s.push(y[..., :100])                                           # no frame completes: no mask_fn needed
    with pytest.raises(ValueError, match="mask_fn"):
        s.push(y)
    with pytest.raises(ValueError, match="clean=True"):
        s.push(y, ok, s_chunk=y, n_chunk=y)
    s.push(y[..., 100:], ok)
    with pytest.raises(ValueError, match="mask_fn"):
        s.flush()
    assert not s.closed and s.samples_in == 600
    s.flush(ok)
    s = OnlineTangoStream(1, 8, 2, device=dev, vads=("irm1", "irm1"), wide=True)
    assert s.clean
    with pytest.raises(ValueError, match="vads"):
        s.push(y, ok, s_chunk=y, n_chunk=y)
    with pytest.raises(ValueError, match="s_chunk and n_chunk"):
        s.push(y, s_chunk=y)                                       # s without n
    with pytest.raises(ValueError, match="s_chunk and n_chunk"):
        s.push(y)
    with pytest.raises(ValueError):
        s.push(y, s_chunk=y, n_chunk=y[..., :599])
    with pytest.raises(TypeError):
        s.push(y, s_chunk=y.cpu(), n_chunk=y)
    with pytest.raises(TypeError):
        s.push(y, s_chunk=y, n_chunk=y.double())
    assert not s.closed and s.samples_in == 0
    out = s.push(y, s_chunk=y, n_chunk=y)
    assert out["masks_z"].shape == (1, 8, 2, F) and set(k + "_time" for k in TIME_NAMES) <= set(out)
    with pytest.raises(ValueError, match="vads"):
        s.flush(ok)
    assert not s.closed
    s.flush()
    assert s.closed
