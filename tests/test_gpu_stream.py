"""The online Tango stream (disco_b200/stream.py, csrc/stream.cu) against the whole-signal run: whatever the chunk
sizes, its outputs equal online_tango + ops.istft on the whole signal value for value (torch.equal), with the masks
its mask_fn returned; the spectra handed to mask_fn equal ops.stft; the filters after block j equal online_tango's
W1[:, :, j], W2[:, :, j]."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CFGS = [(3, 1, 4), (1, 1, 3), (3, 1, 3), (2, 3, 2), (1, 4, 2), (1, 1, 8)]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _schedule(kind, L, H, P, rng):
    """Chunk sizes summing to L."""
    if kind == "whole":
        return [L]
    step = {"ones": 1, "H-1": H - 1, "H": H, "H+1": H + 1, "PH": P * H, "3PH+7": 3 * P * H + 7}.get(kind)
    if step is not None:
        return [step] * (L // step) + ([L % step] if L % step else [])
    sizes, left = [], L                       # "random": seeded sizes up to a few blocks, zeros included
    while left > 0:
        n = 0 if rng.random() < 0.15 else int(rng.integers(1, 2 * P * H + 3 * H))
        n = min(n, left)
        sizes.append(n)
        left -= n
    return [0] + sizes[:2] + [0] + sizes[2:] + [0]


def _r0(B, K, C, F, seed, dev):
    rng = np.random.default_rng(seed)
    A = (rng.standard_normal((B, K, F, C, C)) + 1j * rng.standard_normal((B, K, F, C, C))).astype(np.complex64)
    R = A @ A.conj().transpose(0, 1, 2, 4, 3) * 0.01 + 0.001 * np.eye(C, dtype=np.complex64)
    Rn = A.conj() @ A.transpose(0, 1, 2, 4, 3) * 0.02 + 0.002 * np.eye(C, dtype=np.complex64)
    return torch.from_numpy(R.astype(np.complex64)).to(dev), torch.from_numpy(Rn.astype(np.complex64)).to(dev)


def _run(y, mask_fn, sizes, **kw):
    """Push y [B, K, C, L] in chunks of `sizes`, then flush; returns the concatenated outputs, the Y and masks
    mask_fn saw and returned, and the filters after every push."""
    from disco_b200.stream import OnlineTangoStream
    B, K, C, L = y.shape
    s = OnlineTangoStream(B, K, C, **kw)
    got = {"z_y": [], "zn": [], "yf": [], "yf_time": [], "Y": [], "mz": [], "mw": [], "W": []}

    def fn(t0, Y, z, zn):
        assert t0 == sum(m.shape[2] for m in got["mz"])        # runs follow each other
        mz, mw = mask_fn(t0, Y, z, zn)
        got["Y"].append(Y.clone())
        got["mz"].append(mz.clone())
        got["mw"].append((mz if mw is None else mw).clone())
        return mz, mw

    pos = 0
    for n in sizes + [None]:
        if n is None:
            out = s.flush(fn)
        else:
            out = s.push(y[..., pos:pos + n], fn)
            pos += n
        assert out["t0"] == sum(z.shape[2] for z in got["z_y"])
        for k in ("z_y", "zn", "yf", "yf_time"):
            got[k].append(out[k])
        got["W"].append((s.frames_out, None if s.W1 is None else s.W1.clone(), None if s.W2 is None else s.W2.clone()))
    assert s.samples_in == L and s.samples_out == L and s.closed
    cat = {k: torch.cat(got[k], dim=3 if k == "Y" else 2) for k in ("z_y", "zn", "yf", "Y", "mz", "mw")}
    cat["yf_time"] = torch.cat(got["yf_time"], dim=2)
    cat["W"] = got["W"]
    return cat


def _check(y, got, n_fft, block, R0=None, **kw):
    from disco_b200 import ops
    from disco_b200.online import online_tango
    L = y.shape[-1]
    ref = online_tango(y, (got["mz"], got["mw"]), block=block, n_fft=n_fft, R0=R0, **kw)
    assert ref["W1"].shape[2] == (ops.n_frames(L, n_fft) + block - 1) // block
    T = ops.n_frames(L, n_fft)
    assert got["yf"].shape[2] == T
    assert torch.equal(got["Y"], ops.stft(y, n_fft))
    for k in ("z_y", "zn", "yf"):
        assert torch.equal(got[k], ref[k]), k
    assert torch.equal(got["yf_time"], ops.istft(ref["yf"], L, n_fft))
    J = ref["W1"].shape[2]
    for i, (frames, W1, W2) in enumerate(got["W"]):
        closed = frames // block if i + 1 < len(got["W"]) else J       # blocks whose masks are all in
        if closed == 0:
            assert W1 is None and W2 is None
        else:
            assert torch.equal(W1, ref["W1"][:, :, closed - 1]) and torch.equal(W2, ref["W2"][:, :, closed - 1]), i


# (n_fft, (B, K, C), block, lag, lambda, R0 given, hops, offset in the hop (None: H + 1 samples), schedule)
CASES = [
    (256, CFGS[0], 8, 1, 0.95, False, 40, 0, "whole"),
    (256, CFGS[1], 8, 1, 0.95, True, None, None, "whole"),
    (256, CFGS[1], 1, 2, 0.5, False, 3, 1, "ones"),
    (512, CFGS[2], 8, 2, 0.95, True, 30, 128, "H-1"),
    (512, CFGS[3], 8, 1, 0.5, False, 41, 255, "H"),
    (1024, CFGS[4], 1, 1, 0.95, True, 12, 0, "H+1"),
    (512, CFGS[5], 64, 1, 0.95, False, 200, 17, "PH"),
    (256, CFGS[3], 64, 2, 0.5, True, 230, 1, "3PH+7"),
    (1024, CFGS[0], 8, 2, 0.95, False, 50, 511, "random"),
    (256, CFGS[2], 1, 1, 0.95, False, 30, 127, "random"),
    (512, CFGS[4], 64, 2, 0.95, True, 140, 64, "random"),
    (1024, CFGS[5], 8, 1, 0.5, True, 27, 300, "3PH+7"),
    (256, CFGS[5], 1, 1, 0.95, True, 2, 1, "ones"),
    (1024, CFGS[1], 64, 1, 0.5, False, 70, 0, "H"),
    (512, CFGS[0], 1, 2, 0.95, False, 25, 1, "PH"),
    (1024, CFGS[2], 8, 1, 0.95, True, None, None, "ones"),
    (256, CFGS[4], 8, 2, 0.5, False, 33, 64, "H-1"),
    (512, CFGS[1], 8, 1, 0.95, False, 9, 200, "H+1"),
]


@pytest.mark.parametrize("case", CASES, ids=["%d-%dx%dx%d-P%d-lag%d-lam%s-R0%d-%s-%s" % (
    c[0], *c[1], c[2], c[3], c[4], c[5], "H+1" if c[6] is None else "%dh+%d" % (c[6], c[7]), c[8]) for c in CASES])
def test_stream_equals_whole_signal(dev, case):
    n_fft, (B, K, C), P, lag, lam, with_r0, hops, off, sched = case
    H, F = n_fft // 2, n_fft // 2 + 1
    L = H + 1 if hops is None else hops * H + off
    i = CASES.index(case)
    rng = np.random.default_rng(100 + i)
    y = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
    T = 1 + L // H
    mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
    mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
    two = i % 2 == 0                # every other case: mask_w = None (the step-2 mask is mask_z)
    mask_fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]] if two else None)
    R0 = _r0(B, K, C, F, L, dev) if with_r0 else None
    kw = dict(lambda_cor=lam, lag=lag, mu=1.0, rank=1, ref_mic=C - 1 if lag == 2 else 0)
    got = _run(y, mask_fn, _schedule(sched, L, H, P, rng), n_fft=n_fft, block=P, R0=R0, **kw)
    assert torch.equal(got["mz"], mz) and torch.equal(got["mw"], mw if two else mz)
    _check(y, got, n_fft, P, R0=R0, **kw)


@pytest.mark.parametrize("n_fft,BKC", [(512, (2, 1, 4)), (256, (1, 3, 2))])
def test_stream_causal_masks(dev, n_fft, BKC):
    """A causal estimator: an irm-like ratio of |Y_ref| and |zn| of the frames just analysed.  online_tango on the
    whole signal with the masks it returned reproduces the stream."""
    B, K, C = BKC
    H, L, P = n_fft // 2, 37 * (n_fft // 2) + 5, 4
    rng = np.random.default_rng(5)
    y = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)

    def irm(t0, Y, z, zn):
        a, b = Y[:, :, 0].abs(), zn.abs()
        return a / (a + b + 1e-3), (a * a) / (a * a + b * b + 1e-6)

    got = _run(y, irm, _schedule("random", L, H, P, rng), n_fft=n_fft, block=P, lag=1, lambda_cor=0.9)
    assert float(got["mz"].std()) > 0.01        # the masks follow the signal
    _check(y, got, n_fft, P, lambda_cor=0.9, lag=1)


def test_stream_errors(dev):
    from disco_b200.stream import OnlineTangoStream
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(1, 2, 8, device=dev)
    with pytest.raises(NotImplementedError):
        OnlineTangoStream(1, 1, 4, lag=0, device=dev)
    with pytest.raises(ValueError):
        OnlineTangoStream(1, 1, 4, n_fft=300, device=dev)
    with pytest.raises(ValueError):
        OnlineTangoStream(1, 1, 4, block=65, device=dev)
    with pytest.raises(ValueError):
        OnlineTangoStream(1, 1, 4, lambda_cor=1.0, device=dev)
    F = 257
    ok = lambda t0, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), None)
    s = OnlineTangoStream(1, 1, 4, device=dev)
    with pytest.raises(TypeError):
        s.push(torch.zeros(1, 1, 4, 100), ok)                      # CPU tensor
    with pytest.raises(TypeError):
        s.push(torch.zeros(1, 1, 4, 100, dtype=torch.float64, device=dev), ok)
    with pytest.raises(ValueError):
        s.push(torch.zeros(1, 2, 4, 100, device=dev), ok)
    s.push(torch.zeros(1, 1, 4, 256, device=dev), ok)
    with pytest.raises(ValueError):
        s.flush(ok)                                                # 256 samples = n_fft / 2: too short
    assert not s.closed
    s.push(torch.zeros(1, 1, 4, 1000, device=dev), ok)
    s.flush(ok)
    with pytest.raises(RuntimeError):
        s.push(torch.zeros(1, 1, 4, 10, device=dev), ok)
    with pytest.raises(RuntimeError):
        s.flush(ok)
    s = OnlineTangoStream(1, 1, 4, device=dev)
    with pytest.raises(ValueError):
        s.push(torch.zeros(1, 1, 4, 600, device=dev), lambda t0, Y, z, zn: (torch.zeros(1, 1, 1, F, device=dev), None))
    assert s.closed
    s = OnlineTangoStream(1, 1, 4, device=dev)
    with pytest.raises(ValueError):
        s.push(torch.zeros(1, 1, 4, 600, device=dev), lambda t0, Y, z, zn: (torch.zeros(z.shape, device=dev),
                                                                            torch.zeros(1, 1, 2, 3, device=dev)))
