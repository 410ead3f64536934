"""The pool of independent online Tango streams (disco_b200/stream.py OnlineTangoPool, csrc/stream.cu and istft.cu per-slot
kernels).  Every slot's outputs, concatenated from open to close, equal (torch.equal) online_tango on the slot's whole
signal with B = 1 plus ops.istft of its yf, and OnlineTangoStream(1, K, C) fed the signal in one push where that
covers D; the filters match after every call.  Slots open, push, idle and close on schedules of their own, next to
NaN in the padding of y, in the rows of free slots and in the masks past each slot's frames.  The per-slot kernels are
also checked through the C ABI against the single-stream entry points slot by slot, inside NaN guard bands."""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
PATTERN = 0x7FC0DEAD        # a NaN with a payload: guard words must keep it bit for bit

# kernel edges: per n_fft, the frames of one warp job (NB = 32 / (n_fft / 32)) and of one CTA (4 jobs); the table
# that tests/test_stream_pool_cpu.py holds against the dispatch sets of the per-slot launchers
SLOT_NFFTS = (256, 512, 1024)
JOB_FRAMES = {256: 4, 512: 2, 1024: 1}
CTA_FRAMES = {n: 4 * f for n, f in JOB_FRAMES.items()}


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _r0(n, K, C, F, seed, dev):
    rng = np.random.default_rng(seed)
    A = (rng.standard_normal((n, K, F, C, C)) + 1j * rng.standard_normal((n, K, F, C, C))).astype(np.complex64)
    R = A @ A.conj().transpose(0, 1, 2, 4, 3) * 0.01 + 0.001 * np.eye(C, dtype=np.complex64)
    Rn = A.conj() @ A.transpose(0, 1, 2, 4, 3) * 0.02 + 0.002 * np.eye(C, dtype=np.complex64)
    return torch.from_numpy(R.astype(np.complex64)).to(dev), torch.from_numpy(Rn.astype(np.complex64)).to(dev)


def _size(kind, H, P, rng):
    if kind == "rand":
        return int(rng.integers(1, 3 * P * H))
    return {"0": 0, "1": 1, "H-1": H - 1, "H": H, "H+1": H + 1, "PH": P * H}[kind]


def _plan(S, steps, H, P, seed):
    """Per step: (slots to open, n per slot, slots to close).  Slot s first opens at step s % 3, pushes sizes of every
    kind, closes after 2 to 5 steps, sits idle 0 or 1 step and opens again; everything closes at the last step."""
    rng = np.random.default_rng(seed)
    kinds = ["0", "1", "H-1", "H", "H+1", "PH", "rand", "rand"]
    opens, closes = [[] for _ in range(steps)], [[] for _ in range(steps)]
    n = np.zeros((steps, S), dtype=np.int64)
    for s in range(S):
        c = s % 3
        while c < steps:
            end = min(steps - 1, c + int(rng.integers(2, 6)))
            opens[c].append(s)
            L = 0
            for t in range(c, end + 1):
                n[t, s] = _size(kinds[int(rng.integers(len(kinds)))], H, P, rng)
                if t == end:
                    n[t, s] = max(n[t, s], H + 1 - L)
                L += n[t, s]
            closes[end].append(s)
            c = end + 1 + int(rng.integers(0, 2))
    return opens, n, closes


class _Streams:
    """Drives a pool through a plan and collects, per opened stream, its samples, outputs, masks and filters."""

    def __init__(self, pool, dev, seed, r0_every=0):
        self.pool, self.dev, self.rng = pool, dev, np.random.default_rng(seed)
        self.r0_every = r0_every
        self.cur = {}           # slot -> stream record
        self.done = []
        self.count = 0

    def mask_fn(self, t0, n_fr, Y, z, zn):
        S, K, f, F = z.shape
        mz = torch.rand((S, K, f, F), device=self.dev)
        mw = torch.rand((S, K, f, F), device=self.dev)
        for s in range(S):
            mz[s, :, n_fr[s]:] = NAN                       # never read
            mw[s, :, n_fr[s]:] = NAN
            if n_fr[s]:
                rec = self.cur[s]
                assert t0[s] == rec["t_next"]
                rec["t_next"] += int(n_fr[s])
                rec["mz"].append(mz[s, :, :n_fr[s]].clone())
                rec["mw"].append(mw[s, :, :n_fr[s]].clone())
        return mz, mw

    def _take(self, out, slots):
        p = self.pool
        for s in slots:
            rec = self.cur[s]
            f, m = int(out["frames"][s]), int(out["samples"][s])
            assert out["t0"][s] == sum(z.shape[1] for z in rec["z_y"]) and out["s0"][s] == rec["s_out"]
            for k in ("z_y", "zn", "yf"):
                rec[k].append(out[k][s, :, :f].clone())
                assert not out[k][s, :, f:].any()                      # exactly 0 past the slot's frames
            rec["yf_time"].append(out["yf_time"][s, :, :m].clone())
            assert not out["yf_time"][s, :, m:].any()
            rec["s_out"] += m
            W = p.filters(s)
            rec["W"].append((int(p.frames_out[s]), None if W is None else (W[0].clone(), W[1].clone())))

    def open(self, slots):
        if not slots:
            return
        p = self.pool
        R0 = None
        if self.r0_every and self.count % self.r0_every == 0:
            R0 = _r0(len(slots), p.K, p.C, p.F, self.count, self.dev)
        p.open(slots, R0)
        for i, s in enumerate(slots):
            assert p.is_open(s) and p.filters(s) is None
            self.cur[s] = {"y": [], "z_y": [], "zn": [], "yf": [], "yf_time": [], "mz": [], "mw": [], "W": [],
                           "t_next": 0, "s_out": 0, "slot": s,
                           "R0": None if R0 is None else (R0[0][i:i + 1].clone(), R0[1][i:i + 1].clone())}
        self.count += 1

    def push(self, n):
        p = self.pool
        n_max = max(int(n.max()), 1)
        y = torch.full((p.S, p.K, p.C, n_max), NAN, device=self.dev)     # padding and free rows: NaN
        for s, rec in self.cur.items():
            if n[s]:
                seg = torch.from_numpy(self.rng.standard_normal((p.K, p.C, int(n[s]))).astype(np.float32)).to(self.dev)
                y[s, :, :, :n[s]] = seg
                rec["y"].append(seg)
        out = p.push(y, n, self.mask_fn)
        self._take(out, list(self.cur))

    def close(self, slots):
        if not slots:
            return
        out = self.pool.close(slots, self.mask_fn)
        self._take(out, slots)
        for s in slots:
            assert not self.pool.is_open(s)
            self.done.append(self.cur.pop(s))

    def run(self, plan):
        opens, n, closes = plan
        for t in range(len(opens)):
            self.open(opens[t])
            self.push(n[t])
            self.close(closes[t])
        assert not self.cur
        return self.done


def _check_stream(rec, pool):
    """One closed stream against the whole-signal run (and the lockstep stream where it covers D)."""
    from disco_b200 import ops
    from disco_b200.online import online_tango
    from disco_b200.stream import OnlineTangoStream
    K, C, P, n_fft = pool.K, pool.C, pool.block, pool.n_fft
    y = torch.cat(rec["y"], dim=-1)[None]
    L = y.shape[-1]
    mz, mw = torch.cat(rec["mz"], dim=1)[None], torch.cat(rec["mw"], dim=1)[None]
    kw = dict(lambda_cor=pool.lambda_cor, lag=pool.lag, mu=pool.mu, rank=pool.rank, ref_mic=pool.ref_mic)
    ref = online_tango(y, (mz, mw), block=P, n_fft=n_fft, R0=rec["R0"], **kw)
    T = ops.n_frames(L, n_fft)
    got = {k: torch.cat(rec[k], dim=1) for k in ("z_y", "zn", "yf", "yf_time")}
    assert got["yf"].shape[1] == T and got["yf_time"].shape[1] == L
    for k in ("z_y", "zn", "yf"):
        assert torch.equal(got[k], ref[k][0]), k
    assert torch.equal(got["yf_time"], ops.istft(ref["yf"], L, n_fft)[0])
    J = ref["W1"].shape[2]
    for i, (frames, W) in enumerate(rec["W"]):
        closed = frames // P if i + 1 < len(rec["W"]) else J
        if closed == 0:
            assert W is None, i
        else:
            assert torch.equal(W[0], ref["W1"][0, :, closed - 1]) and torch.equal(W[1], ref["W2"][0, :, closed - 1]), i
    if C + K - 1 <= 8:      # the lockstep stream, one push and a flush
        s = OnlineTangoStream(1, K, C, n_fft=n_fft, block=P, R0=rec["R0"], device=y.device, **kw)
        fn = lambda t0, Yv, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]])
        a, b = s.push(y, fn), s.flush(fn)
        for k in ("z_y", "zn", "yf", "yf_time"):
            assert torch.equal(torch.cat((a[k], b[k]), dim=2)[0], got[k]), k
    return got


# (n_fft, K, C, block, lag, lambda, R0 every n-th open (0: never), slots, steps)
CASES = [
    (256, 1, 4, 8, 1, 0.95, 2, 5, 9),        # K C even, single node, R0 on some slots
    (512, 1, 3, 1, 2, 0.9, 0, 4, 8),         # K C odd: a lone last signal per slot
    (1024, 3, 1, 64, 1, 0.95, 3, 4, 7),      # K > 1, K C odd
    (512, 2, 3, 8, 2, 0.95, 2, 5, 8),        # K > 1, K C even, lag 2
    (256, 8, 2, 8, 1, 0.95, 0, 3, 7),        # D = 9 (8 x 2)
    (256, 1, 12, 8, 2, 0.95, 2, 3, 6),       # D = 12, R0
    (1024, 1, 8, 1, 1, 0.5, 0, 3, 6),        # D = 8
    (512, 4, 9, 64, 1, 0.95, 0, 3, 5),       # D = 12 over 4 nodes
]


@pytest.mark.parametrize("case", CASES, ids=["%d-%dx%d-P%d-lag%d" % c[:5] for c in CASES])
def test_pool_equals_lone_streams(dev, case):
    from disco_b200.stream import OnlineTangoPool
    n_fft, K, C, P, lag, lam, r0_every, S, steps = case
    H = n_fft // 2
    pool = OnlineTangoPool(S, K, C, n_fft=n_fft, lambda_cor=lam, block=P, lag=lag, ref_mic=C - 1 if lag == 2 else 0,
                           device=dev)
    done = _Streams(pool, dev, seed=CASES.index(case), r0_every=r0_every).run(_plan(S, steps, H, P, 7 + CASES.index(case)))
    assert len(done) >= S
    for rec in done:
        _check_stream(rec, pool)


def test_pool_neighbours_and_position(dev):
    """One slot signal next to two different neighbour schedules and at two slot indices: identical outputs."""
    from disco_b200.stream import OnlineTangoPool
    n_fft, K, C, P, H = 512, 2, 3, 4, 256
    rng = np.random.default_rng(3)
    sizes = [300, 0, 1, 255, 2000, 257, 4 * H, 77]
    y = torch.from_numpy(rng.standard_normal((K, C, sum(sizes))).astype(np.float32)).to(dev)
    masks = torch.from_numpy(rng.uniform(0.05, 0.95, (K, 1 + sum(sizes) // H, 257)).astype(np.float32)).to(dev)
    results = []
    for S, me, seed in ((3, 0, 1), (5, 3, 2)):
        pool = OnlineTangoPool(S, K, C, n_fft=n_fft, block=P, device=dev)
        nrng = np.random.default_rng(seed)
        others = [s for s in range(S) if s != me]
        pool.open([me] + others[:1])
        got = {"yf": [], "yf_time": [], "z_y": []}

        def fn(t0, n_fr, Yv, z, zn):
            m = torch.rand(z.shape, device=dev)
            m[me, :, :n_fr[me]] = masks[:, t0[me]:t0[me] + n_fr[me]]
            return m, None

        pos = 0
        for i, k in enumerate(sizes + [None]):
            if i == 2:
                pool.open(others[1:])
            n = np.array([int(nrng.integers(0, 3000)) if pool.is_open(s) else 0 for s in range(S)])
            if k is None:
                out = pool.close([me], fn)
            else:
                n[me] = k
                out = pool.push(torch.randn(S, K, C, max(int(n.max()), 1), device=dev).index_copy_(
                    0, torch.tensor([me], device=dev),
                    torch.nn.functional.pad(y[None, ..., pos:pos + k], (0, max(int(n.max()), 1) - k))), n, fn)
                pos += k
            for key in got:
                got[key].append(out[key][me, :, :int(out["samples" if key == "yf_time" else "frames"][me])])
        results.append({k: torch.cat(v, dim=1) for k, v in got.items()})
    for k in results[0]:
        assert torch.equal(results[0][k], results[1][k]), k


def test_pool_causal_masks(dev):
    """A causal irm-like estimator of the frames just analysed, run through the pool; each stream against its lone
    whole-signal run with the masks the estimator returned."""
    from disco_b200.stream import OnlineTangoPool
    n_fft, K, C, P = 256, 1, 3, 4
    pool = OnlineTangoPool(4, K, C, n_fft=n_fft, block=P, lambda_cor=0.9, device=dev)
    drv = _Streams(pool, dev, seed=11)

    def irm(t0, n_fr, Y, z, zn):
        a, b = Y[:, :, 0].abs(), zn.abs()
        mz, mw = a / (a + b + 1e-3), (a * a) / (a * a + b * b + 1e-6)
        for s in range(pool.S):
            if n_fr[s]:
                rec = drv.cur[s]
                rec["t_next"] += int(n_fr[s])
                rec["mz"].append(mz[s, :, :n_fr[s]].clone())
                rec["mw"].append(mw[s, :, :n_fr[s]].clone())
        return mz, mw

    drv.mask_fn = irm
    done = drv.run(_plan(4, 7, n_fft // 2, P, 5))
    assert float(torch.cat([torch.cat(r["mz"], dim=1).flatten() for r in done]).std()) > 0.01
    for rec in done:
        _check_stream(rec, pool)


def test_pool_mask_fn_error_closes_advanced_slots(dev):
    from disco_b200.stream import OnlineTangoPool
    n_fft, K, C, P, H = 512, 1, 4, 4, 256
    pool = OnlineTangoPool(4, K, C, n_fft=n_fft, block=P, device=dev)
    drv = _Streams(pool, dev, seed=21)
    drv.open([0, 1, 2, 3])
    drv.push(np.array([3000, 700, 2000, 100]))

    def boom(*a):
        raise RuntimeError("estimator failed")

    y = torch.randn(4, K, C, 1000, device=dev)
    with pytest.raises(RuntimeError):
        pool.push(y, np.array([1000, 0, 0, 10]), boom)       # slot 0 gets frames, slot 3 only samples
    assert [pool.is_open(s) for s in range(4)] == [False, True, True, False]
    for s in (0, 3):
        drv.cur.pop(s)
    with pytest.raises(ValueError):                          # a wrong mask shape: slot 2 advanced, slot 1 not
        pool.push(y, np.array([0, 0, 1000, 0]), lambda *a: (torch.zeros(1, 1, 1, 257, device=dev), None))
    assert pool.is_open(1) and not pool.is_open(2)
    drv.cur.pop(2)
    drv.push(np.array([0, 5000, 0, 0]))
    drv.close([1])
    _check_stream(drv.done[-1], pool)


def test_pool_validation_on_gpu(dev):
    from disco_b200.stream import OnlineTangoPool
    pool = OnlineTangoPool(3, 1, 2, n_fft=256, device=dev)
    ok = lambda t0, n_fr, Y, z, zn: (torch.full(z.shape, 0.5, device=dev), None)
    pool.open([1])
    with pytest.raises(ValueError):
        pool.open([1])
    with pytest.raises(ValueError):
        pool.push(torch.zeros(3, 1, 2, 10, device=dev), [0, 5, 5], ok)      # slot 2 is free
    with pytest.raises(ValueError):
        pool.push(torch.zeros(3, 1, 2, 10, device=dev), [0, 11, 0], ok)     # n > n_max
    pool.push(torch.zeros(3, 1, 2, 128, device=dev), [0, 128, 0], ok)
    with pytest.raises(ValueError):
        pool.close([1], ok)                                                  # 128 samples = n_fft / 2
    with pytest.raises(ValueError):
        pool.close([0], ok)                                                  # free
    assert pool.is_open(1) and pool.samples_in[1] == 128
    pool.push(torch.zeros(3, 1, 2, 128, device=dev), [0, 1, 0], ok)
    pool.close([1], ok)
    assert not pool.is_open(1)


# ---------------------------------------------------------------- kernel edges through the C ABI
def _guarded(shape, dtype, dev, guard=64):
    """A flat buffer [guard | shape | guard] filled with PATTERN; returns (flat int32 view, region tensor)."""
    words = int(np.prod(shape)) * (2 if dtype == torch.complex64 else 1)
    flat = torch.full((words + 2 * guard,), PATTERN, dtype=torch.int32, device=dev)
    region = flat[guard:guard + words].view(torch.float32)
    if dtype == torch.complex64:
        region = region.view(torch.complex64)
    return flat, region.view(shape)


def _guards_kept(flat, guard=64):
    return bool((flat[:guard] == PATTERN).all() and (flat[-guard:] == PATTERN).all())


def _stft_slot_records(n_fft, n_sig, rng):
    """Per-slot (L0, n_new, t0, n_fr, final, write) covering the kernel's edges."""
    H, N = n_fft // 2, n_fft
    job, cta = JOB_FRAMES[n_fft], CTA_FRAMES[n_fft]
    recs = []
    for n_fr in sorted({0, 1, max(job - 1, 1), job, job + 1, cta - 1, cta, cta + 1}):
        for far in (False, True):
            L0 = int(rng.integers(0, H)) if not far else int(rng.integers(40, 60)) * 8 * H + int(rng.integers(0, H))
            n_new = (n_fr + 2) * H + int(rng.integers(0, H))
            L = L0 + n_new
            recs.append((L0, n_new, L // H - n_fr, n_fr, False, True))
    recs.append((5 * H + 3, 17, 0, 0, False, True))               # new samples, no complete frame: history only
    recs.append((900 * H + 7, 0, 0, 0, False, False))            # untouched
    for L in (3 * H + 1, 4 * H, 77 * H + 5):                     # final slots: the last frame reflected at the end
        recs.append((L, 0, L // H, 1, True, False))
    recs.append((H + 1, 0, 0, 2, True, False))                   # the whole of a short stream at its end
    return recs


@pytest.mark.parametrize("n_fft", SLOT_NFFTS)
@pytest.mark.parametrize("n_sig", [1, 3, 4])
def test_stream_stft_slots_kernel_edges(dev, n_fft, n_sig):
    from disco_b200 import _lib, ops
    H, N, F, P = n_fft // 2, n_fft, n_fft // 2 + 1, 40
    rng = np.random.default_rng(n_fft + n_sig)
    recs = _stft_slot_records(n_fft, n_sig, rng)
    S = len(recs)
    n_max = max(r[1] for r in recs) + 3
    f_max = max(r[3] for r in recs)
    sigs = [rng.standard_normal((n_sig, r[0] + r[1])).astype(np.float32) for r in recs]
    sel = rng.integers(0, 2, S)
    hist = torch.full((2, S, n_sig, N), NAN, device=dev)
    chunk = torch.full((S, n_sig, n_max), NAN, device=dev)
    for s, (L0, n_new, t0, n_fr, final, write) in enumerate(recs):
        h = np.zeros((n_sig, N), np.float32)
        lo = max(L0 - N, 0)
        h[:, N - (L0 - lo):] = sigs[s][:, lo:L0]
        hist[sel[s], s] = torch.from_numpy(h).to(dev)
        chunk[s, :, :n_new] = torch.from_numpy(sigs[s][:, L0:]).to(dev)
    blk = [int(rng.integers(0, P - r[3] + 1)) for r in recs]
    rec = np.array([[L0 + n_new, n_new, t0, n_fr, blk[s], int(final), int(sel[s]), int(write)]
                    for s, (L0, n_new, t0, n_fr, final, write) in enumerate(recs)], dtype=np.int32)
    fy, Y = _guarded((S, n_sig, f_max, F), torch.complex64, dev)
    fb, Yb = _guarded((S, n_sig, P, F), torch.complex64, dev)
    hist_before = hist.clone()
    lib = _lib.load()
    d = torch.from_numpy(rec).to(dev)
    _lib.check(lib.disco_stream_stft_slots(ops._ptr(hist), ops._ptr(chunk), ops._ptr(Y), ops._ptr(Yb), ops._ptr(d),
                                           rec.ctypes.data_as(_lib.c_int_p), S, n_sig, n_max, f_max, P, n_fft, None))
    torch.cuda.synchronize()
    assert _guards_kept(fy) and _guards_kept(fb)
    yw, bw = fy[64:-64].view(S, n_sig, f_max, 2 * F), fb[64:-64].view(S, n_sig, P, 2 * F)
    for s, (L0, n_new, t0, n_fr, final, write) in enumerate(recs):
        ho = torch.zeros((n_sig, N), device=dev)
        rb = torch.full((n_sig, P, F), NAN, dtype=torch.complex64, device=dev)
        want = ops.stream_stft(hist_before[sel[s], s].contiguous(), chunk[s, :, :n_new].contiguous(), L0 + n_new, t0,
                               n_fr, n_fft, hist_out=ho if write else None, Y_blk=rb, blk_slot=blk[s], final=final)
        assert torch.equal(Y[s, :, :n_fr], want), s
        assert (yw[s, :, n_fr:] == PATTERN).all(), s                   # rows past n_fr are not written
        assert torch.equal(Yb[s, :, blk[s]:blk[s] + n_fr], want), s
        assert (bw[s, :, :blk[s]] == PATTERN).all() and (bw[s, :, blk[s] + n_fr:] == PATTERN).all(), s
        assert torch.equal(hist[sel[s], s], hist_before[sel[s], s])     # the buffer read stays as it was
        other = hist[1 - sel[s], s]
        if write:
            assert torch.equal(other, ho), s
        else:
            assert torch.isnan(other).all(), s


@pytest.mark.parametrize("n_fft", SLOT_NFFTS)
@pytest.mark.parametrize("n_sig", [1, 3, 4])
def test_stream_istft_slots_kernel_edges(dev, n_fft, n_sig):
    from disco_b200 import _lib, ops
    H, F = n_fft // 2, n_fft // 2 + 1
    rng = np.random.default_rng(3 * n_fft + n_sig)
    job, cta = JOB_FRAMES[n_fft], CTA_FRAMES[n_fft]
    recs = []
    for n_fr in sorted({0, 1, max(job - 1, 1), job, job + 1, cta - 1, cta, cta + 1, 16, 17, 40}):
        for t0 in (0, 1, int(rng.integers(2, 9)), int(rng.integers(300, 400))):
            recs.append((t0, n_fr, False))
    for t0 in (0, 3, 250):
        for n_fr in (0, 1, 2):
            recs.append((t0, n_fr, True))
    S = len(recs)
    f_max = max(r[1] for r in recs)
    rows = []
    for t0, n_fr, final in recs:
        L = (t0 + n_fr) * H - int(rng.integers(0, H)) if final else (t0 + n_fr + 5) * H
        L = max(L, 1)
        lo = max(t0 - 1, 0) * H
        hi = min(L, L if final else (t0 + n_fr - 1) * H)
        rows.append((L, lo, hi, lo - int(rng.integers(0, 50))))
    s_max = max(max(hi - xf, 0) for (L, lo, hi, xf) in rows) + int(rng.integers(0, 30))
    rec = np.array([[t0, n_fr, r[0], int(final), max(r[3], 0)] for (t0, n_fr, final), r in zip(recs, rows)],
                   dtype=np.int32)
    Yv = torch.full((S, n_sig, f_max, F), complex(NAN, NAN), dtype=torch.complex64, device=dev)
    for s, (t0, n_fr, final) in enumerate(recs):
        Yv[s, :, :n_fr] = torch.from_numpy((rng.standard_normal((n_sig, n_fr, F)) +
                                            1j * rng.standard_normal((n_sig, n_fr, F))).astype(np.complex64)).to(dev)
    carry = torch.from_numpy(rng.standard_normal((S, n_sig, H)).astype(np.float32)).to(dev)
    carry_before = carry.clone()
    fx, x = _guarded((S, n_sig, s_max), torch.float32, dev)
    lib = _lib.load()
    d = torch.from_numpy(rec).to(dev)
    _lib.check(lib.disco_stream_istft_slots(ops._ptr(Yv), ops._ptr(carry), ops._ptr(x), ops._ptr(d),
                                            rec.ctypes.data_as(_lib.c_int_p), S, n_sig, f_max, s_max, n_fft, None))
    torch.cuda.synchronize()
    assert _guards_kept(fx)
    xw = fx[64:-64].view(S, n_sig, s_max)
    for s, (t0, n_fr, final) in enumerate(recs):
        L, lo, hi, _ = rows[s]
        xf = int(rec[s, 4])
        c = carry_before[s].clone()
        run = n_fr > 0 or final
        if run:
            want = ops.stream_istft(Yv[s, :, :n_fr].contiguous(), c, t0, L, n_fft, final=final)
            a, b = lo - xf, hi - xf
            if hi > lo:
                assert torch.equal(x[s, :, a:b], want), s
                assert not torch.isnan(x[s, :, a:b]).any(), s
            assert (xw[s, :, :max(a, 0)] == PATTERN).all() and (xw[s, :, max(b, a, 0):] == PATTERN).all(), s
            assert torch.equal(carry[s], c), s
        else:
            assert (xw[s] == PATTERN).all() and torch.equal(carry[s], carry_before[s]), s
