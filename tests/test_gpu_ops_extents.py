"""Every ops call checked against the memory its kernel will address (tests/abi_extents.py), and every mismatched
operand rejected by its wrapper before anything is launched.

The library only receives pointers and scalars, so each kernel's extent follows from the scalars alone.  The fixture
`proxy` replaces ops._ptr with a version that registers every tensor handed to the library (address -> tensor) and
_lib.load with a proxy of the library.  Before forwarding a call of an entry point that takes pointers, the proxy
evaluates that entry point's row of the extent model: every device pointer must be a registered contiguous tensor of
the row's dtype on the current device, aligned to its element, whose span holds the extent; host int arrays must
hold the declared count; a workspace must be one a fused STFT+SCM call wrote, consumed with the (groups, channels,
length, n_fft, mask sets, reserved SMs) it was written with.  A call that fails is refused with `Refused` and never
reaches the library, so no out-of-extent launch reaches the GPU.

- Positive sweep: every public op at n_fft 256, 512 and 1024 with and without node_sel, frames / lengths, R0, both
  layouts and both Z layouts, then the flows that compose them (every tango_batched route of
  test_gpu_tango_routes.py, online_tango, OnlineTangoStream, OnlineTangoPool, post.to_time and post.tango_scores with
  stoi=True).  No call may be refused, and every entry point that takes pointers must be reached.
- Negative matrix: for each public op, a valid call with one thing changed (wrong F for n_fft, a wrong leading or
  trailing dimension, mismatched Rss / Rnn, a W / R0 / mask shape that does not match Y, wrong dtype, non-contiguous,
  CPU tensor, another GPU, a workspace too small / from another plan / written under another reserved-SM setting).
  Each must raise ValueError or TypeError from the wrapper with no call of a pointer-taking entry point reaching the
  proxy (the host-side queries, such as the workspace size functions, take no pointers)."""
import collections
import ctypes

import numpy as np
import pytest
import torch

import abi_extents as M

pytestmark = pytest.mark.gpu

DTYPES = {torch.complex64: "c64", torch.float32: "f32", torch.float64: "f64", torch.int32: "i32"}
# entry points that address a strided operand (row_stride) rather than a dense one
STRIDED = {("disco_band_stats", "x"), ("disco_band_stats", "sel")}


class LibSizes:
    """The library's workspace size functions, evaluated at the current reserved-SM setting."""

    def __init__(self, lib):
        self.lib = lib

    def stft_ws(self, n_grp, C, length, n_fft, n_set):
        f = self.lib.disco_stft_scm_workspace if n_set == 1 else self.lib.disco_stft_scm2_workspace
        return f(n_grp, C, length, n_fft) if n_set in (1, 2) else 0

    def bss_ws(self, n_set, nsrc, n_est, length, flen):
        return self.lib.disco_bss_eval_workspace(n_set, nsrc, n_est, length, flen)

    def stoi_ws(self, n_clean, n_pair, length):
        return self.lib.disco_stoi_workspace(n_clean, n_pair, length)


def _span(t):
    if t.numel() == 0:
        return 0
    return (sum((s - 1) * st for s, st in zip(t.shape, t.stride())) + 1) * t.element_size()


def _raw(v):
    """Address of a pointer argument (0 for NULL); host arrays are returned as they are."""
    if v is None:
        return 0
    if isinstance(v, ctypes.c_void_p):
        return v.value or 0
    if isinstance(v, (ctypes.Array, ctypes._Pointer)):
        return v
    if isinstance(v, ctypes._SimpleCData):
        return v.value
    return v


def _host_len(v):
    if isinstance(v, ctypes.Array):
        return len(v), "i32" if v._type_ is ctypes.c_int else str(v._type_)
    arr = getattr(v, "_arr", None)     # numpy's ndarray.ctypes.data_as keeps the array it points into
    if arr is None:
        return -1, "?"
    return arr.size, "i32" if arr.dtype == np.int32 else str(arr.dtype)


class Proxy:
    """The library as ops sees it under the fixture: pointer-taking entry points are checked, then forwarded."""

    def __init__(self, lib, registry, reserved):
        self._lib, self._reg = lib, registry
        self._params = M.header_params()
        self._sizes = LibSizes(lib)
        self.reserved = reserved
        self.forwarded = collections.Counter()
        self.refused = collections.Counter()
        self.written = {}    # workspace address -> (tensor, plan it was written with)

    def pointer_calls(self):
        return sum(self.forwarded.values()) + sum(self.refused.values())

    def _lookup(self, addr):
        return self._reg.get(addr)

    def _check(self, name, a):
        M.check_call(name, a, self._lookup, self._sizes, torch.cuda.current_device(), _host_len)
        for p in M.ROWS[name]:
            sp = self._reg.get(a[p]) if M.ROWS[name][p][0] != "host" and a.get(p) else None
            if sp is not None and not sp.contiguous and (name, p) not in STRIDED:
                raise M.Refused("%s: %s is not contiguous" % (name, p))
        if name in M.WS_CONSUMERS:
            n_set = M.WS_CONSUMERS[name]
            n_set = a[n_set] if isinstance(n_set, str) else n_set
            want = (a["n_grp"], a["C"], a["length"], a["n_fft"], n_set, self.reserved)
            got = self.written.get(a["workspace"])
            if got is None or got[0] is not self._reg[a["workspace"]].owner:
                raise M.Refused("%s: the workspace was not written by a fused STFT+SCM call" % name)
            if got[1] != want:
                raise M.Refused("%s: workspace written as %s (groups, C, length, n_fft, sets, reserved SMs), read as %s"
                                % (name, got[1], want))

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name == "disco_set_reserved_sms":
            def setter(n):
                rc = fn(n)
                if rc == 0:
                    self.reserved = int(n)
                return rc
            return setter
        if name not in M.ROWS:
            return fn          # host-side queries: no pointers
        names = [p for _, p in self._params[name]]

        def call(*args):
            a = {p: _raw(v) for p, v in zip(names, args)}
            try:
                self._check(name, a)
            except M.Refused:
                self.refused[name] += 1
                raise
            self.forwarded[name] += 1
            rc = fn(*args)
            if rc == 0 and name in M.WS_PRODUCERS:
                ws = self._reg[a["workspace"]].owner
                self.written[a["workspace"]] = (ws, (a["n_grp"], a["C"], a["length"], a["n_fft"],
                                                     M.WS_PRODUCERS[name], self.reserved))
            return rc
        return call


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture
def proxy(dev, monkeypatch):
    from disco_b200 import _lib, ops
    lib = _lib.load()
    registry = {}
    orig_ptr = ops._ptr

    def ptr(t):
        p = orig_ptr(t)
        if t is not None:
            registry[t.data_ptr()] = M.Span(t.data_ptr(), _span(t), DTYPES.get(t.dtype, str(t.dtype)),
                                            t.device.index if t.is_cuda else "cpu", t, t.is_contiguous())
        return p

    px = Proxy(lib, registry, ops._reserved_sms)
    monkeypatch.setattr(ops, "_ptr", ptr)
    monkeypatch.setattr(_lib, "load", lambda: px)
    yield px
    lib.disco_set_reserved_sms(ops._reserved_sms)


# ---- positive sweep ---------------------------------------------------------------------------------------------------
def _rand(dev, shape, dtype=torch.float32, seed=0, lo=None):
    g = torch.Generator(device="cpu").manual_seed(seed)
    if dtype == torch.complex64:
        return torch.randn(shape, generator=g, dtype=torch.complex64).to(dev)
    if dtype == torch.int32:
        return torch.zeros(shape, dtype=torch.int32).to(dev)
    t = torch.randn(shape, generator=g, dtype=torch.float64)
    if lo is not None:       # masks: in (lo, 1)
        t = lo + (1 - lo) * torch.rand(shape, generator=g, dtype=torch.float64)
    return t.to(dtype).to(dev)


def _hermitian(dev, lead, D, seed):
    A = _rand(dev, lead + (D, D), torch.complex64, seed)
    return A @ A.conj().transpose(-1, -2) + torch.eye(D, device=dev)


def sweep_ops(dev, n_fft):
    """Every public op at this n_fft, with its options."""
    from disco_b200 import ops
    H, F = n_fft // 2, n_fft // 2 + 1
    L = 6 * n_fft + 37
    T = ops.n_frames(L, n_fft)
    c64, f32 = torch.complex64, torch.float32
    m = lambda shape, s=0: _rand(dev, shape, f32, s, lo=0.05)
    ops.init(n_fft)
    # whole-signal transforms
    x = _rand(dev, (2, 3, L), f32, 1)
    Y = ops.stft(x, n_fft)
    ops.istft(Y, L, n_fft)
    lens = [L, L - n_fft]
    ops.istft_lengths(ops.stft_lengths(x, lens, n_fft), lens, L, n_fft)
    # fused STFT + SCM, its workspace consumers, the fused filters
    G, C = 3, 4
    xg = _rand(dev, (G, C, L), f32, 2)
    for lay in ("TF", "FT"):
        mk = m((G, T, F) if lay == "TF" else (G, F, T), 3)
        ops.stft_scm(xg, mk, n_fft, mask_layout=lay)
        _, ws = ops.stft_scm(xg, mk, n_fft, mask_layout=lay, keep_partials=True)
        ops.mwf_solve_workspace(ws, G, C, L, n_fft)
        ops.mwf_solve_workspace(ws, G, C, L, n_fft, type="mwf", want_scm=True)
        ops.scm_from_workspace(ws, G, C, L, n_fft)
        if ops.stft_scm_supported(n_fft, C, 2):
            for want_Y in (True, False):
                _, ws2 = ops.stft_scm2(xg, mk, m(mk.shape, 4), n_fft, mask_layout=lay, want_Y=want_Y)
                ops.mwf_solve_workspace2(ws2, G, C, L, n_fft, rank="full")
                for q in (0, 1):
                    ops.scm_from_workspace(ws2, G, C, L, n_fft, n_set=2, set=q)
            W1, W2 = _rand(dev, (G, F, C), c64, 5), _rand(dev, (G, F, C), c64, 6)
            for want_zn in (True, False):
                ops.stft_filter_dual(xg, W1, W2, 1, n_fft, out_layout=lay, want_zn=want_zn)
    # spectra already in memory: single-node groups
    Yg = _rand(dev, (G, C, T, F), c64, 7)
    W1, W2 = _rand(dev, (G, F, C), c64, 8), _rand(dev, (G, F, C), c64, 9)
    for lay in ("TF", "FT"):
        ops.filter_dual(W1, W2, Yg, 2, n_fft, out_layout=lay)
        ops.filter_dual(W1, W2, Yg, 0, n_fft, out_layout=lay, want_zn=False)
        ops.filter_sum_scm(W1, Yg, m((G, T, F) if lay == "TF" else (G, F, T), 10), 1, n_fft, mask_layout=lay)
    S, N = _rand(dev, (G, T, F), c64, 11), _rand(dev, (G, T, F), c64, 12)
    mask = ops.tf_mask(S, N, "irm2")
    ops.apply_mask(Yg, mask)
    ops.apply_mask(S, mask, one_minus=True)
    ops.transpose_last2(S)
    ops.transpose_last2(mask)
    # concatenated channels [Y ; z of the other nodes]: B utterances of K nodes, node_sel, both Z layouts
    B, K, C = 2, 3, 2
    D = C + K - 1
    Yb = _rand(dev, (B, K, C, T, F), c64, 13)
    Zb = _rand(dev, (B, K, T, F), c64, 14)
    Zkb = Zb.transpose(0, 1).contiguous()
    sel = [0, 2]
    Ys = Yb[:, sel].contiguous()
    for lay in ("TF", "FT"):
        mb = m((B, K, T, F) if lay == "TF" else (B, K, F, T), 15)
        ops.masked_scm(Yb, mb, Zb, n_fft, mask_layout=lay)
        ops.masked_scm(Yb, mb, Zkb, n_fft, mask_layout=lay, z_layout="KB")
        ops.masked_scm(Ys, mb[:, sel].contiguous(), Zb, n_fft, mask_layout=lay, node_sel=sel)
        ops.masked_scm(Yb, None, None, n_fft, mask_layout=lay)
        W = _rand(dev, (B, K, F, D), c64, 16)
        ops.filter_sum(W, Yb, Zb, True, 0, n_fft, out_layout=lay)
        ops.filter_sum(W, Yb, Zkb, False, None, n_fft, out_layout=lay, z_layout="KB")
        ops.filter_sum(W[:, sel].contiguous(), Ys, Zkb, True, D - 1, n_fft, out_layout=lay, node_sel=sel,
                       z_layout="KB")
        ops.filter_sum(_rand(dev, (B, K, F, C), c64, 17), Yb, None, True, 1, n_fft, out_layout=lay)
    Rss, Rnn = ops.masked_scm(Yb, m((B, K, T, F), 18), Zb, n_fft)
    for typ, rank in (("gevd", 1), ("gevd", "full"), ("r1-mwf", 1), ("mwf", 1)):
        ops.mwf_solve(Rss, Rnn, type=typ, rank=rank)
    if ops.tango_mid_supported(C, K):
        ops.tango_mid(_rand(dev, (B, K, F, C), c64, 19), Yb, m((B, K, T, F), 20), 1, n_fft)
    # recursive statistics and block filters: R0, frames, node_sel, Z or none
    block = 4
    J = -(-T // block)
    frames = [T, T - 5]
    R0 = (_hermitian(dev, (B, K, F), D, 21), _hermitian(dev, (B, K, F), D, 22))
    R0s = tuple(r[:, sel].contiguous() for r in R0)
    R0c = (_hermitian(dev, (B, K, F), C, 23), _hermitian(dev, (B, K, F), C, 24))
    mb = m((B, K, T, F), 25)
    for fr in (None, frames):
        ops.scm_recursive(Yb, mb, Zb, 0.9, block, 2, None, n_fft, frames=fr)
        ops.scm_recursive(Yb, mb, Zb, 0.9, block, 1, R0, n_fft, frames=fr)
        ops.scm_recursive(Ys, mb[:, sel].contiguous(), Zb, 0.9, block, 2, R0s, n_fft, node_sel=sel, frames=fr)
        ops.scm_recursive(Yb, None, None, 0.9, block, 2, R0c, n_fft, frames=fr)
        ops.filter_sum_blocks(_rand(dev, (B, K, J, F, D), c64, 26), Yb, Zb, block, 1, True, 1, n_fft, frames=fr)
        ops.filter_sum_blocks(_rand(dev, (B, 2, J, F, D), c64, 27), Ys, Zb, block, 0, False, 0, n_fft, node_sel=sel,
                              frames=fr)
        ops.filter_sum_blocks(_rand(dev, (B, K, J, F, C), c64, 28), Yb, None, block, 2, True, C - 1, n_fft, frames=fr)
    # streaming transforms, one stream and a pool of slots
    n_sig, n_new = 3, 2 * n_fft
    hist, hist_out = torch.zeros((n_sig, n_fft), device=dev), torch.empty((n_sig, n_fft), device=dev)
    chunk = _rand(dev, (n_sig, n_new), f32, 29)
    Y_blk = torch.zeros((n_sig, 8, F), dtype=c64, device=dev)
    Yst = ops.stream_stft(hist, chunk, n_new, 0, n_new // H, n_fft, hist_out=hist_out, Y_blk=Y_blk, blk_slot=1)
    ops.stream_stft(hist_out, chunk[:, :0], n_new, n_new // H, 1, n_fft, final=True)
    carry = torch.zeros((n_sig, H), device=dev)
    ops.stream_istft(Yst, carry, 0, n_new, n_fft)
    xo = torch.zeros((n_sig, n_new), device=dev)
    ops.stream_istft(Yst[:, :1].contiguous(), carry, Yst.shape[1], n_new, n_fft, final=True, x=xo, x_first=0)
    Sl = 2
    hist2 = torch.zeros((2, Sl, n_sig, n_fft), device=dev)
    ch2 = _rand(dev, (Sl, n_sig, n_new), f32, 30)
    recs = np.array([[n_new, n_new, 0, n_new // H, 0, 0, 0, 1], [H + 1, H + 1, 0, 1, 2, 0, 0, 1]], dtype=np.int32)
    Yb2 = torch.zeros((Sl, n_sig, 4, F), dtype=c64, device=dev)
    Ysl = ops.stream_stft_slots(hist2, ch2, recs, n_new // H, n_fft, Y_blk=Yb2)
    irecs = np.array([[0, n_new // H, n_new, 0, 0], [0, 1, H + 1, 1, 0]], dtype=np.int32)
    ops.stream_istft_slots(Ysl, torch.zeros((Sl, n_sig, H), device=dev), irecs,
                           torch.zeros((Sl, n_sig, n_new), device=dev), n_fft)


def sweep_metrics(dev):
    """The n_fft-free ops: filter bank statistics, BSS-eval, resampling, STOI."""
    from disco_b200 import ops
    from scipy.signal import butter
    x = _rand(dev, (2, 3, 4000), torch.float32, 31)
    ba = torch.from_numpy(np.stack([np.stack(butter(o, [0.1, 0.3], btype="band")) for o in (2, 2)]))
    ops.band_stats(x, ba)
    ops.band_stats(x, torch.tensor([[[1, 0, 0], [1, 0, 0]]]))        # an integer pass-through filter is converted
    ops.band_stats(x[..., 100:3900], ba, sel=(x[..., 100:3900] > 0).float())
    ops.bss_eval(_rand(dev, (2, 2, 3000), torch.float32, 32), _rand(dev, (2, 3, 3000), torch.float32, 33), flen=64)
    taps = torch.from_numpy(np.hanning(61)).to(dev)
    xr = _rand(dev, (3, 5000), torch.float32, 34)
    ops.resample_poly(xr, taps, 5, 8)
    ops.resample_poly(xr, taps, 5, 8, lengths=[5000, 3000, 2000])
    cl = _rand(dev, (2, 12000), torch.float64, 35)
    dg = cl + 0.3 * _rand(dev, (3, 12000), torch.float64, 36)[:2]
    pairs = torch.tensor([[0, 0], [1, 1], [0, 1]], dtype=torch.int32, device=dev)
    ops.stoi(cl, dg, pairs)
    ops.stoi(cl, dg, pairs, lengths=[12000, 9000])


def sweep_flows(dev, n_fft):
    """The flows that compose the ops at this n_fft: online Tango whole-signal (uniform and lengths=), the lockstep
    stream, the pool of slots."""
    from disco_b200 import online
    from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
    from disco_b200.synth import make_batch
    B, K, C = 2, 2, 2
    L = 20 * n_fft
    y, s, n = (torch.from_numpy(a).to(dev) for a in make_batch(B, K, C, L, seed0=40 + n_fft))
    online.online_tango(y, n_fft=n_fft, block=4, s=s, n=n, vads=("irm1", "irm2"))
    online.online_tango(y, n_fft=n_fft, block=4, s=s, n=n, lengths=[L, L - 3 * n_fft])
    st = OnlineTangoStream(B, K, C, n_fft=n_fft, block=4, device=dev)
    mfn = lambda t0, Y, z, zn: (Y[:, :, 0].abs() / (Y[:, :, 0].abs() + zn.abs() + 1e-3), None)
    for a in range(0, L, 3 * n_fft + 17):
        st.push(y[..., a:a + 3 * n_fft + 17].contiguous(), mfn)
    st.flush(mfn)
    pool = OnlineTangoPool(3, K, C, n_fft=n_fft, block=4, device=dev)
    pfn = lambda t0, n_fr, Y, z, zn: (Y[:, :, 0].abs() / (Y[:, :, 0].abs() + zn.abs() + 1e-3), None)
    pool.open([0, 2])
    for step in range(4):
        nn = np.array([2 * n_fft + 5, n_fft + 3 if step >= 2 else 0, n_fft + step], dtype=np.int64)
        pool.push(_rand(dev, (3, K, C, int(nn.max())), torch.float32, 50 + step), nn, pfn)
        if step == 1:
            pool.open([1])
    pool.close([0, 1, 2], pfn)


def sweep_tango(dev):
    """Every tango_batched route of test_gpu_tango_routes.py under two filter settings, the reference-signature
    adapter on ragged arrays, then post.to_time and post.tango_scores with stoi=True."""
    import test_gpu_tango_routes as R
    from disco_b200 import ops, post
    from disco_b200.tango import offline_tango, tango_batched
    for row in R.ROUTES:
        for fi in (0, 1):
            typ, rank, mu, ref, kind, layout = R.case_options(row, fi)
            (y, s, n), L = R._make_inputs(row, fi)
            if row["chans"] is not None:
                offline_tango(y, s, n, list(row["vads"]), [None, None], row["mfz"], n_fft=row["n_fft"], mu=mu,
                              filter_type=typ, rank=rank)
                continue
            K, B, n_fft = row["K"], row["B"], row["n_fft"]
            T, F = ops.n_frames(L, n_fft), n_fft // 2 + 1
            yd, sd, nd = (torch.from_numpy(a).to(dev) for a in (y, s, n))
            rng = np.random.default_rng(fi)
            ext = lambda: torch.from_numpy(R._external(rng, B, K, T, F)).to(dev)
            masks = {"oracle": None, "external": (ext(), ext()), "same": (ext(), None),
                     "callable": (ext(), R._estimator(ext(), []))}[kind]
            tango_batched(yd, sd, nd, masks=masks, vads=row["vads"], mask_for_z=row["mfz"], n_fft=n_fft, mu=mu,
                          filter_type=typ, rank=rank, ref_mic=ref, out_layout=layout, diagnostics=True)
    # scoring
    from disco_b200.synth import make_batch
    fs, L, n_fft = 16000, 2 * 16000 + 300, 512
    y, s, n = (torch.from_numpy(a).to(dev) for a in make_batch(2, 2, 2, L, seed0=77))
    for lengths in (None, [L, L - 4000]):
        out = tango_batched(y, s, n, n_fft=n_fft, out_layout="TF", lengths=lengths)
        times = post.to_time(out, L, n_fft=n_fft, layout="TF", lengths=lengths)
        post.tango_scores(y[:, :, 0], s[:, :, 0], n[:, :, 0], s[:, 0, 0], n[:, 0, 0], times, fs, stoi=True,
                          lengths=lengths)
    out = tango_batched(y, s, n, n_fft=n_fft, out_layout="FT")
    post.to_time(out, L, n_fft=n_fft, layout="FT")


REACHED = collections.Counter()
SWEEPS = {"ops256": lambda d: sweep_ops(d, 256), "ops512": lambda d: sweep_ops(d, 512),
          "ops1024": lambda d: sweep_ops(d, 1024), "metrics": sweep_metrics, "flows256": lambda d: sweep_flows(d, 256),
          "flows512": lambda d: sweep_flows(d, 512), "flows1024": lambda d: sweep_flows(d, 1024), "tango": sweep_tango}
DONE = set()


def _run_sweep(name, dev, px):
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        SWEEPS[name](dev)
    torch.cuda.synchronize()
    assert not px.refused, px.refused
    REACHED.update(px.forwarded)
    DONE.add(name)


@pytest.mark.parametrize("name", list(SWEEPS))
def test_positive_sweep(dev, proxy, name):
    _run_sweep(name, dev, proxy)
    assert sum(proxy.forwarded.values()) > 0


def test_every_pointer_entry_point_reached(dev, proxy):
    """Runs the sweeps not run yet in this session, then requires a call of every entry point that takes pointers."""
    for name in SWEEPS:
        if name not in DONE:
            _run_sweep(name, dev, proxy)
            proxy.forwarded.clear()
    hp = M.header_params()
    want = {n for n, ps in hp.items() if M.pointer_params(ps)}
    missing = sorted(want - set(REACHED))
    assert not missing, missing
    print("calls per entry point:", dict(sorted(REACHED.items())))


# ---- negative matrix --------------------------------------------------------------------------------------------------
# n_fft 512: F = 257, L = 3037 samples -> T = 12 frames; B = 2 utterances of K = 3 nodes of C = 2 mics (D = 4); G = 2
NF, FB, LN, TN, FW = 512, 257, 3037, 12, 129     # FW: the bins of 256-point spectra, wrong for n_fft 512
B_, K_, C_, D_, G_ = 2, 3, 2, 4, 2


def _c(dev, *shape):
    return _rand(dev, shape, torch.complex64, len(shape))


def _f(dev, *shape):
    return _rand(dev, shape, torch.float32, len(shape), lo=0.05)


def _good(op, dev, F=FB):
    """A valid call of `op` (kwargs by parameter name) at n_fft 512; F other than 257 builds every spectrum, filter and
    mask with that many bins instead (a call consistent in itself whose spectra are not n_fft's)."""
    from disco_b200 import ops
    T, L = TN, LN
    if op == "stft":
        return dict(x=_rand(dev, (2, 3, L), seed=1), n_fft=NF)
    if op in ("stft_scm", "stft_scm2", "stft_filter_dual"):
        x = _rand(dev, (G_, C_, L), seed=2)
        if op == "stft_scm":
            return dict(x=x, mask=_f(dev, G_, T, FB), n_fft=NF)
        if op == "stft_scm2":
            return dict(x=x, mask_a=_f(dev, G_, T, FB), mask_b=_f(dev, G_, T, FB), n_fft=NF)
        return dict(x=x, W1=_c(dev, G_, FB, C_), W2=_c(dev, G_, FB, C_), n_fft=NF)
    if op == "mwf_solve_workspace":
        return dict(ws=ops.stft_scm(_rand(dev, (G_, C_, L), seed=3), _f(dev, G_, T, FB), NF, keep_partials=True)[1],
                    G=G_, C=C_, L=L, n_fft=NF)
    if op in ("mwf_solve_workspace2", "scm_from_workspace"):
        ws = ops.stft_scm2(_rand(dev, (G_, C_, L), seed=4), _f(dev, G_, T, FB), _f(dev, G_, T, FB), NF)[1]
        kw = dict(ws=ws, G=G_, C=C_, L=L, n_fft=NF)
        return dict(kw, n_set=2, set=1) if op == "scm_from_workspace" else kw
    if op == "filter_dual":
        return dict(W1=_c(dev, G_, F, C_), W2=_c(dev, G_, F, C_), Y=_c(dev, G_, C_, T, F), n_fft=NF)
    if op == "tf_mask":
        return dict(S=_c(dev, G_, T, F), N=_c(dev, G_, T, F))
    if op == "masked_scm":
        return dict(Y=_c(dev, B_, K_, C_, T, F), mask=_f(dev, B_, K_, T, F), Z=_c(dev, B_, K_, T, F), n_fft=NF)
    if op == "filter_sum_scm":
        return dict(W1=_c(dev, G_, F, C_), Y=_c(dev, G_, C_, T, F), mask=_f(dev, G_, T, F), n_fft=NF)
    if op == "tango_mid":
        return dict(W1=_c(dev, B_, K_, F, C_), Y=_c(dev, B_, K_, C_, T, F), mask_w=_f(dev, B_, K_, T, F), n_fft=NF)
    if op == "mwf_solve":
        return dict(Rss=_hermitian(dev, (G_, F), D_, 5), Rnn=_hermitian(dev, (G_, F), D_, 6))
    if op == "filter_sum":
        return dict(W=_c(dev, B_, K_, F, D_), Y=_c(dev, B_, K_, C_, T, F), Z=_c(dev, B_, K_, T, F), ref=0, n_fft=NF)
    if op == "istft":
        return dict(Y=_c(dev, 2, T, F), length=L, n_fft=NF)
    if op == "stft_lengths":
        return dict(x=_rand(dev, (2, L), seed=7), lengths=[L, L - 700], n_fft=NF)
    if op == "istft_lengths":
        return dict(Y=_c(dev, 2, T, F), lengths=[L, L - 700], length=L, n_fft=NF)
    if op == "scm_recursive":
        return dict(Y=_c(dev, B_, K_, C_, T, F), mask=_f(dev, B_, K_, T, F), Z=_c(dev, B_, K_, T, F), block=4,
                    R0=(_hermitian(dev, (B_, K_, F), D_, 8), _hermitian(dev, (B_, K_, F), D_, 9)), n_fft=NF)
    if op == "filter_sum_blocks":
        return dict(W=_c(dev, B_, K_, 3, F, D_), Y=_c(dev, B_, K_, C_, T, F), Z=_c(dev, B_, K_, T, F), block=4, n_fft=NF)
    if op == "stream_stft":
        return dict(hist=torch.zeros((3, NF), device=dev), chunk=_rand(dev, (3, 2 * NF), seed=10), length=2 * NF, t0=0,
                    n_fr=4, n_fft=NF, hist_out=torch.zeros((3, NF), device=dev), Y_blk=_c(dev, 3, 8, F))
    if op == "stream_istft":
        return dict(Y=_c(dev, 3, 4, F), carry=torch.zeros((3, NF // 2), device=dev), t0=0, length=2 * NF, n_fft=NF,
                    x=torch.zeros((3, 2 * NF), device=dev))
    if op == "stream_stft_slots":
        return dict(hist=torch.zeros((2, 2, 3, NF), device=dev), chunk=_rand(dev, (2, 3, 2 * NF), seed=11),
                    slots=np.array([[2 * NF, 2 * NF, 0, 4, 0, 0, 0, 1], [0] * 8], dtype=np.int32), f_max=4, n_fft=NF,
                    Y_blk=_c(dev, 2, 3, 4, F))
    if op == "stream_istft_slots":
        return dict(Y=_c(dev, 2, 3, 4, F), carry=torch.zeros((2, 3, NF // 2), device=dev),
                    slots=np.array([[0, 4, 2 * NF, 0, 0], [0] * 5], dtype=np.int32),
                    x=torch.zeros((2, 3, 2 * NF), device=dev), n_fft=NF)
    if op == "band_stats":
        return dict(x=_rand(dev, (2, 3, 2000), seed=12), ba=torch.tensor([[[1.0, 0, 0], [1.0, -0.5, 0.1]]] * 2,
                                                                        dtype=torch.float64),
                    sel=torch.ones((2, 3, 2000), device=dev))
    if op == "bss_eval":
        return dict(refs=_rand(dev, (2, 2, 2000), seed=13), ests=_rand(dev, (2, 3, 2000), seed=14), flen=32)
    if op == "resample_poly":
        return dict(x=_rand(dev, (3, 2000), seed=15), taps=torch.ones(31, dtype=torch.float64, device=dev), up=2, down=3)
    if op == "stoi":
        return dict(cleans=_rand(dev, (2, 5000), torch.float64, 16), degraded=_rand(dev, (2, 5000), torch.float64, 17),
                    pairs=torch.tensor([[0, 0], [1, 1]], dtype=torch.int32, device=dev))
    if op == "transpose_last2":
        return dict(a=_c(dev, 2, T, F))
    if op == "apply_mask":
        return dict(X=_c(dev, G_, C_, T, F), m=_f(dev, G_, T, F))
    raise KeyError(op)


def _wrong_dtype(t):
    return t.to(torch.float32 if t.dtype == torch.float64 else torch.int64 if t.dtype == torch.int32 else torch.float64)


def _noncontig(t):
    out = torch.empty(tuple(t.shape) + (2,), dtype=t.dtype, device=t.device)[..., 0]
    out.copy_(t)
    return out


# per op: tensor arguments the generic mutations (dtype, non-contiguous, CPU, another GPU) leave alone because the
# wrapper converts them on purpose (band_stats takes a time slice of x in place and moves `ba` to the device as float64)
CONVERTS = {"band_stats": {"x": ("noncontig",), "sel": ("noncontig",), "ba": ("dtype", "noncontig", "cpu", "gpu")}}
# tf_mask keeps the reference's AssertionError (a deliberate exception to "ValueError or TypeError") for spectrograms of different shapes (sigproc_utils.py:71)
RAISES = {"tf_mask": (AssertionError,)}


def _device_operands(op):
    """The tensor arguments of op's valid call that have to share its device (not converted by the wrapper)."""
    return [a for a in _TENSOR_ARGS[op] if "gpu" not in CONVERTS.get(op, {}).get(a, ())]


def _generic(op):
    """(case id, mutate(kwargs, dev) -> kwargs) of every tensor argument of op's valid call.  Moving an operand to
    another GPU is a mismatch only while another operand stays on the first one: an op whose only device operand is
    on cuda:1 runs there (test_ops_run_on_their_operands_gpu)."""
    out = []
    for arg in _TENSOR_ARGS[op]:
        for kind, fn in (("dtype", _wrong_dtype), ("noncontig", _noncontig), ("cpu", lambda t: t.cpu()),
                         ("gpu", lambda t: t.to("cuda:1"))):
            if kind in CONVERTS.get(op, {}).get(arg, ()):
                continue
            if kind == "gpu" and len(_device_operands(op)) < 2:
                continue

            def mut(kw, dev, arg=arg, fn=fn):
                v = kw[arg]
                kw[arg] = tuple(fn(r) for r in v) if isinstance(v, tuple) else fn(v)
                return kw
            out.append(("%s:%s" % (arg, kind), mut))
    return out


_TENSOR_ARGS = {
    "stft": ("x",), "stft_scm": ("x", "mask"), "stft_scm2": ("x", "mask_a", "mask_b"),
    "stft_filter_dual": ("x", "W1", "W2"), "mwf_solve_workspace": ("ws",), "mwf_solve_workspace2": ("ws",),
    "scm_from_workspace": ("ws",), "filter_dual": ("W1", "W2", "Y"), "tf_mask": ("S", "N"),
    "masked_scm": ("Y", "mask", "Z"), "filter_sum_scm": ("W1", "Y", "mask"), "tango_mid": ("W1", "Y", "mask_w"),
    "mwf_solve": ("Rss", "Rnn"), "filter_sum": ("W", "Y", "Z"), "istft": ("Y",), "stft_lengths": ("x",),
    "istft_lengths": ("Y",), "scm_recursive": ("Y", "mask", "Z", "R0"), "filter_sum_blocks": ("W", "Y", "Z"),
    "stream_stft": ("hist", "chunk", "hist_out", "Y_blk"), "stream_istft": ("Y", "carry", "x"),
    "stream_stft_slots": ("hist", "chunk", "Y_blk"), "stream_istft_slots": ("Y", "carry", "x"),
    "band_stats": ("x", "ba", "sel"), "bss_eval": ("refs", "ests"), "resample_poly": ("x", "taps"),
    "stoi": ("cleans", "degraded", "pairs"), "transpose_last2": ("a",), "apply_mask": ("X", "m")}


def _set(**changes):
    """Mutation replacing arguments: each value is a function of (kwargs, dev) or a constant."""
    def mut(kw, dev):
        for k, v in changes.items():
            kw[k] = v(kw, dev) if callable(v) else v
        return kw
    return mut


def _wrong_F(op):
    """The whole call built with 129-bin spectra while n_fft stays 512."""
    return ("F129_for_n_fft512", lambda kw, dev: dict(_good(op, dev, F=FW), **{k: v for k, v in kw.items()
                                                                           if not isinstance(v, torch.Tensor)
                                                                           and not isinstance(v, tuple)}))


def _ws_cases(op):
    """Workspace mutations: too small (its record claims the plan, it holds one slot less), another plan, another
    mask-set count, another reserved-SM setting."""
    from disco_b200 import ops

    def short(kw, dev):
        ws = kw["ws"]
        slot = (2 if op != "mwf_solve_workspace" else 1) * 2 * C_ * C_ * FB    # floats of one group slot
        w2 = ws[: ws.numel() - slot]
        for k, v in vars(ws).items():
            setattr(w2, k, v)
        kw["ws"] = w2
        return kw

    def other_sets(kw, dev):
        if op == "mwf_solve_workspace":
            kw["ws"] = _good("mwf_solve_workspace2", dev)["ws"]
        else:
            kw["ws"] = _good("mwf_solve_workspace", dev)["ws"]
        return kw

    def reserved(kw, dev):
        ops.set_reserved_sms(8)
        return kw
    out = [("ws:one_slot_short", short), ("ws:G+1", _set(G=G_ + 1)), ("ws:C+1", _set(C=C_ + 1)),
           ("ws:L+hop", _set(L=LN + NF // 2)), ("ws:L+1_same_frames", _set(L=LN + 1)), ("ws:n_fft256", _set(n_fft=256)),
           ("ws:other_mask_sets", other_sets), ("ws:reserved_sms", reserved)]
    if op == "scm_from_workspace":
        out.append(("ws:n_set1_of_2", _set(n_set=1, set=0)))
    return out


SPECIFIC = {
    "stft": [("x:0d", _set(x=lambda kw, dev: torch.zeros((), device=dev)))],
    "stft_scm": [("mask:T+1", _set(mask=lambda kw, dev: _f(dev, G_, TN + 1, FB))),
                 ("mask:F129", _set(mask=lambda kw, dev: _f(dev, G_, TN, FW))),
                 ("mask:G+1", _set(mask=lambda kw, dev: _f(dev, G_ + 1, TN, FB)))],
    "stft_scm2": [("mask_b:T+1", _set(mask_b=lambda kw, dev: _f(dev, G_, TN + 1, FB)))],
    "stft_filter_dual": [("W2:F129", _set(W2=lambda kw, dev: _c(dev, G_, FW, C_))),
                         ("W1:C+1", _set(W1=lambda kw, dev: _c(dev, G_, FB, C_ + 1)))],
    "filter_dual": [_wrong_F("filter_dual"), ("W2:C+1", _set(W2=lambda kw, dev: _c(dev, G_, FB, C_ + 1))),
                    ("W1:G+1", _set(W1=lambda kw, dev: _c(dev, G_ + 1, FB, C_)))],
    "tf_mask": [("N:T+1", _set(N=lambda kw, dev: _c(dev, G_, TN + 1, FB)))],
    "masked_scm": [_wrong_F("masked_scm"), ("mask:T+1", _set(mask=lambda kw, dev: _f(dev, B_, K_, TN + 1, FB))),
                   ("Z:T+1", _set(Z=lambda kw, dev: _c(dev, B_, K_, TN + 1, FB))),
                   ("Z:B+1", _set(Z=lambda kw, dev: _c(dev, B_ + 1, K_, TN, FB))),
                   ("Y:4d", _set(Y=lambda kw, dev: _c(dev, B_ * K_, C_, TN, FB)))],
    "filter_sum_scm": [_wrong_F("filter_sum_scm"), ("mask:T-1", _set(mask=lambda kw, dev: _f(dev, G_, TN - 1, FB))),
                       ("W1:C+1", _set(W1=lambda kw, dev: _c(dev, G_, FB, C_ + 1)))],
    "tango_mid": [_wrong_F("tango_mid"), ("mask_w:K+1", _set(mask_w=lambda kw, dev: _f(dev, B_, K_ + 1, TN, FB))),
                  ("W1:F129", _set(W1=lambda kw, dev: _c(dev, B_, K_, FW, C_)))],
    "mwf_solve": [("Rnn:F-1", _set(Rnn=lambda kw, dev: _hermitian(dev, (G_, FB - 1), D_, 1))),
                  ("Rnn:D-1", _set(Rnn=lambda kw, dev: _hermitian(dev, (G_, FB), D_ - 1, 2))),
                  ("Rss,Rnn:not_square", _set(Rss=lambda kw, dev: _c(dev, G_, FB, D_ + 1, D_),
                                              Rnn=lambda kw, dev: _c(dev, G_, FB, D_ + 1, D_)))],
    "filter_sum": [_wrong_F("filter_sum"), ("W:D-1", _set(W=lambda kw, dev: _c(dev, B_, K_, FB, D_ - 1))),
                   ("Z:F129", _set(Z=lambda kw, dev: _c(dev, B_, K_, TN, FW)))],
    "istft": [_wrong_F("istft")],
    "stft_lengths": [("lengths:count", _set(lengths=[LN, LN, LN]))],
    "istft_lengths": [_wrong_F("istft_lengths")],
    "scm_recursive": [_wrong_F("scm_recursive"), ("mask:T+1", _set(mask=lambda kw, dev: _f(dev, B_, K_, TN + 1, FB))),
                      ("R0:D-1", _set(R0=lambda kw, dev: tuple(_hermitian(dev, (B_, K_, FB), D_ - 1, s)
                                                               for s in (1, 2)))),
                      ("R0:one", _set(R0=lambda kw, dev: (kw["R0"][0], kw["R0"][1][:, :2].contiguous()))),
                      ("Z:T-1", _set(Z=lambda kw, dev: _c(dev, B_, K_, TN - 1, FB))),
                      ("frames:count", _set(frames=[TN, TN, TN]))],
    "filter_sum_blocks": [_wrong_F("filter_sum_blocks"), ("W:J+1", _set(W=lambda kw, dev: _c(dev, B_, K_, 4, FB, D_))),
                          ("W:D+1", _set(W=lambda kw, dev: _c(dev, B_, K_, 3, FB, D_ + 1)))],
    "stream_stft": [("Y_blk:F129", _set(Y_blk=lambda kw, dev: _c(dev, 3, 8, FW))),
                    ("hist_out:n_sig+1", _set(hist_out=lambda kw, dev: torch.zeros((4, NF), device=dev))),
                    ("chunk:n_sig-1", _set(chunk=lambda kw, dev: kw["chunk"][:2].contiguous()))],
    "stream_istft": [_wrong_F("stream_istft"), ("carry:H+1", _set(carry=lambda kw, dev: torch.zeros((3, NF // 2 + 1),
                                                                                                   device=dev))),
                     ("x:n_sig-1", _set(x=lambda kw, dev: torch.zeros((2, 2 * NF), device=dev)))],
    "stream_stft_slots": [("Y_blk:F129", _set(Y_blk=lambda kw, dev: _c(dev, 2, 3, 4, FW))),
                          ("hist:one_buffer", _set(hist=lambda kw, dev: torch.zeros((1, 2, 3, NF), device=dev))),
                          ("slots:S+1", _set(slots=np.zeros((3, 8), dtype=np.int32)))],
    "stream_istft_slots": [_wrong_F("stream_istft_slots"),
                           ("carry:S+1", _set(carry=lambda kw, dev: torch.zeros((3, 3, NF // 2), device=dev))),
                           ("slots:fields", _set(slots=np.zeros((2, 4), dtype=np.int32)))],
    "band_stats": [("sel:L-1", _set(sel=lambda kw, dev: torch.ones((2, 3, 1999), device=dev))),
                   ("ba:2d", _set(ba=torch.ones((2, 3), dtype=torch.float64))),
                   ("ba:not_a_tensor", _set(ba=[[[1.0, 0, 0], [1.0, 0, 0]]]))],
    "bss_eval": [("ests:L+1", _set(ests=lambda kw, dev: _rand(dev, (2, 3, 2001), seed=1))),
                 ("ests:S+1", _set(ests=lambda kw, dev: _rand(dev, (3, 3, 2000), seed=1)))],
    "resample_poly": [("lengths:count", _set(lengths=[5, 5]))],
    "stoi": [("degraded:L-1", _set(degraded=lambda kw, dev: _rand(dev, (2, 4999), torch.float64, 1))),
             ("pairs:3_cols", _set(pairs=lambda kw, dev: torch.zeros((2, 3), dtype=torch.int32, device=dev)))],
    "transpose_last2": [],
    "apply_mask": [("m:T+1", _set(m=lambda kw, dev: _f(dev, G_, TN + 1, FB)))],
}
for _op in ("mwf_solve_workspace", "mwf_solve_workspace2", "scm_from_workspace"):
    SPECIFIC[_op] = _ws_cases(_op)
# per op where frames= / lengths= adds a twin entry point: the same cases run through it too
WITH_FRAMES = {"scm_recursive": dict(frames=[TN, TN - 3]), "filter_sum_blocks": dict(frames=[TN, TN - 3]),
               "resample_poly": dict(lengths=[2000, 1500, 900])}


def negative_cases(op):
    cases = list(SPECIFIC[op]) + _generic(op)
    if op in WITH_FRAMES:
        extra = WITH_FRAMES[op]
        cases += [(cid + "|" + ",".join(extra), (lambda kw, dev, f=f: f(dict(kw, **extra), dev))) for cid, f in cases
                  if not any(k in cid for k in ("frames", "lengths"))]
    return cases


@pytest.mark.parametrize("op", sorted(_TENSOR_ARGS))
def test_negative_matrix(dev, proxy, op):
    """Every mutation of a valid call of `op` raises ValueError or TypeError from the wrapper, and not one call of an
    entry point that takes pointers reaches the library proxy."""
    from disco_b200 import ops
    two = torch.cuda.device_count() >= 2
    getattr(ops, op)(**_good(op, dev))        # the unchanged call is valid and reaches the library
    torch.cuda.synchronize()
    assert proxy.forwarded and not proxy.refused, (proxy.forwarded, proxy.refused)
    fails = []
    ran = 0
    for cid, mut in negative_cases(op):
        if ":gpu" in cid and not two:
            continue
        kw = mut(_good(op, dev), dev)
        torch.cuda.synchronize()
        before = proxy.pointer_calls()
        try:
            getattr(ops, op)(**kw)
            fails.append("%s: accepted" % cid)
        except (ValueError, TypeError) + RAISES.get(op, ()) as e:
            if proxy.pointer_calls() != before:
                fails.append("%s: raised %r after %d library call(s)" % (cid, e, proxy.pointer_calls() - before))
        except M.Refused as e:
            fails.append("%s: refused by the extent model: %s" % (cid, e))
        except Exception as e:     # noqa: BLE001 -- any other failure is a finding of this matrix
            fails.append("%s: %s: %s" % (cid, type(e).__name__, e))
        finally:
            if proxy.reserved != ops._reserved_sms or cid.endswith("reserved_sms"):
                ops.set_reserved_sms(0)
        ran += 1
    assert ran >= 3, ran
    assert not fails, "\n".join(fails)


@pytest.mark.parametrize("op", sorted(_TENSOR_ARGS))
def test_ops_run_on_their_operands_gpu(dev, proxy, op):
    """The valid call built entirely on cuda:1 runs there: the wrapper makes its operands' device current, the proxy
    finds every pointer on that device, and the outputs live on it.  Needs two visible GPUs."""
    from disco_b200 import ops
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    other = torch.device("cuda:1")
    kw = _good(op, other)
    with torch.cuda.device(0):
        out = getattr(ops, op)(**kw)
    torch.cuda.synchronize(other)
    assert proxy.forwarded and not proxy.refused, (proxy.forwarded, proxy.refused)
    stack, seen = [out], 0
    while stack:
        v = stack.pop()
        if isinstance(v, (tuple, list)):
            stack.extend(v)
        elif isinstance(v, torch.Tensor):
            assert v.device == other, (op, v.device)
            seen += 1
    assert seen, op
