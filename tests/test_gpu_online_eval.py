"""online_tango from the clean components (s, n): oracle masks, exchange modes, filter settings and the filtered
images z_s, z_n, sf, nf, checked against tango_batched's masks, the explicit filter_sum_blocks compositions and the
float64 composition of oracle/online_split_np (librosa_np spectra, the float64 solver); uneven batches against each
utterance alone; scoring through post.to_time / post.tango_scores.

SITES names, for every `ops.<name>(` call site of the helpers online_tango calls for evaluation, the test that must
reach it (the spy checks it there); tests/test_online_eval_cpu.py parses the sources and fails on CPU when a site is
named by no row, or a row names a site the sources do not have."""
import inspect
import os
import sys
import warnings

import numpy as np
import pytest
import torch

import test_gpu_tango_routes as routes
from conftest import TOL, rel_l2

pytestmark = pytest.mark.gpu

EVAL_FUNCS = ("_clean_spectra", "_online_mwf_split", "_filtered_pair")
SITES = {
    "_clean_spectra:stft#1": "test_masks_and_main_outputs",
    "_clean_spectra:stft#2": "test_masks_and_main_outputs",
    "_clean_spectra:stft_lengths#1": "test_uneven_batches",
    "_clean_spectra:stft_lengths#2": "test_uneven_batches",
    "_online_mwf_split:apply_mask#1": "test_exchange_modes",
    "_online_mwf_split:apply_mask#2": "test_exchange_modes",
    "_online_mwf_split:scm_recursive#1": "test_exchange_modes",
    "_online_mwf_split:scm_recursive#2": "test_exchange_modes",
    "_online_mwf_split:mwf_solve": "test_exchange_modes",
    "_online_mwf_split:filter_sum_blocks": "test_exchange_modes",
    "_filtered_pair:filter_sum_blocks#1": "test_diagnostics",
    "_filtered_pair:filter_sum_blocks#2": "test_diagnostics",
}
MODES = ("distant", "compressed", "use_oracle_refs", "use_oracle_zs", "previous")
MAIN = ("yf", "z_y", "zn", "W1", "W2")
DIAG = ("z_s", "z_n", "sf", "nf")
WIDE_TOL = 2e-4          # DESIGN §4.5: float32 statistics move a D >= 9 filter by up to 2.9e-4 in its first blocks


def eval_sites():
    """{site: (path, line, col)} of the ops calls inside EVAL_FUNCS, by the rule of test_gpu_tango_routes.call_sites."""
    saved = routes.SITE_FUNCS
    routes.SITE_FUNCS = {"online.py": EVAL_FUNCS}
    try:
        return routes.call_sites()
    finally:
        routes.SITE_FUNCS = saved


def sites_of(test):
    return {s for s, t in SITES.items() if t == test}


class Spy:
    """Records every spied ops call: (site of EVAL_FUNCS or None, op, bound arguments, return value)."""

    def __init__(self, monkeypatch):
        from disco_b200 import ops
        index = {v: k for k, v in eval_sites().items()}
        path = os.path.join(routes.PKG, "online.py")
        self.calls = []
        for name in routes.SPIED:
            orig = getattr(ops, name)
            sig = inspect.signature(orig)

            def wrap(*a, _orig=orig, _sig=sig, _name=name, **kw):
                fr = sys._getframe(1)
                out = _orig(*a, **kw)
                site = None
                if os.path.abspath(fr.f_code.co_filename) == path:
                    pos = list(fr.f_code.co_positions())[fr.f_lasti // 2]
                    site = index.get((path, pos[0], pos[2]))
                    if site is None:
                        same = [s for (p, ln, _), s in index.items() if ln == pos[0] and
                                s.split(":")[1].split("#")[0] == _name]
                        site = same[0] if len(same) == 1 else None
                b = _sig.bind(*a, **kw)
                b.apply_defaults()
                self.calls.append((site, _name, dict(b.arguments), out))
                return out
            monkeypatch.setattr(ops, name, wrap)

    def sites(self):
        return {s for s, _, _, _ in self.calls if s is not None}

    def solves(self):
        return [(a["type"], a["rank"], float(a["mu"])) for _, nm, a, _ in self.calls if nm == "mwf_solve"]


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _inputs(dev, B, K, C, L, seed):
    from disco_b200.synth import make_batch
    y, s, n = make_batch(B, K, C, L, seed0=seed)
    Td = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return (y, s, n), (Td(y), Td(s), Td(n))


def _start(D, block, lag):
    """First frame compared with float64: the block whose filter saw >= 4 D frames (test_online_tango_options)."""
    return (-(-4 * D // block) + lag) * block


# ---- the float64 composition ----------------------------------------------------------------------------------------
def _blocks(W, X, block, lag, ref):
    """Frame t of X (D, F, T) filtered by W[t // block - lag] (J, F, D), channel ref before the first filter."""
    T = X.shape[2]
    j = np.arange(T) // block - lag
    out = X[ref].astype(np.complex128).copy()
    live = j >= 0
    out[:, live] = np.einsum("tfd,dft->ft", np.conj(W[j[live]]), X[:, :, live])
    return out


def _spec64(x, n_fft, fsel):
    """[K, C, L] float32 -> [K, C, len(fsel), T] complex128 (librosa_np)."""
    from oracle import librosa_np
    return np.stack([np.stack([librosa_np.stft(c.astype(np.float64), n_fft=n_fft, hop_length=n_fft // 2)[fsel]
                               for c in node]) for node in x])


def f64_online(Y, S, N, mz, mw, mode, vad0, ref, o, R0=None):
    """One utterance in float64: Y, S, N [K, C, F', T] complex128, mz, mw [K, F', T] (the kernels' masks), o =
    dict(lam, block, lag, mu, typ, rank); R0 (Rs0, Rn0) [K, F', C, C] seeds step 1 (and step 2 at K = 1).
    Returns {name: [K, F', T]} for yf, z_y, zn, z_s, z_n, sf, nf."""
    from oracle import solve_f64, tango_np
    from oracle.online_split_np import online_mwf_split
    K, C = Y.shape[:2]
    fn = (tango_np.spatial_correlation_matrix, lambda Rs, Rn, mu, ft, r: solve_f64.solve(Rs, Rn, mu, ft, r))
    kw = dict(lambda_cor=o["lam"], block=o["block"], lag=o["lag"], mu=o["mu"], filter_type=o["typ"], rank=o["rank"],
              ref=ref)
    blk = lambda W, X: _blocks(W, X, o["block"], o["lag"], ref)
    r0 = lambda k: None if R0 is None else (R0[0][k], R0[1][k])
    out = {nm: np.empty((K,) + Y.shape[2:], np.complex128) for nm in ("yf", "z_y", "zn", "z_s", "z_n", "sf", "nf")}
    for k in range(K):
        if "use_oracle_" in mode:
            z, W, _, _ = online_mwf_split(Y[k], S[k], N[k], *fn, R0=r0(k), **kw)
        else:
            z, W, _, _ = online_mwf_split(Y[k], mz[k] * Y[k], (1 - mz[k]) * Y[k], *fn, R0=r0(k), **kw)
        out["z_y"][k], out["zn"][k] = z, Y[k, ref] - z
        out["z_s"][k], out["z_n"][k] = blk(W, S[k]), blk(W, N[k])
    zy, zs, zn_ = out["z_y"], out["z_s"], out["z_n"]
    for k in range(K):
        oth = [j for j in range(K) if j != k]
        m = mw[k]
        if mode == "local":
            rs, rn = m * zy[oth], (1 - m) * zy[oth]
        elif mode == "distant":
            rs, rn = mw[oth] * zy[oth], (1 - mw[oth]) * zy[oth]
        elif mode == "compressed":
            mc = np.stack([tango_np.tf_mask(zs[j], zn_[j], vad0) for j in oth]).reshape((len(oth),) + zy.shape[1:])
            rs, rn = mc * zy[oth], (1 - mc) * zy[oth]
        elif mode == "use_oracle_refs":
            rs, rn = S[oth, ref], N[oth, ref]
        elif mode == "use_oracle_zs":
            rs, rn = zs[oth], zn_[oth]
        else:
            rs, rn = zy[oth], zy[oth]
        cat = lambda own, z: np.concatenate([own, z], axis=0)
        z, W2, _, _ = online_mwf_split(cat(Y[k], zy[oth]), cat(m * Y[k], rs), cat((1 - m) * Y[k], rn), *fn,
                                       R0=r0(k) if K == 1 else None, **kw)
        out["yf"][k] = z
        out["sf"][k], out["nf"][k] = blk(W2, cat(S[k], zs[oth])), blk(W2, cat(N[k], zn_[oth]))
    return out


def _compare(got, truth, starts, bar, what):
    """Per (node, output) complex relative L2 from the output's first compared frame on."""
    for nm, t0 in starts.items():
        for k in range(truth[nm].shape[0]):
            e = rel_l2(got[nm][k][..., t0:], truth[nm][k][..., t0:])
            assert e <= bar, "%s: %s node %d from frame %d: complex rel %.3g (bar %.3g)" % (what, nm, k, t0, e, bar)


def _got(out, b, fsel):
    """[B, K, T, F] outputs of utterance b -> {name: [K, F', T]} numpy."""
    return {nm: out[nm][b].cpu().numpy()[:, :, fsel].transpose(0, 2, 1) for nm in ("yf", "z_y", "zn") + DIAG}


def _starts(C, K, block, lag):
    s1, s2 = _start(C, block, lag), _start(C + K - 1, block, lag)
    return dict(z_y=s1, zn=s1, z_s=s1, z_n=s1, yf=s2, sf=s2, nf=s2)


# ---- 1. the new arguments do not perturb the main outputs ----------------------------------------------------------
VADS = [("irm1", "irm2"), ("irm1", "irm1"), ("ibm1", "ibm1"), ("iam1", "irm1"), ("ivad", "ivad")]


@pytest.mark.parametrize("ref", ["0", "last"])
@pytest.mark.parametrize("vads", VADS, ids=["%s-%s" % v for v in VADS])
@pytest.mark.parametrize("K,C", [(1, 4), (3, 2)])
def test_masks_and_main_outputs(dev, monkeypatch, K, C, vads, ref):
    """s, n next to external masks leave yf, z_y, zn, W1, W2 bit-identical; masks=None builds the masks tango_batched
    builds, and with them the outputs of the masks-only call, bit for bit."""
    from disco_b200 import online
    from disco_b200.tango import tango_batched
    ref_mic = 0 if ref == "0" else C - 1
    _, (y, s, n) = _inputs(dev, 2, K, C, 16000, 400 + 10 * K + VADS.index(vads))
    off = tango_batched(y, s, n, vads=vads, ref_mic=ref_mic, out_layout="TF", diagnostics=False)
    mz, mw = off["masks_z"], off["mask_w"]
    kw = dict(block=8, ref_mic=ref_mic, n_fft=512)
    base = online.online_tango(y, (mz, mw), **kw)
    assert set(base) == set(MAIN)
    with_sn = online.online_tango(y, (mz, mw), s=s, n=n, **kw)
    spy = Spy(monkeypatch)
    own = online.online_tango(y, s=s, n=n, vads=vads, **kw)
    torch.cuda.synchronize()
    assert sites_of("test_masks_and_main_outputs") <= spy.sites(), sorted(spy.sites())
    assert set(with_sn) == set(MAIN + DIAG) and set(own) == set(MAIN + DIAG + ("masks_z", "mask_w"))
    for nm in MAIN:
        assert torch.equal(with_sn[nm], base[nm]), (nm, "s, n moved it")
        assert torch.equal(own[nm], base[nm]), (nm, "masks built from s, n")
    assert torch.equal(own["masks_z"], mz) and torch.equal(own["mask_w"], mw)
    if vads[0] == vads[1] and ref_mic == 0:
        assert own["mask_w"] is own["masks_z"]
    for nm in DIAG:
        assert torch.equal(own[nm], with_sn[nm]), nm


# ---- 2. diagnostics -------------------------------------------------------------------------------------------------
# (K, C, n_fft, block, lag, L): D = C + K - 1
DIAG_CASES = [(1, 4, 512, 8, 1, 24000), (3, 2, 256, 4, 1, 24000), (2, 3, 512, 8, 2, 24000), (2, 4, 256, 16, 0, 24000),
              (8, 2, 256, 16, 1, 64000)]


@pytest.mark.parametrize("K,C,n_fft,block,lag,L", DIAG_CASES,
                         ids=["k%dc%d-n%d-p%d-l%d" % c[:5] for c in DIAG_CASES])
def test_diagnostics(dev, monkeypatch, K, C, n_fft, block, lag, L):
    """z_s, z_n, sf, nf are the filter_sum_blocks compositions bit for bit, pass channel ref_mic through before the
    first filter, match the float64 composition, and yf = sf + nf on y = s + n."""
    from disco_b200 import online, ops
    lam, ref = 0.98, C - 1
    (yh, sh, nh), (y, s, n) = _inputs(dev, 2, K, C, L, 600 + 10 * K + C)
    spy = Spy(monkeypatch)
    out = online.online_tango(y, lambda_cor=lam, block=block, lag=lag, ref_mic=ref, n_fft=n_fft, s=s, n=n,
                              vads=("irm1", "irm2"))
    torch.cuda.synchronize()
    assert sites_of("test_diagnostics") <= spy.sites(), sorted(spy.sites())
    what = "k%dc%d n_fft %d block %d lag %d" % (K, C, n_fft, block, lag)
    S, N = ops.stft(s, n_fft), ops.stft(n, n_fft)
    fb = lambda W, X, Z: ops.filter_sum_blocks(W, X, Z, block, lag, True, ref, n_fft)[0]
    z_s, z_n = fb(out["W1"], S, None), fb(out["W1"], N, None)
    want = {"z_s": z_s, "z_n": z_n, "sf": fb(out["W2"], S, z_s if K > 1 else None),
            "nf": fb(out["W2"], N, z_n if K > 1 else None)}
    for nm in DIAG:
        assert torch.equal(out[nm], want[nm]), (what, nm)
        assert bool(torch.isfinite(torch.view_as_real(out[nm])).all()), (what, nm)
    if lag >= 1:
        t1 = lag * block
        for nm, X in (("z_s", S), ("sf", S), ("z_n", N), ("nf", N)):
            assert torch.equal(out[nm][:, :, :t1], X[:, :, ref, :t1]), (what, nm, "pass-through frames")
    T, F = out["yf"].shape[-2:]
    fsel = [0, 37, F // 2, F - 1]
    st = _starts(C, K, block, lag)
    assert max(st.values()) < T - block, what
    bar = TOL if C + K - 1 <= 8 else WIDE_TOL
    o = dict(lam=lam, block=block, lag=lag, mu=1.0, typ="gevd", rank=1)
    for b in range(2):
        mz = out["masks_z"][b].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
        mw = out["mask_w"][b].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
        truth = f64_online(_spec64(yh[b], n_fft, fsel), _spec64(sh[b], n_fft, fsel), _spec64(nh[b], n_fft, fsel),
                           mz, mw, "local", "irm1", ref, o)
        _compare(_got(out, b, fsel), truth, st, bar, "%s b%d" % (what, b))
    # the images add up to the output: a wrong filter on sf or nf cannot pass
    t2 = st["yf"]
    for b in range(2):
        for k in range(K):
            yf, sf, nf = (out[nm][b, k, t2:].cpu().numpy().astype(np.complex128) for nm in ("yf", "sf", "nf"))
            e = np.linalg.norm(yf - sf - nf) / np.linalg.norm(yf)
            assert e <= 1e-5, (what, b, k, "yf - sf - nf", e)


# ---- 3. every exchange mode -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_fft", [256, 512])
@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("mode", MODES)
def test_exchange_modes(dev, monkeypatch, mode, K, n_fft):
    """Each mask_for_z mode against the float64 composition; the spy sees the step-2 scans (and for use_oracle_*
    the step-1 scans) receive the stacks tango._z_for_stats defines; the mode moves the float64 answer > 10x the bar."""
    from disco_b200 import online, ops
    C, block, lag, lam, ref = 2, 8, 1, 0.98, 1
    use_r0 = mode.startswith("use_oracle_") and n_fft == 512
    (yh, sh, nh), (y, s, n) = _inputs(dev, 1, K, C, 24000, 800 + 10 * K + MODES.index(mode) + n_fft)
    T, F = ops.n_frames(24000, n_fft), n_fft // 2 + 1
    fsel = [0, 37, F // 2, F - 1]
    Y64, S64, N64 = (_spec64(a[0], n_fft, fsel) for a in (yh, sh, nh))
    R0 = R0d = None
    if use_r0:
        Sf, Nf = (_spec64(a[0], n_fft, list(range(F))) for a in (sh, nh))
        R0 = [routes._prior(X[None], np.ones((1, K, T, F)))[0][0] for X in (Sf, Nf)]    # [K, F, C, C] each
        R0d = tuple(torch.from_numpy(r[None]).to(dev) for r in R0)
    spy = Spy(monkeypatch)
    out = online.online_tango(y, lambda_cor=lam, block=block, lag=lag, ref_mic=ref, n_fft=n_fft, R0=R0d, s=s, n=n,
                              vads=("irm1", "irm2"), mask_for_z=mode)
    torch.cuda.synchronize()
    what = "%s K=%d n_fft %d" % (mode, K, n_fft)
    hit = spy.sites()
    want_sites = sites_of("test_exchange_modes")
    assert want_sites <= hit, (what, sorted(want_sites - hit))
    # the stacks the scans received
    scans = [a for s_, nm, a, _ in spy.calls if nm == "scm_recursive"]
    assert len(scans) == (4 if mode.startswith("use_oracle_") else 3), (what, len(scans))
    S, N = ops.stft(s, n_fft), ops.stft(n, n_fft)
    z_y, mw = out["z_y"], out["mask_w"]
    if mode.startswith("use_oracle_"):
        s1 = scans[:2]
        assert torch.equal(s1[0]["Y"], S) and torch.equal(s1[1]["Y"], N), what
        assert all(a["mask"] is None and a["Z"] is None for a in s1), what
        if use_r0:
            assert s1[0]["R0"][0] is R0d[0] and s1[1]["R0"][0] is R0d[1], what
    s2 = scans[-2:]
    zr = {"distant": (ops.apply_mask(z_y, mw, False), ops.apply_mask(z_y, mw, True)),
          "use_oracle_refs": (S[:, :, ref].contiguous(), N[:, :, ref].contiguous()),
          "use_oracle_zs": (out["z_s"], out["z_n"]), "previous": (z_y, z_y)}
    if mode == "compressed":
        mc = ops.tf_mask(out["z_s"], out["z_n"], "irm1")
        zr[mode] = (ops.apply_mask(z_y, mc, False), ops.apply_mask(z_y, mc, True))
    for i, a in enumerate(s2):
        assert a["mask"] is None and a["R0"] is None, what
        assert torch.equal(a["Z"], zr[mode][i]), (what, "step-2 scan %d received the wrong z" % i)
    # their own channels: mask_w Y and (1 - mask_w) Y
    own = [o_ for s_, _, _, o_ in spy.calls
           if s_ in ("_online_mwf_split:apply_mask#1", "_online_mwf_split:apply_mask#2")]
    assert len(own) == 2 and all(a["Y"] is o_ for a, o_ in zip(s2, own)), what
    Yd = ops.stft(y, n_fft)
    assert torch.equal(own[0], ops.apply_mask(Yd, mw, False)) and torch.equal(own[1], ops.apply_mask(Yd, mw, True))
    # values
    o = dict(lam=lam, block=block, lag=lag, mu=1.0, typ="gevd", rank=1)
    mz64 = out["masks_z"][0].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
    mw64 = mw[0].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
    r0 = None if R0 is None else tuple(r[:, fsel] for r in R0)
    truth = f64_online(Y64, S64, N64, mz64, mw64, mode, "irm1", ref, o, r0)
    st = _starts(C, K, block, lag)
    _compare(_got(out, 0, fsel), truth, st, TOL, what)
    local = f64_online(Y64, S64, N64, mz64, mw64, "local", "irm1", ref, o, r0)
    d = max(rel_l2(local["yf"][k][..., st["yf"]:], truth["yf"][k][..., st["yf"]:]) for k in range(K))
    assert d > 10 * TOL, (what, "mode is within %.3g of 'local'" % d)


# ---- 4. filter settings ---------------------------------------------------------------------------------------------
SETTINGS = [("r1-mwf", 1, 2.5, "local"), ("mwf", 1, 1.0, "distant"), ("gevd", 2, 2.5, "use_oracle_zs")]


@pytest.mark.parametrize("typ,rank,mu,mode", SETTINGS, ids=["%s-r%d-mu%g-%s" % c for c in SETTINGS])
def test_filter_settings(dev, monkeypatch, typ, rank, mu, mode):
    """filter_type, rank and mu reach both solves and the outputs match the float64 composition under them."""
    from disco_b200 import online, ops
    K, C, n_fft, block, lag, lam, ref = 2, 3, 256, 8, 1, 0.98, 0
    (yh, sh, nh), (y, s, n) = _inputs(dev, 1, K, C, 24000, 900 + SETTINGS.index((typ, rank, mu, mode)))
    spy = Spy(monkeypatch)
    out = online.online_tango(y, lambda_cor=lam, block=block, lag=lag, mu=mu, rank=rank, ref_mic=ref, n_fft=n_fft,
                              s=s, n=n, vads=("irm1", "irm2"), mask_for_z=mode, filter_type=typ)
    torch.cuda.synchronize()
    assert spy.solves() == [(typ, rank, mu)] * 2, spy.solves()
    F = n_fft // 2 + 1
    fsel = [0, 37, F // 2, F - 1]
    o = dict(lam=lam, block=block, lag=lag, mu=mu, typ=typ, rank=rank)
    mz = out["masks_z"][0].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
    mw = out["mask_w"][0].cpu().numpy()[:, :, fsel].transpose(0, 2, 1)
    specs = [_spec64(a[0], n_fft, fsel) for a in (yh, sh, nh)]
    truth = f64_online(*specs, mz, mw, mode, "irm1", ref, o)
    st = _starts(C, K, block, lag)
    _compare(_got(out, 0, fsel), truth, st, TOL, "%s rank %d mu %g" % (typ, rank, mu))
    gevd = f64_online(*specs, mz, mw, mode, "irm1", ref, dict(o, typ="gevd", rank=1, mu=1.0))
    d = max(rel_l2(gevd["yf"][k][..., st["yf"]:], truth["yf"][k][..., st["yf"]:]) for k in range(K))
    assert d > 10 * TOL, ("the default filter is within %.3g" % d)


# ---- 5. uneven batches ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ("local",) + MODES)
def test_uneven_batches(dev, monkeypatch, mode):
    """lengths= with s, n: each utterance's outputs, masks and diagnostics included, equal the utterance alone bit for
    bit (K * C even), are exactly 0 past T_b / J_b, and NaN in y, s, n past each length reaches no output."""
    from disco_b200 import online
    from disco_b200.synth import make_batch
    K, C, n_fft, block = 2, 2, 256, 8
    hop = n_fft // 2
    lengths = [12000, 9000 + 37, 6400, 12000 - 3 * hop]
    L, B = max(lengths), len(lengths)
    vads = ("ivad", "irm2") if mode == "local" else ("irm1", "irm2")
    arrs = make_batch(B, K, C, L, seed0=1000 + 10 * (("local",) + MODES).index(mode))
    Td = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    poisoned = []
    for a in arrs:
        a = a.copy()
        for b, Lb in enumerate(lengths):
            a[b, ..., Lb:] = np.nan
        poisoned.append(Td(a))
    y, s, n = poisoned
    kw = dict(lambda_cor=0.95, block=block, lag=1, ref_mic=1, n_fft=n_fft, vads=vads, mask_for_z=mode)
    spy = Spy(monkeypatch)
    got = online.online_tango(y, s=s, n=n, lengths=lengths, **kw)
    torch.cuda.synchronize()
    assert sites_of("test_uneven_batches") <= spy.sites(), sorted(spy.sites())
    names = MAIN + DIAG + ("masks_z", "mask_w")
    assert set(got) == set(names)
    for nm in names:
        assert bool(torch.isfinite(torch.view_as_real(got[nm]) if got[nm].is_complex() else got[nm]).all()), nm
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        Jb = -(-Tb // block)
        sl = slice(b, b + 1)
        alone = online.online_tango(Td(arrs[0][sl, ..., :Lb]), s=Td(arrs[1][sl, ..., :Lb]), n=Td(arrs[2][sl, ..., :Lb]),
                                    **kw)
        for nm in names:
            cut = Jb if nm in ("W1", "W2") else Tb
            assert torch.equal(got[nm][b, :, :cut], alone[nm][0]), (mode, nm, b)
            assert not bool(got[nm][b, :, cut:].any()), (mode, nm, b, "not 0 past the end")


# ---- 6. scoring -----------------------------------------------------------------------------------------------------
def test_scores_match_the_hand_composition(dev):
    """post.tango_scores(..., stoi=True, lengths=) on post.to_time(online_tango(s=, n=, lengths=)) equals the scores
    of the hand composition of tests/test_gpu_online_lengths.py (filter_sum_blocks of W1 / W2 on S, N) for the same
    inputs; a K = 2 batch scores finite."""
    from disco_b200 import online, ops, post
    from disco_b200.synth import make_batch, make_utterance
    from test_gpu_stoi import speechlike
    fs, L, n_fft, block = 16000, 3 * 16000, 512, 8
    B, K, C = 3, 1, 2
    lengths = [L, 40000, 33001]
    frames = ops.n_frames(np.asarray(lengths), n_fft)
    ys, ss, ns = zip(*[make_utterance(b, K, C, L, gate_period=6000) for b in range(B)])
    y, s, n = np.stack(ys), np.stack(ss), np.stack(ns)
    for b, Lb in enumerate(lengths):
        for a in (y, s, n):
            a[b, ..., Lb:] = 0
    s_dry = np.stack([speechlike(50 + b, L + 100, period=6000, gain=0.05) for b in range(B)])
    n_dry = (0.02 * np.random.default_rng(4).standard_normal((B, L + 100))).astype(np.float32)
    Td = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    # the hand composition
    S, N = (ops.stft_lengths(Td(a), lengths, n_fft) for a in (s, n))
    masks = (ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), "irm1"),
             ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), "irm2"))
    hand = online.online_tango(Td(y), masks, block=block, n_fft=n_fft, lengths=lengths)
    for nm, W, X in (("z_s", "W1", S), ("z_n", "W1", N), ("sf", "W2", S), ("nf", "W2", N)):
        hand[nm] = ops.filter_sum_blocks(hand[W], X, None, block, 1, True, 0, n_fft, frames=frames)[0]
    out = online.online_tango(Td(y), block=block, n_fft=n_fft, lengths=lengths, s=Td(s), n=Td(n),
                              vads=("irm1", "irm2"))
    for nm in hand:
        assert torch.equal(out[nm], hand[nm]), nm
    score = lambda o, yy, s0, n0, sd, nd, lens: post.tango_scores(
        yy, s0, n0, sd, nd, post.to_time(o, yy.shape[-1], n_fft=n_fft, layout="TF", lengths=lens), fs, stoi=True,
        lengths=lens)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        got = score(out, Td(y[:, :, 0]), Td(s[:, :, 0]), Td(n[:, :, 0]), Td(s_dry), Td(n_dry), lengths)
        want = score(hand, Td(y[:, :, 0]), Td(s[:, :, 0]), Td(n[:, :, 0]), Td(s_dry), Td(n_dry), lengths)
        for g, w in zip(got, want):
            assert g.keys() == w.keys()
            for key in w:
                assert bool(torch.isfinite(g[key]).all()), key
                assert bool(((g[key] - w[key]).abs() <= 1e-12 * w[key].abs()).all()), (key, g[key], w[key])
        # K = 2: the outputs hold the images of both nodes, and every score is finite
        y2, s2, n2 = make_batch(2, 2, 2, 40000, seed0=77)
        lens2 = [40000, 30001]
        for b, Lb in enumerate(lens2):
            for a in (y2, s2, n2):
                a[b, ..., Lb:] = 0
        sd2, nd2 = Td(s_dry[:2, :40000]), Td(n_dry[:2, :40000])
        o2 = online.online_tango(Td(y2), block=block, n_fft=n_fft, lengths=lens2, s=Td(s2), n=Td(n2),
                                 vads=("irm1", "irm2"), mask_for_z="distant")
        res = score(o2, Td(y2[:, :, 0]), Td(s2[:, :, 0]), Td(n2[:, :, 0]), sd2, nd2, lens2)
        for r in res:
            for key, v in r.items():
                assert v.shape[:2] == (2, 2), key
                assert bool(torch.isfinite(v).all()), key
