"""STOI on the device (csrc/stoi.cu, disco_b200/stoi.py, post.tango_scores(stoi=True), compat.stoi) against the float64
oracle (oracle/stoi_np.py, pystoi 0.3's algorithm) and, for the resampler, against scipy.signal.resample_poly.

Every output of the C ABI calls below lands between NaN-patterned guard bands: every output word must be written and
no guard word may change.  Tolerances: a resampled sample within (taps per phase + 2) 2^-53 sum |up h| |x| of scipy's
(one rounding per product and per addition of the polyphase sum, plus scipy's own); a score within 1e-9 of the
oracle's (both are float64 restatements of the same operations, summed in different orders); a kept-frame count equal
to the oracle's, on inputs whose frame energies stay at least 1e-9 dB away from the 40 dB threshold."""
import warnings

import numpy as np
import pytest
import torch
from scipy.signal import resample_poly

from oracle import stoi_np

pytestmark = pytest.mark.gpu

SENT64 = 0x7FF8DEADDEADBEEF
SENT32 = -0x21524111          # 0xDEADBEEF
G = 256                       # guard words on each side


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def guarded(n, dtype, dev):
    """(buffer, view of its n middle words): the buffer pre-filled with the sentinel pattern."""
    if dtype == torch.float64:
        buf = torch.full((n + 2 * G,), SENT64, dtype=torch.int64, device=dev)
        return buf, buf[G:G + n].view(torch.float64)
    buf = torch.full((n + 2 * G,), SENT32, dtype=torch.int32, device=dev)
    return buf, buf[G:G + n]


def check_guards(buf, n):
    s = SENT64 if buf.dtype == torch.int64 else SENT32
    assert bool((buf[:G] == s).all()) and bool((buf[G + n:] == s).all()), "guard word changed"
    assert int((buf[G:G + n] == s).sum()) == 0, "output word not written"


def speechlike(seed, L, period=4000, noise=0.0, gain=1.0):
    """Gated low-passed noise (on 60 % of every period, phase-shifted by the seed) plus optional white noise."""
    rng = np.random.default_rng(seed)
    x = np.convolve(rng.standard_normal(L + 31), np.hanning(32), mode="valid")[:L]
    x *= ((np.arange(L) + seed * 997) % period) < 0.6 * period
    return (gain * (x + noise * rng.standard_normal(L))).astype(np.float32)


# ---- resampler ---------------------------------------------------------------------------------------------------

def resample_abi(x, taps, up, down, dev):
    from disco_b200 import _lib, ops
    n_sig, L = x.shape
    n_out = -(-L * up // down)
    buf, y = guarded(n_sig * n_out, torch.float64, dev)
    xt = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    tt = torch.from_numpy(taps).to(dev)
    _lib.check(_lib.load().disco_resample_poly(ops._ptr(xt), ops._ptr(y), ops._ptr(tt), len(taps), up, down, n_sig, L,
                                               ops._stream()))
    torch.cuda.synchronize()
    check_guards(buf, n_sig * n_out)
    got = y.view(n_sig, n_out).cpu().numpy()
    assert torch.equal(ops.resample_poly(xt, tt, up, down), y.view(n_sig, n_out))
    return got


def resample_ok(got, x, taps, up, down):
    x64 = x.astype(np.float64)
    want = resample_poly(x64, up, down, axis=-1, window=taps)
    assert got.shape == want.shape
    mag = resample_poly(np.abs(x64), up, down, axis=-1, window=np.abs(taps))       # sum |up h| |x| per output
    bound = (-(-len(taps) // up) + 2) * 2.0 ** -53 * mag
    return bool(np.all(np.abs(got - want) <= bound)), np.max(np.abs(got - want) - bound)


@pytest.mark.parametrize("fs", [8000, 16000, 22050, 44100, 48000])
def test_resampler_against_scipy(dev, fs):
    from disco_b200 import stoi
    taps, up, down = stoi.resample_taps(fs)
    rng = np.random.default_rng(fs)
    for L in (1, 7 * down, 7 * down - 1, 7 * down + 1, 3 * fs // 2 + 1):
        x = rng.standard_normal((2, L)).astype(np.float32)
        got = resample_abi(x, taps, up, down, dev)
        ok, worst = resample_ok(got, x, taps, up, down)
        assert ok, (fs, L, worst)


def test_resampler_checker_rejects_misalignment(dev):
    """A one-sample shift of the output, or the gain `up` left out, is far outside the bound."""
    from disco_b200 import stoi
    taps, up, down = stoi.resample_taps(16000)
    x = speechlike(5, 4000)[None]
    got = resample_abi(x, taps, up, down, dev)
    assert resample_ok(got, x, taps, up, down)[0]
    assert not resample_ok(np.roll(got, 1, axis=-1), x, taps, up, down)[0]
    assert not resample_ok(got / up, x, taps, up, down)[0]


# ---- STOI through the C ABI --------------------------------------------------------------------------------------

def stoi_abi(cleans, degraded, pairs, dev):
    """disco_stoi on float64 10 kHz signals with guard-banded outputs; also checks ops.stoi gives the same bits."""
    from disco_b200 import _lib, ops
    lib = _lib.load()
    C, L = cleans.shape
    D, P = degraded.shape[0], len(pairs)
    T = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
    xc, xd, pr = T(cleans, np.float64), T(degraded, np.float64), T(pairs, np.int32)
    bd, d = guarded(P, torch.float64, dev)
    bs, n_sel = guarded(C, torch.int32, dev)
    bf, n_frames = guarded(P, torch.int32, dev)
    ws_bytes = lib.disco_stoi_workspace(C, P, L)
    ws = torch.full((ws_bytes // 8 + 1,), float("nan"), dtype=torch.float64, device=dev)
    _lib.check(lib.disco_stoi(ops._ptr(xc), ops._ptr(xd), ops._ptr(pr), ops._ptr(d), ops._ptr(n_sel),
                              ops._ptr(n_frames), C, D, P, L, ops._ptr(ws), ws_bytes, ops._stream()))
    torch.cuda.synchronize()
    for b, n in ((bd, P), (bs, C), (bf, P)):
        check_guards(b, n)
    d2, s2, f2 = ops.stoi(xc, xd, pr)
    assert torch.equal(d, d2) and torch.equal(n_frames, f2)
    named = sorted(set(int(c) for c, _ in pairs))
    assert torch.equal(n_sel[named], s2[named])
    return d.cpu().numpy(), n_sel.cpu().numpy(), n_frames.cpu().numpy()


def energy_margin(x):
    e = stoi_np.frame_energies(x)
    return np.min(np.abs(np.max(e) - stoi_np.DYN_RANGE - e))


def selection_cases():
    """(name, clean) at 10 kHz, float32-representable."""
    L = 30000
    cases = []
    x = speechlike(1, L, period=5000)
    x[:3000] = 0                                                   # silence at the start ...
    x[14000:17000] = 0                                             # ... in the middle ...
    x[-2500:] = 0                                                  # ... and at the end
    cases.append(("gated", x))
    cases.append(("gated_tail77", speechlike(2, L + 77, period=3000)))      # (L - 256) mod 128 != 0
    cases.append(("zero", np.zeros(L, np.float32)))
    one = np.zeros(L, np.float32)
    one[128 * 100:128 * 100 + 256] = speechlike(3, 256, period=1 << 30)    # a single loud frame
    cases.append(("one_frame", one))
    for n_stft in (29, 30, 31):                                    # every frame loud: n_sel = n_stft + 1
        cases.append(("frames%d" % n_stft, speechlike(10 + n_stft, 256 + 128 * n_stft, period=1 << 30)))
    cases.append(("frames30_tail5", speechlike(40, 256 + 128 * 30 + 5, period=1 << 30)))
    return cases


@pytest.mark.parametrize("name,clean", selection_cases())
def test_selection_and_score_at_10k(dev, name, clean):
    x = clean.astype(np.float64)
    assert energy_margin(x) >= 1e-9, name
    rng = np.random.default_rng(len(x))
    degraded = np.stack([x + 0.3 * rng.standard_normal(len(x)) * x.std(),            # noisy
                         np.zeros_like(x),                                          # y = 0
                         -x,                                                        # y = -x
                         x + 5.0 * rng.standard_normal(len(x)) * max(x.std(), 1e-3)]  # heavy noise
                        ).astype(np.float32).astype(np.float64)
    pairs = [(0, j) for j in range(4)]
    d, n_sel, n_frames = stoi_abi(x[None], degraded, pairs, dev)
    keep = stoi_np.selection(x)
    assert n_sel[0] == len(keep), (name, n_sel[0], len(keep))
    assert np.all(n_frames == len(keep) - 1)
    for j in range(4):
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            want = stoi_np.stoi_10k(x, degraded[j])
        assert abs(d[j] - want) <= 1e-9, (name, j, d[j], want)
    if len(keep) - 1 < 30:
        assert np.all(d == 1e-5)
    else:
        assert d[1] == 0.0


@pytest.mark.parametrize("fs,seconds", [(10000, 3), (16000, 3), (8000, 4), (16000, 10)])
def test_stoi_against_oracle(dev, fs, seconds):
    from disco_b200 import stoi
    L = fs * seconds
    x = np.stack([speechlike(s, L, period=fs // 2) for s in (1, 2)])
    n = np.random.default_rng(fs).standard_normal((2, L)).astype(np.float32)
    y = np.stack([x[0] + 0.2 * n[0], x[1] + 3.0 * n[1]]).astype(np.float32)
    if seconds == 10:
        x, y = x[:1], y[:1]
    T = lambda a: torch.from_numpy(a).to(dev)
    got = stoi.stoi(T(x), T(y), fs).cpu().numpy()
    for i in range(len(x)):
        assert energy_margin(stoi_np.to_10k(x[i], fs)) >= 1e-9
        want = stoi_np.stoi(x[i], y[i], fs)
        assert abs(got[i] - want) <= 1e-9, (fs, i, got[i], want)
    if seconds == 3:
        for yy in (np.zeros_like(x), -x):
            got = stoi.stoi(T(x), T(yy), fs).cpu().numpy()
            for i in range(len(x)):
                assert abs(got[i] - stoi_np.stoi(x[i], yy[i], fs)) <= 1e-9


def test_short_signal_warns_and_errors(dev):
    from disco_b200 import stoi
    x = torch.from_numpy(speechlike(7, 256 + 128 * 28, period=1 << 30)).to(dev)
    with pytest.warns(RuntimeWarning):
        d = stoi.stoi(x, x + 0.1, 10000)
    assert d.item() == 1e-5
    with pytest.raises(ValueError):
        stoi.stoi(x[:255], x[:255], 10000)


def test_bit_identical_across_batch_rerun_and_chunks(dev):
    from disco_b200 import ops
    L = 25000
    cleans = np.stack([speechlike(s, L, period=3000 + 500 * s) for s in range(3)]).astype(np.float64)
    rng = np.random.default_rng(0)
    deg = (np.repeat(cleans, 2, axis=0) + 0.5 * rng.standard_normal((6, L))).astype(np.float32).astype(np.float64)
    pairs = np.array([(c, 2 * c + k) for c in range(3) for k in range(2)] + [(2, 0), (0, 5)], np.int32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    xc, xd, pr = T(cleans), T(deg), T(pairs)
    a = ops.stoi(xc, xd, pr)
    b = ops.stoi(xc, xd, pr)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    perm = [7, 3, 0, 5, 1, 6, 2, 4]                          # other batch positions, cleans reordered
    c = ops.stoi(xc[[2, 0, 1]].contiguous(), xd, T(np.stack([[[1, 2, 0][p[0]], p[1]] for p in pairs[perm]]).astype(np.int32)))
    assert torch.equal(c[0], a[0][perm]) and torch.equal(c[2], a[2][perm])
    assert torch.equal(c[1], a[1][[2, 0, 1]])
    old = ops.STOI_WORKSPACE_CAP
    try:
        for cap in (1, 3 * ops._lib.load().disco_stoi_workspace(1, 1, L)):   # one pair / three pairs per chunk
            ops.STOI_WORKSPACE_CAP = cap
            e = ops.stoi(xc, xd, pr)
            assert all(torch.equal(u, v) for u, v in zip(a, e)), cap
    finally:
        ops.STOI_WORKSPACE_CAP = old


# ---- checkers reject subtly wrong results ------------------------------------------------------------------------

def variant_d(x, y, shift=0, edges=None, last=False):
    """The oracle's score with one step changed: the kept-frame list shifted by `shift` frames, other band edges, or
    the last full STFT frame included."""
    w = stoi_np.hann()
    hop = 128
    keep = stoi_np.selection(x) + shift
    keep = keep[(keep >= 0) & (keep * hop + 256 <= len(x))]
    fx = np.array([w * x[f * hop:f * hop + 256] for f in keep])
    fy = np.array([w * y[f * hop:f * hop + 256] for f in keep])
    xs, ys = stoi_np._overlap_and_add(fx, hop), stoi_np._overlap_and_add(fy, hop)
    stop = len(xs) - 256 + (1 if last else 0)
    sx = np.array([np.fft.rfft(w * xs[i:i + 256], 512) for i in range(0, stop, hop)])
    sy = np.array([np.fft.rfft(w * ys[i:i + 256], 512) for i in range(0, stop, hop)])
    edges = edges or stoi_np.band_edges()
    X = np.array([np.sqrt((np.abs(sx[:, a:b]) ** 2).sum(1)) for a, b in edges])
    Y = np.array([np.sqrt((np.abs(sy[:, a:b]) ** 2).sum(1)) for a, b in edges])
    J = X.shape[1] - 29
    xs_ = np.array([X[:, m:m + 30] for m in range(J)])
    ys_ = np.array([Y[:, m:m + 30] for m in range(J)])
    nx = np.linalg.norm(xs_, axis=2, keepdims=True)
    yp = np.minimum(ys_ * nx / (np.linalg.norm(ys_, axis=2, keepdims=True) + stoi_np.EPS), xs_ * (1 + 10 ** 0.75))
    yp = yp - yp.mean(2, keepdims=True)
    xc = xs_ - xs_.mean(2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + stoi_np.EPS
    xc /= np.linalg.norm(xc, axis=2, keepdims=True) + stoi_np.EPS
    return np.sum(yp * xc) / (J * 15)


def test_checkers_reject_subtly_wrong_results(dev):
    L = 30000
    x = speechlike(21, L, period=4000).astype(np.float64)
    y = (x + 0.4 * np.random.default_rng(1).standard_normal(L) * x.std()).astype(np.float32).astype(np.float64)
    d, _, _ = stoi_abi(x[None], y[None], [(0, 0)], dev)
    assert abs(variant_d(x, y) - stoi_np.stoi_10k(x, y)) <= 1e-12      # the variant machinery is faithful
    assert abs(d[0] - variant_d(x, y)) <= 1e-9
    edges = stoi_np.band_edges()
    wrong = {"selection shifted by one frame": variant_d(x, y, shift=1),
             "band edge off by one bin": variant_d(x, y, edges=edges[:7] + [(edges[7][0], edges[7][1] + 1)] + edges[8:]),
             "last STFT frame included": variant_d(x, y, last=True)}
    for what, v in wrong.items():
        assert abs(d[0] - v) > 1e-9, what


# ---- tango_scores and compat -------------------------------------------------------------------------------------

def test_tango_scores_stoi_against_oracle(dev):
    from disco_b200 import post
    from disco_b200.synth import make_utterance
    from disco_b200.tango import tango_batched
    fs, L = 16000, 3 * 16000
    B, K, C = 2, 2, 2
    ys, ss, ns = zip(*[make_utterance(b, K, C, L, gate_period=6000) for b in range(B)])
    y, s, n = np.stack(ys), np.stack(ss), np.stack(ns)
    s_dry = np.stack([speechlike(50 + b, L + 100, period=6000, gain=0.05) for b in range(B)])
    n_dry = (0.02 * np.random.default_rng(4).standard_normal((B, L + 100))).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    times = post.to_time(tango_batched(T(y), T(s), T(n)), L)
    args = (T(y[:, :, 0]), T(s[:, :, 0]), T(n[:, :, 0]), T(s_dry), T(n_dry), times, fs)
    res0, resz0 = post.tango_scores(*args)
    res, resz = post.tango_scores(*args, stoi=True)
    for base, full in ((res0, res), (resz0, resz)):
        assert set(full) - set(base) == ({"delta_stoi_cnv", "delta_stoi_dry"} if full is res
                                         else {"delta_stoi", "delta_stoi_dry"})
        for k in base:
            assert torch.equal(base[k], full[k]), k
    tn = {k: v.cpu().numpy() for k, v in times.items()}
    for b in range(B):
        for k in range(K):
            cut = lambda a: a[fs:L]
            sk, sd, yk, sh, szh = cut(s[b, k, 0]), cut(s_dry[b]), cut(y[b, k, 0]), cut(tn["yf"][b, k]), cut(tn["z_y"][b, k])
            st = lambda c, e: stoi_np.stoi(c, e, fs)
            want = {"delta_stoi_cnv": st(sk, sh) - st(sk, yk), "delta_stoi_dry": st(sd, sh) - st(sd, yk)}
            wantz = {"delta_stoi": st(sk, szh) - st(sk, yk), "delta_stoi_dry": st(sd, szh) - st(sd, yk)}
            for d, w in ((res, want), (resz, wantz)):
                for key, v in w.items():
                    assert abs(d[key][b, k].item() - v) <= 2e-9, (b, k, key, d[key][b, k].item(), v)


def test_compat_stoi(dev):
    from disco_b200.compat import stoi
    x = speechlike(8, 32000, period=8000)
    y = (x + 0.5 * np.random.default_rng(2).standard_normal(32000) * x.std()).astype(np.float32)
    got = stoi.stoi(x, y, 16000)
    assert isinstance(got, float)
    assert abs(got - stoi_np.stoi(x, y, 16000)) <= 1e-9
    assert abs(stoi.stoi(x.astype(np.float64), y.astype(np.float64), 16000) - got) == 0.0
    with pytest.raises(Exception, match="same length"):
        stoi.stoi(x, y[:-1], 16000)
    with pytest.raises(ValueError):
        stoi.stoi(x[:300], y[:300], 16000)          # 188 samples at 10 kHz
    with pytest.raises(NotImplementedError):
        stoi.stoi(x, y, 16000, extended=True)
