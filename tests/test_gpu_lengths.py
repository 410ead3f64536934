"""Batches of utterances of different lengths (the `lengths=` argument): the length-aware STFT and iSTFT against the
plain ones on the trimmed signals, bit for bit under the same pairing, through guarded outputs; and tango_batched /
post.to_time on uneven batches against the float64 oracle and against each utterance processed alone."""
import numpy as np
import pytest
import torch

from conftest import TOL, rel_l2_mag
from test_gpu_post_instances import Guarded, _call, _p, cplx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _lengths_ptrs(lengths, dev):
    from disco_b200 import _lib
    host = np.ascontiguousarray(lengths, dtype=np.int32)
    return torch.from_numpy(host).to(dev), host, host.ctypes.data_as(_lib.c_int_p)


def _signals(rng, lengths, L):
    x = np.zeros((len(lengths), L), np.float32)
    for i, Lb in enumerate(lengths):
        x[i, :Lb] = rng.standard_normal(Lb).astype(np.float32)
    return x


def _frames64(x, n_fft):
    """Reflect-padded, Hann-windowed frames of x (float64) [T, n_fft] (librosa center=True)."""
    H = n_fft // 2
    xp = np.pad(np.asarray(x, np.float64), H, mode="reflect")
    T = 1 + len(x) // H
    w = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(n_fft) / n_fft)
    return np.stack([xp[t * H:t * H + n_fft] for t in range(T)]) * w


def _length_sets(n_fft, L):
    H = n_fft // 2
    return {
        "pairs_share": [L, L, H + 1, H + 1, L - 3 * H - 7, L - 3 * H - 7, L - 1],            # odd count: last alone
        "pairs_differ": [L, H + 1, L - 1, L - H, L - 2 * H + 5, L - 5 * H - H // 3, H + 2, L],
    }


@pytest.mark.parametrize("n_fft", [256, 512, 1024])
@pytest.mark.parametrize("kind", ["pairs_share", "pairs_differ"])
def test_stft_lengths_matches_trimmed_stft(dev, n_fft, kind):
    from disco_b200 import ops
    H, F = n_fft // 2, n_fft // 2 + 1
    L = 20 * H + 77
    lengths = _length_sets(n_fft, L)[kind]
    rng = np.random.default_rng(n_fft + len(kind))
    x = _signals(rng, lengths, L)
    xd = torch.from_numpy(x).to(dev)
    n_sig, T = len(lengths), 1 + L // H
    g = Guarded(dev)
    Y = g.new((n_sig, T, F), torch.complex64)
    ld, _, hp = _lengths_ptrs(lengths, dev)
    _call("disco_stft_lengths", _p(xd), _p(ld), hp, _p(Y), n_sig, L, n_fft)
    g.check("stft_lengths n_fft=%d %s" % (n_fft, kind))
    Yh = Y.cpu().numpy()
    u = 2.0 ** -24
    eps = np.sqrt(2) * (4 * np.log2(n_fft) + 6) * u
    for s, Lb in enumerate(lengths):
        Tb = 1 + Lb // H
        assert not np.any(Yh[s, Tb:]), (s, "frames past T_b not zero")
        p = s ^ 1
        partner = p < n_sig
        if partner and lengths[p] == Lb:
            pair = np.stack([x[min(s, p), :Lb], x[max(s, p), :Lb]])
            ref = ops.stft(torch.from_numpy(pair).to(dev), n_fft)[s - min(s, p)].cpu().numpy()
            assert np.array_equal(Yh[s, :Tb], ref), (s, "not bit-identical to the trimmed pair")
        elif not partner:
            ref = ops.stft(torch.from_numpy(x[s:s + 1, :Lb].copy()).to(dev), n_fft)[0].cpu().numpy()
            assert np.array_equal(Yh[s, :Tb], ref), (s, "not bit-identical to the trimmed signal alone")
        else:
            # the STFT bound of DESIGN §2 over the pair's padded frames (the partner's are zero once it has ended)
            fa = _frames64(x[s, :Lb], n_fft)
            Lp = lengths[p]
            fb = np.zeros_like(fa)
            fp = _frames64(x[p, :Lp], n_fft)
            m = min(len(fp), Tb)
            fb[:m] = fp[:m]
            bound = eps * (np.abs(fa).sum(1) + np.abs(fb).sum(1))
            exact = np.fft.rfft(fa, axis=1)
            err = np.abs(Yh[s, :Tb].astype(np.complex128) - exact).max(1)
            assert np.all(err <= bound), (s, float((err / bound).max()))


@pytest.mark.parametrize("n_fft", [256, 512, 1024])
@pytest.mark.parametrize("kind", ["pairs_share", "pairs_differ"])
def test_istft_lengths_matches_trimmed_istft(dev, n_fft, kind):
    from disco_b200 import ops
    H, F = n_fft // 2, n_fft // 2 + 1
    L = 70 * H + 31                     # several chunks in the plan of the longest signal
    lengths = _length_sets(n_fft, L)[kind]
    rng = np.random.default_rng(7 * n_fft + len(kind))
    n_sig, T = len(lengths), 1 + L // H
    Yd = torch.from_numpy(cplx(rng, n_sig, T, F)).to(dev)
    g = Guarded(dev)
    x = g.new((n_sig, L), torch.float32)
    ld, _, hp = _lengths_ptrs(lengths, dev)
    _call("disco_istft_lengths", _p(Yd), _p(ld), hp, _p(x), n_sig, T, L, n_fft)
    g.check("istft_lengths n_fft=%d %s" % (n_fft, kind))
    xh = x.cpu().numpy()
    for s, Lb in enumerate(lengths):
        Tb = 1 + Lb // H
        assert not np.any(xh[s, Lb:]), (s, "samples past L_b not zero")
        p = s ^ 1
        if p < n_sig and lengths[p] == Lb:
            lo = min(s, p)
            ref = ops.istft(Yd[lo:lo + 2, :Tb].contiguous(), Lb, n_fft)[s - lo]
        else:
            ref = ops.istft(Yd[s:s + 1, :Tb].contiguous(), Lb, n_fft)[0]
        assert np.array_equal(xh[s, :Lb], ref.cpu().numpy()), s
    # the op: per-utterance lengths repeated over the trailing axes
    Y4 = Yd[:6].reshape(3, 2, T, F).contiguous()
    per = [lengths[0], lengths[2], lengths[4]]
    x4 = ops.istft_lengths(Y4, per, L, n_fft)
    x4b = ops.istft_lengths(Y4, np.repeat(per, 2).reshape(3, 2), L, n_fft)
    assert torch.equal(x4, x4b)


# ---- the beamformer --------------------------------------------------------------------------------------------

CASES = {
    # name: (K, C, vads, mask_for_z, external masks)
    "k1c4_same_mask": (1, 4, ("irm1", "irm1"), "local", False),
    "k1c4_two_masks": (1, 4, ("irm1", "irm2"), "local", False),
    "k1c2_iam1": (1, 2, ("iam1", "irm1"), "local", False),
    "k2c2_irm1": (2, 2, ("irm1", "irm1"), "local", False),
    "k3c2_distant": (3, 2, ("irm1", "irm1"), "distant", False),
    "k2c2_compressed": (2, 2, ("irm1", "irm1"), "compressed", False),
    "k2c2_ibm1": (2, 2, ("ibm1", "ibm1"), "local", False),
    "k2c2_ivad": (2, 2, ("ivad", "ivad"), "local", False),
    "k2c3_masks": (2, 3, None, "local", True),
    "k2c2_oracle_refs": (2, 2, ("irm1", "irm1"), "use_oracle_refs", False),
    "k2c2_oracle_zs": (2, 2, ("irm1", "irm1"), "use_oracle_zs", False),
    "k2c2_callable_mask_w": (2, 2, None, "local", True),
}
OUTS = ("yf", "z_y", "zn")


def _batch(K, C, L, lengths, seed):
    from disco_b200.synth import make_batch
    y, s, n = make_batch(len(lengths), K, C, L, seed0=seed)
    for b, Lb in enumerate(lengths):
        for a in (y, s, n):
            a[b, ..., Lb:] = 0
    return y, s, n


def _run(dev, y, s, n, vads, mfz, masks, lengths, callable_w=False):
    from disco_b200.tango import tango_batched
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if masks is not None:
        mw = t(masks[1])
        if callable_w:     # a step-2 estimator called with (Y, z_y, zn) after step 1
            return tango_batched(t(y), masks=(t(masks[0]), lambda Y, z_y, zn: mw), mask_for_z=mfz, lengths=lengths)
        return tango_batched(t(y), masks=(t(masks[0]), mw), mask_for_z=mfz, lengths=lengths)
    return tango_batched(t(y), t(s), t(n), vads=vads, mask_for_z=mfz, lengths=lengths)


@pytest.mark.parametrize("name", sorted(CASES))
def test_tango_lengths(dev, name):
    from oracle import tango_f64
    K, C, vads, mfz, ext = CASES[name]
    L = 14000
    lengths = [L, 9001, 11519]
    T, F = 1 + L // 256, 257
    y, s, n = _batch(K, C, L, lengths, seed=300 + len(name))
    masks = None
    if ext:
        rng = np.random.default_rng(5)
        masks = tuple(rng.uniform(0.05, 0.95, size=(len(lengths), K, T, F)).astype(np.float32) for _ in range(2))
    cw = "callable" in name
    if cw:                 # whatever the estimator returns past an utterance's frames is replaced by 0
        for b, Lb in enumerate(lengths):
            masks[1][b, :, 1 + Lb // 256:] = np.nan
    out = _run(dev, y, s, n, vads, mfz, masks, lengths, cw)
    for nm, v in out.items():
        assert bool(torch.isfinite(v).all()), nm
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // 256
        for nm, v in out.items():                      # [B, K, F, T]
            assert not bool(v[b, ..., Tb:].any()), (nm, b, "not zero past T_b")
        yb, sb, nb = y[b:b + 1, ..., :Lb], s[b:b + 1, ..., :Lb], n[b:b + 1, ..., :Lb]
        mb = None if masks is None else tuple(m[b:b + 1, :, :Tb] for m in masks)
        solo = _run(dev, yb, sb, nb, vads, mfz, mb, None, cw)
        for nm in ("masks_z", "mask_w"):
            got, ref = out[nm][b, ..., :Tb].cpu().numpy(), solo[nm][0].cpu().numpy()
            if vads is not None and "ivad" in vads:
                assert np.mean(got != ref) < 1e-3, nm
            else:
                assert np.allclose(got, ref, rtol=5e-6, atol=1e-6), nm
        if "ibm" in name:      # exactly singular bins: only the masks are compared (as in test_gpu_tango.py)
            continue
        for nm in OUTS:
            got, ref = out[nm][b, ..., :Tb].cpu().numpy(), solo[nm][0].cpu().numpy()
            if not np.any(ref):    # e.g. an 'ivad' mask of 1 in every frame: R_nn = 0, w = 0 exactly (DESIGN §2)
                assert not np.any(got), (nm, b)
                continue
            assert rel_l2_mag(got, ref) < TOL, (nm, b, rel_l2_mag(got, ref))
        if mfz == "local" and vads is not None and vads[0][:3] in ("irm", "iam") and vads[1][:3] in ("irm", "iam") \
                or ext:
            mz, mw = out["masks_z"][b, ..., :Tb].cpu().numpy(), out["mask_w"][b, ..., :Tb].cpu().numpy()
            ref = tango_f64.offline_tango(y[b, ..., :Lb], masks=(mz, mw))
            for nm in OUTS:
                got = out[nm][b, ..., :Tb].cpu().numpy()
                for k in range(K):
                    assert rel_l2_mag(got[k], ref[nm][k]) < TOL, (nm, b, k, rel_l2_mag(got[k], ref[nm][k]))


def test_tango_lengths_uniform_is_bit_identical(dev):
    """All lengths equal to L take the uniform routes: bit-identical to lengths=None (fused routes included)."""
    for K, C, vads in ((1, 4, ("irm1", "irm2")), (2, 2, ("irm1", "irm1")), (1, 2, ("irm1", "irm1"))):
        L = 12000
        y, s, n = _batch(K, C, L, [L, L], seed=11)
        a = _run(dev, y, s, n, vads, "local", None, None)
        b = _run(dev, y, s, n, vads, "local", None, [L, L])
        assert a.keys() == b.keys()
        for nm in a:
            assert torch.equal(a[nm], b[nm]), nm


def test_tango_lengths_independent_of_the_rest_of_the_batch(dev):
    """An utterance's outputs move by rounding only when another utterance, its length or L_max change."""
    L = 13000
    lengths = [9000, 12000, 13000]
    y, s, n = _batch(2, 2, L, lengths, seed=41)
    base = _run(dev, y, s, n, ("irm1", "irm1"), "local", None, lengths)
    y2, s2, n2 = _batch(2, 2, L, lengths, seed=42)
    y2[0], s2[0], n2[0] = y[0], s[0], n[0]
    other = _run(dev, y2, s2, n2, ("irm1", "irm1"), "local", None, [9000, 10500, 13000])
    Lm = 15000
    pad = lambda a: np.concatenate([a, np.zeros(a.shape[:-1] + (Lm - L,), a.dtype)], axis=-1)
    longer = _run(dev, pad(y), pad(s), pad(n), ("irm1", "irm1"), "local", None, lengths)
    Tb = 1 + 9000 // 256
    for nm in OUTS:
        ref = base[nm][0, ..., :Tb].cpu().numpy()
        for alt in (other, longer):
            got = alt[nm][0, ..., :Tb].cpu().numpy()
            assert rel_l2_mag(got, ref) < TOL, nm
        assert not bool(longer[nm][0, ..., Tb:].any())


def test_to_time_lengths(dev):
    from disco_b200 import ops, post
    L = 14000
    lengths = [9001, L, 11519]
    y, s, n = _batch(2, 2, L, lengths, seed=77)
    out = _run(dev, y, s, n, ("irm1", "irm1"), "local", None, lengths)
    times = post.to_time(out, L, lengths=lengths)
    for nm, x in times.items():
        assert x.shape == (3, 2, L)
        for b, Lb in enumerate(lengths):
            Tb = 1 + Lb // 256
            assert not bool(x[b, :, Lb:].any()), nm
            spec = ops.transpose_last2(out[nm][b, :, :, :Tb].contiguous())
            assert torch.equal(x[b, :, :Lb], ops.istft(spec, Lb)), (nm, b)


# ---- scores -----------------------------------------------------------------------------------------------------

def test_si_sdr_and_snr_ignore_trailing_zeros(dev):
    from disco_b200 import post
    rng = np.random.default_rng(12)
    L, Lb = 9000, 6001
    a = np.zeros((2, L), np.float32)
    b = np.zeros((2, L), np.float32)
    a[:, :Lb] = rng.standard_normal((2, Lb))
    b[:, :Lb] = a[:, :Lb] + 0.3 * rng.standard_normal((2, Lb))
    T = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    for fn in (post.si_sdr, post.snr, post.sd):
        full, trim = fn(T(a), T(b)), fn(T(a[:, :Lb]), T(b[:, :Lb]))
        assert torch.allclose(full, trim, rtol=1e-9, atol=0), fn.__name__


def test_stoi_pairs_lengths_against_oracle(dev):
    from disco_b200 import stoi
    from oracle import stoi_np
    from test_gpu_stoi import energy_margin, speechlike
    for fs in (10000, 16000):
        L = 3 * fs
        lengths = [L, 2 * fs + 4321, fs + 2001]
        x = np.stack([speechlike(3 + i, L, period=fs // 2) for i in range(3)])
        y = (x + 0.3 * np.random.default_rng(fs).standard_normal(x.shape)).astype(np.float32)
        for i, Lb in enumerate(lengths):
            x[i, Lb:] = 0
            y[i, Lb:] = 7.0      # past its end a degraded row is ignored, whatever it holds
        T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        pairs = [(0, 0), (1, 1), (2, 2), (1, 0)]
        with pytest.raises(ValueError):                       # degraded 0 paired with cleans of two lengths
            stoi.stoi_pairs(T(x), T(y), pairs, fs, lengths=lengths)
        got = stoi.stoi_pairs(T(x), T(y), pairs[:3], fs, lengths=lengths).cpu().numpy()
        for i, Lb in enumerate(lengths):
            assert energy_margin(stoi_np.to_10k(x[i, :Lb], fs)) >= 1e-9
            want = stoi_np.stoi(x[i, :Lb], y[i, :Lb], fs)
            assert abs(got[i] - want) <= 1e-9, (fs, i, got[i], want)
        # every length = L: the uniform result, bit for bit
        y[:] = x + 0.3
        a = stoi.stoi_pairs(T(x), T(y), pairs[:3], fs)
        b = stoi.stoi_pairs(T(x), T(y), pairs[:3], fs, lengths=[L, L, L])
        assert torch.equal(a, b)


def test_resample_lengths_matches_trimmed(dev):
    from disco_b200 import stoi
    fs, L = 16000, 20011
    lengths = [L, 12345, 300]
    rng = np.random.default_rng(1)
    x = rng.standard_normal((3, L)).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    got = stoi.to_10k(T(x), fs, lengths=lengths)
    for i, Lb in enumerate(lengths):
        n10 = int(stoi.length_10k(Lb, fs))
        ref = stoi.to_10k(T(x[i:i + 1, :Lb]), fs)[0]
        assert ref.shape[-1] == n10
        assert torch.equal(got[i, :n10], ref), i
        assert not bool(got[i, n10:].any())


def test_tango_scores_lengths_match_each_utterance_alone(dev):
    """tango_scores(..., lengths=) per (utterance, node) against tango_scores of that utterance alone, trimmed, on the
    same time signals: BSS within 1e-9 relative, fw_snr / fw_sd within 1e-6 dB, the STOI deltas within 1e-9."""
    import warnings
    from disco_b200 import post
    from disco_b200.synth import make_utterance
    from disco_b200.tango import tango_batched
    from test_gpu_stoi import speechlike
    fs, L = 16000, 3 * 16000
    B, K, C = 3, 2, 2
    lengths = [L, 40000, 33001]
    ys, ss, ns = zip(*[make_utterance(b, K, C, L, gate_period=6000) for b in range(B)])
    y, s, n = np.stack(ys), np.stack(ss), np.stack(ns)
    for b, Lb in enumerate(lengths):
        for a in (y, s, n):
            a[b, ..., Lb:] = 0
    s_dry = np.stack([speechlike(50 + b, L + 100, period=6000, gain=0.05) for b in range(B)])
    n_dry = (0.02 * np.random.default_rng(4).standard_normal((B, L + 100))).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    out = tango_batched(T(y), T(s), T(n), lengths=lengths)
    times = post.to_time(out, L, lengths=lengths)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        res, resz = post.tango_scores(T(y[:, :, 0]), T(s[:, :, 0]), T(n[:, :, 0]), T(s_dry), T(n_dry), times, fs,
                                      stoi=True, lengths=lengths)
        for b, Lb in enumerate(lengths):
            tb = {k: v[b:b + 1, ..., :Lb].contiguous() for k, v in times.items()}
            r1, rz1 = post.tango_scores(T(y[b:b + 1, :, 0, :Lb]), T(s[b:b + 1, :, 0, :Lb]), T(n[b:b + 1, :, 0, :Lb]),
                                        T(s_dry[b:b + 1]), T(n_dry[b:b + 1]), tb, fs, stoi=True)
            for got_all, want_all in ((res, r1), (resz, rz1)):
                assert got_all.keys() == want_all.keys()
                for key in want_all:
                    got, want = got_all[key][b].cpu().numpy(), want_all[key][0].cpu().numpy()
                    assert np.all(np.isfinite(got)), key
                    if key.startswith(("sdr", "sir", "sar")):
                        assert np.all(np.abs(got - want) <= 1e-9 * np.abs(want)), (key, b, got, want)
                    elif key.startswith(("snr", "fw_sd")):
                        assert np.all(np.abs(got - want) <= 1e-6), (key, b, got, want)
                    else:
                        assert np.all(np.abs(got - want) <= 1e-9), (key, b, got, want)
