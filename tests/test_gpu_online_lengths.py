"""Online (recursive) Tango on batches of utterances of different lengths: ops.scm_recursive / ops.filter_sum_blocks
with frames=, online_mwf(frames=) and online_tango(lengths=).

The kernels compute every (group, block, bin) entry from that group's own frames in a fixed order, so an utterance of
an uneven batch is the utterance run alone, bit for bit (torch.equal), with exact zeros past its frames and blocks.
At the spectrum level that holds for every channel stack; through online_tango it needs K * C even (the STFT
transforms signals 2p, 2p + 1 together, so pairs must not span two utterances)."""
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
TS, NS = 4, 4     # online_wide.cu: frames per ring stage, stages in the ring


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def _cplx(rng, *s):
    return (rng.standard_normal(s) + 1j * rng.standard_normal(s)).astype(np.complex64)


def _frames(P, T, wide):
    """Frame counts at the block edges (kP - 1, kP, kP + 1), one short of a block, the full T, and for the staged
    engine one frame either side of a ring stage and a block straddling the ring's wrap."""
    fr = [T, 2 * P - 1, 2 * P, 2 * P + 1, max(1, P // 2), 1]
    if wide:
        fr += [TS * 3 - 1, TS * 3 + 1, TS * NS - 1, TS * NS + 2]
    return [min(max(f, 1), T) for f in fr]


def _hermitian(rng, B, K, F, D):
    A = _cplx(rng, B, K, F, D, D)
    return (np.einsum("...ij,...kj->...ik", A, A.conj()) * 0.05 + np.eye(D) * 0.01).astype(np.complex64)


def _check_utterance(got, alone, b, Tb, Jb):
    """got: batched online_mwf dict, alone: the dict of utterance b run alone."""
    for nm in ("z", "zn"):
        assert torch.equal(got[nm][b, :, :Tb], alone[nm][0]), nm
        assert not bool(got[nm][b, :, Tb:].any()), nm
    for nm in ("Rss", "Rnn", "W"):
        assert torch.equal(got[nm][b, :, :Jb], alone[nm][0]), nm
        assert not bool(got[nm][b, :, Jb:].any()), nm


# (K, C, step 2, block, lag, lambda, R0): every D = 1..16 as one stack (step 1), and D = 9..16 over node splits
MWF_CASES = ([(1, D, False, 8, 1, 0.95, D % 2 == 0) for D in range(1, 17)] +
             [(8, 2, True, 8, 1, 0.95, False), (2, 8, True, 5, 1, 0.9, True), (5, 5, True, 4, 2, 0.98, False),
              (3, 8, True, 8, 0, 0.95, False), (9, 2, True, 5, 1, 0.95, False), (4, 8, True, 8, 1, 0.0, False),
              (6, 6, True, 1, 1, 0.95, False), (12, 1, True, 8, 1, 0.95, False), (7, 7, True, 8, 2, 0.98, True),
              (3, 12, True, 4, 1, 0.95, False), (8, 8, True, 8, 1, 0.95, False), (16, 1, True, 5, 0, 0.9, False),
              (9, 8, True, 8, 1, 0.95, True),
              (1, 4, False, 1, 0, 0.0, True), (1, 4, False, 64, 1, 0.98, False), (3, 2, True, 64, 2, 0.95, True),
              (2, 3, True, 1, 2, 0.98, False)])


@pytest.mark.parametrize("K,C,step2,block,lag,lam,r0", MWF_CASES,
                         ids=["k%dc%d%s-p%d-l%d-lam%g%s" % (c[0], c[1], "z" if c[2] else "", c[3], c[4], c[5],
                                                           "-r0" if c[6] else "") for c in MWF_CASES])
def test_online_mwf_frames_alone_equals_batched(dev, K, C, step2, block, lag, lam, r0):
    """online_mwf(frames=) per utterance == online_mwf on its first T_b frames alone, under torch.equal, with exact
    zeros past T_b (z, zn) and J_b (Rss, Rnn, W); the masks past T_b are NaN and never read."""
    from disco_b200 import online
    rng = np.random.default_rng(100 * K + C + block)
    D = C + K - 1 if step2 else C
    Ks = K if step2 else 2
    F = 129
    T = 150 if block == 64 else max(4 * block + 3, TS * NS + 6)
    frames = _frames(block, T, D >= 9)
    B = len(frames)
    Y = torch.from_numpy(_cplx(rng, B, Ks, C, T, F)).to(dev)
    Z = torch.from_numpy(_cplx(rng, B, K, T, F)).to(dev) if step2 else None
    m = torch.from_numpy(rng.uniform(0.05, 0.95, size=(B, Ks, T, F)).astype(np.float32)).to(dev)
    for b, Tb in enumerate(frames):
        m[b, :, Tb:] = float("nan")
    R0 = None
    if r0:
        R0 = tuple(torch.from_numpy(_hermitian(rng, B, Ks, F, D)).to(dev) for _ in range(2))
    kw = dict(lambda_cor=lam, block=block, lag=lag, ref=D - 1, n_fft=256)
    got = online.online_mwf(Y, m, Z, R0=R0, frames=frames, **kw)
    for nm in ("z", "zn", "W"):
        assert bool(torch.isfinite(got[nm]).all()), nm
    for b, Tb in enumerate(frames):
        sl = slice(b, b + 1)
        alone = online.online_mwf(Y[sl, :, :, :Tb].contiguous(), m[sl, :, :Tb].contiguous(),
                                  None if Z is None else Z[sl, :, :Tb].contiguous(),
                                  R0=None if R0 is None else tuple(r[sl].contiguous() for r in R0), **kw)
        _check_utterance(got, alone, b, Tb, -(-Tb // block))


@pytest.mark.parametrize("K,C,block", [(1, 4, 8), (3, 2, 5), (8, 2, 8), (1, 12, 4), (2, 9, 8)])
def test_ops_read_nothing_past_the_end(dev, K, C, block):
    """NaN in Y, Z and the mask past each T_b and in W past each J_b: every output is finite and equal to the clean
    run (node subsets and Z included)."""
    from disco_b200 import ops
    rng = np.random.default_rng(7 * K + C)
    T, F = 4 * block + TS * NS + 3, 257
    D = C + K - 1
    frames = _frames(block, T, D >= 9)
    B = len(frames)
    sel = [k for k in range(K) if k % 2 == 0] if K > 1 else None
    Ks = len(sel) if sel else K
    J = -(-T // block)
    Y = torch.from_numpy(_cplx(rng, B, Ks, C, T, F)).to(dev)
    Z = torch.from_numpy(_cplx(rng, B, K, T, F)).to(dev) if K > 1 else None
    m = torch.from_numpy(rng.uniform(0.05, 0.95, size=(B, Ks, T, F)).astype(np.float32)).to(dev)
    W = torch.from_numpy(_cplx(rng, B, Ks, J, F, D)).to(dev)
    Yp, mp, Wp = Y.clone(), m.clone(), W.clone()
    Zp = None if Z is None else Z.clone()
    nan = float("nan")
    for b, Tb in enumerate(frames):
        Yp[b, ..., Tb:, :] = complex(nan, nan)
        mp[b, :, Tb:] = nan
        Wp[b, :, -(-Tb // block):] = complex(nan, nan)
        if Zp is not None:
            Zp[b, :, Tb:] = complex(nan, nan)
    kw = dict(block=block, n_fft=512, node_sel=sel, frames=frames)
    clean = ops.scm_recursive(Y, m, Z, 0.95, R0=None, power=2, **kw)
    dirty = ops.scm_recursive(Yp, mp, Zp, 0.95, R0=None, power=2, **kw)
    fclean = ops.filter_sum_blocks(W, Y, Z, lag=1, ref=0, **kw)
    fdirty = ops.filter_sum_blocks(Wp, Yp, Zp, lag=1, ref=0, **kw)
    for a, c in zip(clean + fclean, dirty + fdirty):
        assert bool(torch.isfinite(c).all())
        assert torch.equal(a, c)
    for b, Tb in enumerate(frames):
        assert not bool(fclean[0][b, :, Tb:].any()) and not bool(fclean[1][b, :, Tb:].any())
        assert not bool(clean[0][b, :, -(-Tb // block):].any())


def _utterances(B, K, C, L, lengths, seed):
    from disco_b200.synth import make_batch
    y, s, n = make_batch(B, K, C, L, seed0=seed)
    for b, Lb in enumerate(lengths):
        for a in (y, s, n):
            a[b, ..., Lb:] = 0
    return y, s, n


def _masks(rng, B, K, T, F, frames):
    out = []
    for _ in range(2):
        m = rng.uniform(0.05, 0.95, size=(B, K, T, F)).astype(np.float32)
        for b, Tb in enumerate(frames):
            m[b, :, Tb:] = np.nan                 # online_tango must select these away, not multiply them
        out.append(m)
    return out


def _lengths_for(frames, n_fft):
    hop = n_fft // 2
    return [(Tb - 1) * hop + 7 for Tb in frames]   # 1 + L_b // hop = T_b


# (K, C, n_fft, block, lag, lambda, R0): K * C even
TANGO_CASES = [(1, 2, 512, 8, 1, 0.95, False), (1, 4, 256, 1, 0, 0.98, True), (2, 2, 1024, 64, 2, 0.0, False),
               (4, 4, 512, 8, 1, 0.95, False), (2, 3, 256, 5, 1, 0.9, True), (8, 2, 256, 8, 1, 0.95, False),
               (1, 10, 256, 4, 2, 0.98, True), (2, 8, 512, 8, 0, 0.95, False)]


def _tango_inputs(dev, K, C, n_fft, block, seed, extra=()):
    hop = n_fft // 2
    T = 150 if block == 64 else max(4 * block + 3, TS * NS + 6)
    frames = _frames(block, T, C + K - 1 >= 9 or C >= 9) + list(extra)
    frames = [max(f, 3) for f in frames]                 # lengths > n_fft / 2
    frames[0] = T
    lengths = _lengths_for(frames, n_fft)
    L = lengths[0]
    B, F = len(frames), n_fft // 2 + 1
    y, _, _ = _utterances(B, K, C, L, lengths, seed)
    rng = np.random.default_rng(seed)
    mz, mw = _masks(rng, B, K, 1 + L // hop, F, frames)
    Td = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return Td(y), Td(mz), Td(mw), frames, lengths, L


@pytest.mark.parametrize("K,C,n_fft,block,lag,lam,r0", TANGO_CASES,
                         ids=["k%dc%d-n%d-p%d-l%d-lam%g%s" % (c[0], c[1], c[2], c[3], c[4], c[5], "-r0" if c[6] else "")
                              for c in TANGO_CASES])
def test_online_tango_alone_equals_batched(dev, K, C, n_fft, block, lag, lam, r0):
    """online_tango(lengths=) of utterance b, sliced to [:T_b], == online_tango of y[b, ..., :L_b] alone (torch.equal)
    for yf, z_y, zn and W1, W2 up to J_b; exact zeros after."""
    from disco_b200 import online
    y, mz, mw, frames, lengths, L = _tango_inputs(dev, K, C, n_fft, block, 300 + 10 * K + C)
    B, F = y.shape[0], n_fft // 2 + 1
    R0 = None
    if r0:
        R0 = tuple(torch.from_numpy(_hermitian(np.random.default_rng(5), B, K, F, C)).to(dev) for _ in range(2))
    kw = dict(lambda_cor=lam, block=block, lag=lag, ref_mic=C - 1, n_fft=n_fft)
    got = online.online_tango(y, (mz, mw), R0=R0, lengths=lengths, **kw)
    for nm in ("yf", "z_y", "zn"):
        assert bool(torch.isfinite(got[nm]).all()), nm
    for b, (Tb, Lb) in enumerate(zip(frames, lengths)):
        sl = slice(b, b + 1)
        alone = online.online_tango(y[sl, ..., :Lb].contiguous(), (mz[sl, :, :Tb].contiguous(),
                                    mw[sl, :, :Tb].contiguous()),
                                    R0=None if R0 is None else tuple(r[sl].contiguous() for r in R0), **kw)
        Jb = -(-Tb // block)
        for nm in ("yf", "z_y", "zn"):
            assert torch.equal(got[nm][b, :, :Tb], alone[nm][0]), (nm, b)
            assert not bool(got[nm][b, :, Tb:].any()), (nm, b)
        for nm in ("W1", "W2"):
            assert torch.equal(got[nm][b, :, :Jb], alone[nm][0]), (nm, b)
            assert not bool(got[nm][b, :, Jb:].any()), (nm, b)


def test_online_tango_odd_stack_against_float64(dev):
    """K * C odd (the STFT pairs span utterances): online_tango(lengths=) against the float64 composition of the
    reference's per-frame recursion on each trimmed utterance, from the block whose filter saw >= 4 D frames on."""
    from disco_b200 import online
    from oracle import librosa_np, online_np, tango_np
    K, C, n_fft, block = 1, 3, 256, 4
    y, mz, mw, frames, lengths, L = _tango_inputs(dev, K, C, n_fft, block, 77)
    got = online.online_tango(y, (mz, mw), block=block, n_fft=n_fft, lambda_cor=0.9, lengths=lengths)
    yn = y.cpu().numpy().astype(np.float64)
    fsel = [0, 37, 128]
    for b, (Tb, Lb) in enumerate(zip(frames, lengths)):
        start = -(-4 * C // block) + 1                     # first block whose filter (lag 1) saw >= 4 D frames
        if Tb <= start * block + 2:
            continue
        X = np.stack([librosa_np.stft(yn[b, 0, c, :Lb], n_fft=n_fft, hop_length=n_fft // 2) for c in range(C)])
        m = mz[b, 0, :Tb].cpu().numpy().T.astype(np.float64)
        z, _, _, _ = online_np.online_mwf(X[:, fsel], m[fsel], tango_np.spatial_correlation_matrix,
                                          tango_np.intern_filter, lambda_cor=0.9, block=block)
        want = z[:, start * block:]
        have = got["z_y"][b, 0, start * block:Tb].cpu().numpy().T[fsel]
        assert np.linalg.norm(np.abs(have) - np.abs(want)) <= 1e-4 * np.linalg.norm(want), b
        assert not bool(got["z_y"][b, :, Tb:].any())


def test_online_tango_independent_of_the_rest_of_the_batch(dev):
    """Another utterance's length and the order of the batch do not move utterance b's outputs."""
    from disco_b200 import online
    K, C, n_fft, block = 2, 2, 512, 8
    y, mz, mw, frames, lengths, L = _tango_inputs(dev, K, C, n_fft, block, 901)
    kw = dict(block=block, n_fft=n_fft)
    base = online.online_tango(y, (mz, mw), lengths=lengths, **kw)
    b = 2
    other = list(lengths)
    other[1] = lengths[1] + 2 * (n_fft // 2) if lengths[1] + n_fft < L else lengths[1] - n_fft // 2
    mz2, mw2 = mz.clone(), mw.clone()
    T1 = 1 + other[1] // (n_fft // 2)
    for m in (mz2, mw2):
        m[1, :, :T1] = torch.nan_to_num(m[1, :, :T1], nan=0.5)
    alt = online.online_tango(y, (mz2, mw2), lengths=other, **kw)
    perm = list(reversed(range(y.shape[0])))
    rev = online.online_tango(y[perm].contiguous(), (mz[perm].contiguous(), mw[perm].contiguous()),
                              lengths=[lengths[i] for i in perm], **kw)
    pb = perm.index(b)
    for nm in ("yf", "z_y", "zn", "W1", "W2"):
        assert torch.equal(base[nm][b], alt[nm][b]), nm
        assert torch.equal(base[nm][b], rev[nm][pb]), nm


def test_online_tango_uniform_lengths_take_the_uniform_path(dev):
    """lengths=None and every length = L give today's online_tango bit for bit."""
    from disco_b200 import online
    from disco_b200.synth import make_batch
    B, K, C, L, n_fft = 3, 2, 2, 6000, 512
    y, _, _ = make_batch(B, K, C, L, seed0=55)
    rng = np.random.default_rng(3)
    T, F = 1 + L // 256, 257
    mz, mw = (torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev) for _ in range(2))
    y = torch.from_numpy(y).to(dev)
    a = online.online_tango(y, (mz, mw))
    for lengths in ([L] * B, np.full(B, L, dtype=np.int64), torch.full((B,), L)):
        c = online.online_tango(y, (mz, mw), lengths=lengths)
        for nm in a:
            assert torch.equal(a[nm], c[nm]), nm


def test_online_ops_validate_frames(dev):
    from disco_b200 import ops
    Y = torch.zeros(2, 1, 2, 10, 129, dtype=torch.complex64, device=dev)
    W = torch.zeros(2, 1, 2, 129, 2, dtype=torch.complex64, device=dev)
    for bad in ([10, 0], [11, 5], [10]):
        with pytest.raises(ValueError):
            ops.scm_recursive(Y, None, None, block=8, n_fft=256, frames=bad)
        with pytest.raises(ValueError):
            ops.filter_sum_blocks(W, Y, None, block=8, n_fft=256, frames=bad)
    with pytest.raises(TypeError):
        ops.scm_recursive(Y, None, None, block=8, n_fft=256, frames=np.array([10.0, 5.0]))


def test_online_tango_lengths_to_time_and_scores(dev):
    """post.to_time(..., layout='TF', lengths=) and post.tango_scores(..., stoi=True, lengths=) on the online outputs
    (target / noise images through the same per-block filters) against each utterance alone: the spectra bit for bit,
    the time signals to float32 rounding (the batch's iSTFT pairs signals of different utterances), the scores of the
    same time signals to 1e-9 (BSS, STOI) and 1e-6 dB (fw_snr, fw_sd), as the offline lengths= tests hold them."""
    from disco_b200 import online, ops, post
    from disco_b200.synth import make_utterance
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
    S, N = (ops.stft_lengths(Td(a), lengths, n_fft) for a in (s, n))      # the images' spectra, masks of them
    masks = (ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), "irm1"),
             ops.tf_mask(S[:, :, 0].contiguous(), N[:, :, 0].contiguous(), "irm2"))

    def run(yy, S_, N_, masks_, lens):
        out = online.online_tango(yy, masks_, block=block, n_fft=n_fft, lengths=lens)
        fr = None if lens is None else frames
        for nm, W, X in (("z_s", "W1", S_), ("z_n", "W1", N_), ("sf", "W2", S_), ("nf", "W2", N_)):
            out[nm] = ops.filter_sum_blocks(out[W], X, None, block, 1, True, 0, n_fft, frames=fr)[0]
        return out

    out = run(Td(y), S, N, masks, lengths)
    times = post.to_time(out, L, n_fft=n_fft, layout="TF", lengths=lengths)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        res, resz = post.tango_scores(Td(y[:, :, 0]), Td(s[:, :, 0]), Td(n[:, :, 0]), Td(s_dry), Td(n_dry), times, fs,
                                      stoi=True, lengths=lengths)
        for b, (Lb, Tb) in enumerate(zip(lengths, frames)):
            sl = slice(b, b + 1)
            cut = lambda X: X[sl, ..., :Tb, :].contiguous()
            o1 = run(Td(y[sl, ..., :Lb]), cut(S), cut(N), tuple(cut(m) for m in masks), None)
            for nm in o1:
                if nm in ("W1", "W2"):
                    continue
                assert torch.equal(out[nm][b, :, :Tb], o1[nm][0]), nm
            t1 = post.to_time(o1, Lb, n_fft=n_fft, layout="TF")
            for nm in t1:
                a, c = times[nm][b, :, :Lb], t1[nm][0]
                assert float((a - c).abs().max()) <= 1e-5 * float(c.abs().max()), nm
                assert not bool(times[nm][b, :, Lb:].any()), nm
            tb = {k: v[sl, ..., :Lb].contiguous() for k, v in times.items()}
            r1, rz1 = post.tango_scores(Td(y[sl, :, 0, :Lb]), Td(s[sl, :, 0, :Lb]), Td(n[sl, :, 0, :Lb]),
                                        Td(s_dry[sl]), Td(n_dry[sl]), tb, fs, stoi=True)
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
