"""Batched Tango on ragged arrays (disco_b200/ragged.py): the reference's ragged fixtures inside batches, every
utterance against the per-utterance adapter tango.offline_tango, uniform channel counts against tango_batched, uneven
lengths, online Tango node by node against the float64 composition, bit-exact batching, and scoring."""
import warnings

import numpy as np
import pytest
import torch

from conftest import TOL, load_golden, record_parity, rel_l2, rel_l2_mag
from oracle.make_golden import NAMES, TANGO_CASES, case_inputs, digest

pytestmark = pytest.mark.gpu

MODES = ("local", "distant", "compressed", "use_oracle_refs", "use_oracle_zs", "previous")


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


def _pack(lists):
    """[node][channel] 1-D signals -> [M, L] float32, node k's microphones at rows off_k .. off_k + C_k - 1."""
    return np.stack([np.asarray(ch, dtype=np.float32) for node in lists for ch in node])


def _utterance(seed, chans, L, gate=0):
    """(y, s, n) as [node][channel] lists of one utterance of the ragged geometry chans."""
    from disco_b200.synth import make_utterance
    y, s, n = make_utterance(seed, len(chans), max(chans), L, gate_period=gate)
    pick = lambda a: [[a[k, c] for c in range(chans[k])] for k in range(len(chans))]
    return pick(y), pick(s), pick(n)


def _batch(dev, utts):
    """list of (y, s, n) lists -> y, s, n [B, M, L] device tensors."""
    return tuple(torch.from_numpy(np.stack([_pack(u[i]) for u in utts])).to(dev) for i in range(3))


def _np(t):
    return t.detach().cpu().numpy()


def _masks_close(got, want, vad):
    """The masks of two runs whose spectra differ in the last float32 bits (the STFT pairs other signals): binary
    masks agree but for a rare flip at the threshold, soft ones within TOL relative L2 (a float32 FFT's error is
    relative to the frame, so a bin far below its frame's energy can move its mask by far more than that); 'iam' =
    |s| / |s + n| is unbounded where s + n cancels and is judged on the 99.5th percentile, as tests/test_gpu_tango.py
    judges it."""
    if want.dtype == bool or (vad or "").startswith("ibm"):
        return np.mean((got != 0) != (want != 0)) < 1e-3
    if "iam" in (vad or ""):
        return np.percentile(np.abs(got - want) / np.maximum(1.0, np.abs(want)), 99.5) < 5e-6
    return rel_l2(got, want) < TOL


def _parity(case, nm, k, got, want, truth):
    """The parity rule of tests/conftest.py with `want` (another route on the same utterance) as the reference: within
    TOL of it, or, where `want` itself is further than TOL from float64 (ill-conditioned masks), as close to float64
    as `want` is, or within TOL of float64 itself (a noise image nf is small and ill-conditioned, so two float32 routes
    can sit 1e-5 apart while both are closer than that to exact arithmetic).  truth() -> {name: [K, F, T]} float64
    outputs of the utterance, evaluated only when needed."""
    e = rel_l2_mag(got, want)
    ours = theirs = None
    if e >= TOL:
        f64 = truth()[nm][k]
        ours, theirs = rel_l2_mag(got, f64), rel_l2_mag(want, f64)
    ok = record_parity(case, nm, k, err_ref=e, err_f64=ours, ref_f64=theirs, note="reference = " + truth.__doc__)
    return ok or (ours is not None and ours < TOL), (e, ours, theirs)


def _f64(lists, masks, mode, n_fft, doc, vads=("irm1", "irm1")):
    """Lazy float64 Tango (oracle/tango_np.py, double precision, per bin) of one utterance under the given masks
    ((mask_z[K], mask_w[K]) of (F, T) arrays; vads[0] is the mask type of the 'compressed' exchange): the yardstick
    where two float32 routes differ by more than TOL."""
    cache = {}

    def truth():
        if not cache:
            from oracle import tango_np
            mk = tuple([np.asarray(m, np.float64) for m in ms] for ms in masks)
            res = tango_np.offline_tango(*lists, vads=vads, mask_for_z=mode, n_fft=n_fft,
                                         n_hop=n_fft // 2, granularity="bin", double=True, masks=mk)
            cache.update({nm: np.array(v) for nm, v in zip(NAMES, res) if not nm.startswith("mask")})
        return cache
    truth.__doc__ = doc
    return truth


# ---- 1. the reference's ragged fixtures, placed inside batches ------------------------------------------------------
RAGGED_CASES = ["tango_k3_ragged_local", "tango_k3_ragged_distant", "tango_k3_ragged_compressed"]


@pytest.mark.parametrize("B,pos", [(3, 0), (4, 2), (5, 4)])
@pytest.mark.parametrize("name", RAGGED_CASES)
def test_reference_fixtures_inside_a_batch(dev, name, B, pos):
    """The fixture's utterance at position pos of a batch of B ragged utterances: yf, sf, nf, z_y of every node meet
    the parity rule against the reference's stored outputs (and float64 where the fixture does not hold them)."""
    from disco_b200.ragged import tango_ragged
    from test_gpu_tango import f64_truth
    seed, chans, L, vads, mfz, keep = TANGO_CASES[name]
    g = load_golden(name)
    y, s, n = case_inputs(seed, chans, L, vads)
    assert digest(y) == str(g["input_sha256"])
    utts = [_utterance(500 + 7 * b + seed, chans, L) for b in range(B)]
    utts[pos] = (y, s, n)
    yd, sd, nd = _batch(dev, utts)
    out = tango_ragged(yd, chans, sd, nd, vads=vads, mask_for_z=mfz)
    truth = f64_truth(name, y, s, n, vads, mfz) or {}
    for nm in ("yf", "sf", "nf", "z_y"):
        for k in range(len(chans)):
            got = _np(out[nm][pos, k])
            key = "%s_%d" % (nm, k)
            err = rel_l2_mag(got, g[key]) if key in g else None
            ours = theirs = None
            if nm in truth:
                ours = rel_l2_mag(got, truth[nm][k])
                theirs = rel_l2_mag(g[key], truth[nm][k]) if key in g else None
            assert err is not None or ours is not None, key
            ok = record_parity("ragged_batch_%s_B%d_at%d" % (name, B, pos), nm, k, err_ref=err, err_f64=ours,
                               ref_f64=theirs, note="tango_ragged, fixture inside a batch")
            assert ok, (key, err, ours, theirs)


# ---- 2. every utterance against the adapter ------------------------------------------------------------------------
GEOMS = ([2, 3, 2], [1, 4], [4, 2, 2, 1], [8, 2])
MASKS = ("irm1", "ibm1", "iam1", "ivad", "external")
ADAPTER = [(g, m, (256, 512, 1024)[(i + j) % 3], MASKS[(i + 2 * j) % len(MASKS)])
           for i, g in enumerate(GEOMS) for j, m in enumerate(MODES)]


def _external_masks(rng, B, K, T, F):
    return tuple(rng.uniform(0.05, 0.95, size=(B, K, T, F)).astype(np.float32) for _ in range(2))


@pytest.mark.parametrize("chans,mode,n_fft,masks", ADAPTER,
                         ids=["%s-%s-n%d-%s" % ("".join(map(str, c[0])), c[1], c[2], c[3]) for c in ADAPTER])
def test_every_utterance_matches_the_adapter(dev, chans, mode, n_fft, masks):
    """Each utterance of a B = 3 batch against tango.offline_tango on that utterance alone: the seven spectra within
    the parity rule per node, the masks to float32 rounding (identical for binary masks)."""
    from disco_b200.ragged import tango_ragged
    from disco_b200.tango import offline_tango
    B, L, K = 3, 16000, len(chans)
    T, F = 1 + L // (n_fft // 2), n_fft // 2 + 1
    utts = [_utterance(40 + 5 * b + sum(chans) + n_fft, chans, L, gate=2000 if masks == "ivad" else 0)
            for b in range(B)]
    yd, sd, nd = _batch(dev, utts)
    kw = dict(mask_for_z=mode, n_fft=n_fft)
    ext = None
    if masks == "external":
        ext = _external_masks(np.random.default_rng(n_fft + K), B, K, T, F)
        out = tango_ragged(yd, chans, sd, nd, masks=tuple(torch.from_numpy(m).to(dev) for m in ext), **kw)
        vads = ("irm1", "irm1")
    else:
        vads = (masks, masks)
        out = tango_ragged(yd, chans, sd, nd, vads=vads, **kw)
    for b in range(B):
        mk = None if ext is None else tuple([m[b, k].T for k in range(K)] for m in ext)
        ref = dict(zip(NAMES, offline_tango(*utts[b], list(vads), None, mode, n_fft=n_fft, masks=mk)))
        truth = _f64(utts[b], (ref["masks_z"], ref["mask_w"]), mode, n_fft, "tango.offline_tango on the utterance alone",
                     vads if vads[0] != "ivad" else ("irm1", "irm1"))
        for nm in NAMES:
            for k in range(K):
                got, want = _np(out[nm][b, k]), np.asarray(ref[nm][k])
                assert got.shape == want.shape, (nm, k)
                if nm.startswith("mask"):
                    assert _masks_close(got, want, None if ext is not None else vads[0]), (nm, b, k)
                    continue
                ok, errs = _parity("ragged_vs_adapter_%s_%s_n%d_%s_b%d" % ("".join(map(str, chans)), mode, n_fft,
                                                                           masks, b), nm, k, got, want, truth)
                assert ok, (nm, b, k, errs)


@pytest.mark.parametrize("K,C,mode,n_fft", [(3, 2, "local", 512), (2, 4, "distant", 256), (4, 3, "compressed", 1024),
                                            (1, 4, "local", 512)])
def test_uniform_channels_match_tango_batched(dev, K, C, mode, n_fft):
    """channels = [C] * K is the uniform array: tango_ragged == tango_batched within the parity rule (tango_batched
    takes its fused routes, so the bits differ)."""
    from disco_b200.ragged import tango_ragged
    from disco_b200.synth import make_batch
    from disco_b200.tango import tango_batched
    B, L = 3, 12000
    y, s, n = (torch.from_numpy(a).to(dev) for a in make_batch(B, K, C, L, seed0=70 + K * C))
    want = tango_batched(y, s, n, vads=("irm1", "irm2"), mask_for_z=mode, n_fft=n_fft)
    got = tango_ragged(y.reshape(B, K * C, L), [C] * K, s.reshape(B, K * C, L), n.reshape(B, K * C, L),
                       vads=("irm1", "irm2"), mask_for_z=mode, n_fft=n_fft)
    assert set(got) == set(want), (sorted(got), sorted(want))
    for b in range(B):
        lists = tuple([[_np(a[b, k, c]) for c in range(C)] for k in range(K)] for a in (y, s, n))
        truth = _f64(lists, tuple([_np(m[b, k]) for k in range(K)] for m in (want["masks_z"], want["mask_w"])), mode,
                     n_fft, "tango_batched")
        for nm in want:
            for k in range(K):
                g, w = _np(got[nm][b, k]), _np(want[nm][b, k])
                if nm.startswith("mask"):
                    assert _masks_close(g, w, "irm1"), (nm, b, k)
                    continue
                ok, errs = _parity("ragged_uniform_k%dc%d_%s_n%d_b%d" % (K, C, mode, n_fft, b), nm, k, g, w, truth)
                assert ok, (nm, b, k, errs)


def test_callable_step2_mask(dev):
    """A callable mask_w receives microphone 0 of every node [B, K, 1, T, F] and z_y, zn [B, K, T, F] after step 1;
    returning the mask it would have been given makes the call identical to the external-mask one."""
    from disco_b200 import ops
    from disco_b200.ragged import tango_ragged
    chans, B, L, n_fft = [2, 3, 1], 2, 8000, 512
    T, F = 1 + L // 256, 257
    yd, _, _ = _batch(dev, [_utterance(90 + b, chans, L) for b in range(B)])
    mz, mw = (torch.from_numpy(m).to(dev) for m in _external_masks(np.random.default_rng(4), B, 3, T, F))
    want = tango_ragged(yd, chans, masks=(mz, mw), n_fft=n_fft)
    seen = {}

    def est(Y0, z_y, zn):
        seen["Y0"], seen["z"] = Y0, (z_y, zn)
        return mw
    got = tango_ragged(yd, chans, masks=(mz, est), n_fft=n_fft)
    assert seen["Y0"].shape == (B, 3, 1, T, F) and seen["z"][0].shape == (B, 3, T, F)
    rows = [0, 2, 5]                                            # microphone 0 of each node
    assert rel_l2(_np(seen["Y0"][:, :, 0]), _np(ops.stft(yd[:, rows].contiguous(), n_fft))) < 1e-6
    assert torch.equal(seen["z"][0], ops.transpose_last2(want["z_y"]))
    for nm in want:
        assert torch.equal(got[nm], want[nm]), nm


# ---- 3. uneven lengths -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,vads", [("local", ("ivad", "irm2")), ("compressed", ("irm1", "irm2")),
                                       ("use_oracle_refs", ("irm1", "irm1"))])
def test_uneven_lengths(dev, mode, vads):
    """lengths=: every output is exactly 0 from T_b on, NaN in y, s, n past each length reaches no output, and each
    utterance matches its lone run on the trimmed signals within the parity rule."""
    from disco_b200.ragged import tango_ragged
    chans, n_fft = [2, 3, 1], 512
    hop = n_fft // 2
    lengths = [12000, 9000 + 37, 6400, 12000 - 3 * hop]
    L, B = max(lengths), len(lengths)
    utts = [_utterance(300 + b, chans, L, gate=2000) for b in range(B)]
    clean = _batch(dev, utts)
    poisoned = []
    for a in clean:
        a = a.clone()
        for b, Lb in enumerate(lengths):
            a[b, :, Lb:] = float("nan")
        poisoned.append(a)
    kw = dict(vads=vads, mask_for_z=mode, n_fft=n_fft, out_layout="TF")
    got = tango_ragged(*poisoned[:1], chans, *poisoned[1:], lengths=lengths, **kw)
    for nm, v in got.items():
        assert bool(torch.isfinite(torch.view_as_real(v) if v.is_complex() else v).all()), nm
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        for nm, v in got.items():
            assert not bool(v[b, :, Tb:].any()), (nm, b, "not 0 past the end")
        alone = tango_ragged(*(a[b:b + 1, :, :Lb].contiguous() for a in clean[:1]), chans,
                             *(a[b:b + 1, :, :Lb].contiguous() for a in clean[1:]), **kw)
        lists = tuple([[_np(a[b, r, :Lb]) for r in rows] for rows in ([0, 1], [2, 3, 4], [5])] for a in clean)
        tr = lambda a: np.swapaxes(_np(a[0]), -1, -2)                     # [K, T, F] -> [K, F, T]
        truth = _f64(lists, (tr(alone["masks_z"]), tr(alone["mask_w"])), mode, n_fft,
                     "tango_ragged on the utterance alone")
        for nm in alone:
            for k in range(len(chans)):
                g, w = _np(got[nm][b, k, :Tb]), _np(alone[nm][0, k])
                if nm.startswith("mask"):
                    assert _masks_close(g, w, vads[0] if nm == "masks_z" else vads[1]), (nm, b, k)
                    continue
                ok, errs = _parity("ragged_lengths_%s_b%d" % (mode, b), nm, k, g.T, w.T, truth)
                assert ok, (nm, b, k, errs)


# ---- 4. online Tango ------------------------------------------------------------------------------------------------
def _start(D, block, lag):
    """First frame compared with float64: the block whose filter saw >= 4 D frames (tests/test_gpu_online_eval.py)."""
    return (-(-4 * D // block) + lag) * block


def _blocks(W, X, block, lag, ref):
    T = X.shape[2]
    j = np.arange(T) // block - lag
    out = X[ref].astype(np.complex128).copy()
    live = j >= 0
    out[:, live] = np.einsum("tfd,dft->ft", np.conj(W[j[live]]), X[:, :, live])
    return out


def _spec64(node, n_fft, fsel):
    """[C, L] float32 -> [C, len(fsel), T] complex128."""
    from oracle import librosa_np
    return np.stack([librosa_np.stft(np.asarray(c, np.float64), n_fft=n_fft, hop_length=n_fft // 2)[fsel]
                     for c in node])


def f64_online_ragged(Y, S, N, mz, mw, mode, vad0, ref, o, R0=None):
    """One utterance of a ragged array in float64, node by node with its own C_k: Y, S, N lists of K [C_k, F', T]
    complex128, mz, mw [K, F', T]; R0 a list of K (Rs0, Rn0) [F', C_k, C_k] or None.  The composition of
    oracle/online_split_np (the reference's spatial_correlation_matrix and intern_filter per frame / block) that
    test_gpu_online_eval.f64_online spells out for one C.  Returns {name: [K, F', T]}."""
    from oracle import solve_f64, tango_np
    from oracle.online_split_np import online_mwf_split
    K = len(Y)
    fn = (tango_np.spatial_correlation_matrix, lambda Rs, Rn, mu, ft, r: solve_f64.solve(Rs, Rn, mu, ft, r))
    kw = dict(lambda_cor=o["lam"], block=o["block"], lag=o["lag"], mu=o["mu"], filter_type=o["typ"], rank=o["rank"],
              ref=ref)
    blk = lambda W, X: _blocks(W, X, o["block"], o["lag"], ref)
    r0 = lambda k: None if R0 is None else R0[k]
    shape = (K,) + Y[0].shape[1:]
    out = {nm: np.empty(shape, np.complex128) for nm in ("yf", "z_y", "zn", "z_s", "z_n", "sf", "nf")}
    for k in range(K):
        if "use_oracle_" in mode:
            z, W, _, _ = online_mwf_split(Y[k], S[k], N[k], *fn, R0=r0(k), **kw)
        else:
            z, W, _, _ = online_mwf_split(Y[k], mz[k] * Y[k], (1 - mz[k]) * Y[k], *fn, R0=r0(k), **kw)
        out["z_y"][k], out["zn"][k] = z, Y[k][ref] - z
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
            rs, rn = np.stack([S[j][ref] for j in oth]), np.stack([N[j][ref] for j in oth])
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


def _r0(specs_full, chans):
    """Per node (Rs0, Rn0) [F, C_k, C_k] complex64 of the scale of the data: the plain SCMs of the first 20 frames of
    the clean spectra, exactly Hermitian with a real diagonal."""
    out = []
    for k, C in enumerate(chans):
        pair = []
        for X in specs_full:
            Xk = X[k][..., :20]
            R = (np.einsum("cft,dft->fcd", Xk, Xk.conj()) / 20).astype(np.complex64)
            R = 0.5 * (R + R.conj().swapaxes(-1, -2))
            R.imag[..., np.arange(C), np.arange(C)] = 0
            pair.append(np.ascontiguousarray(R))
        out.append(tuple(pair))
    return out


# (geometry, mode, (filter type, rank, mu), R0, n_fft, ref_mic)
ONLINE = [([2, 3, 2], "local", ("gevd", 1, 1.0), True, 256, 1),
          ([1, 4], "distant", ("mwf", 1, 1.0), False, 512, 0),
          ([4, 2, 2, 1], "compressed", ("gevd", 1, 1.0), False, 256, 0),
          ([2, 3, 2], "use_oracle_refs", ("gevd", 1, 1.0), True, 256, 0),
          ([2, 3, 2], "use_oracle_zs", ("gevd", 2, 2.5), False, 256, 1),
          ([4, 2, 2, 1], "previous", ("r1-mwf", 1, 2.5), False, 256, 0),
          ([2, 3, 2], "distant", ("gevd", 2, 1.0), False, 512, 0),
          ([1, 4], "local", ("r1-mwf", 1, 1.0), True, 512, 0)]


@pytest.mark.parametrize("chans,mode,setting,use_r0,n_fft,ref", ONLINE,
                         ids=["%s-%s-%s-r%d-mu%g%s-n%d" % ("".join(map(str, c[0])), c[1], *c[2], "-R0" if c[3] else "",
                                                            c[4]) for c in ONLINE])
def test_online_matches_the_float64_composition(dev, chans, mode, setting, use_r0, n_fft, ref):
    """online_tango_ragged, every node of every utterance against float64 with its own C_k and the z of the other
    nodes: from the block whose filter saw >= 4 D frames on (D = C_k in step 1, C_k + K - 1 in step 2), within 1e-5
    complex relative L2 on yf, z_y, zn, z_s, z_n, sf, nf."""
    from disco_b200.ragged import online_tango_ragged
    typ, rank, mu = setting
    B, L, K, block, lag, lam = 2, 24000, len(chans), 8, 1, 0.98
    F = n_fft // 2 + 1
    fsel = [0, 37, F // 2, F - 1]
    utts = [_utterance(700 + 11 * b + ONLINE.index((chans, mode, setting, use_r0, n_fft, ref)), chans, L)
            for b in range(B)]
    yd, sd, nd = _batch(dev, utts)
    R0 = R0d = None
    if use_r0:
        R0 = [_r0([[_spec64(u[i][k], n_fft, slice(None)) for k in range(K)] for i in (1, 2)], chans) for u in utts]
        R0d = [tuple(torch.from_numpy(np.stack([R0[b][k][i] for b in range(B)])).to(dev) for i in (0, 1))
               for k in range(K)]
    out = online_tango_ragged(yd, chans, lambda_cor=lam, block=block, lag=lag, mu=mu, rank=rank, ref_mic=ref,
                              n_fft=n_fft, R0=R0d, s=sd, n=nd, vads=("irm1", "irm2"), mask_for_z=mode,
                              filter_type=typ)
    groups = sorted(set(chans))
    assert sorted(out["W1"]) == groups and sorted(out["W2"]) == groups
    for C in groups:
        nodes = [k for k in range(K) if chans[k] == C]
        assert out["nodes"][C] == nodes
        assert out["W1"][C].shape[-1] == C and out["W2"][C].shape[-1] == C + K - 1
        assert out["W1"][C].shape[:2] == (B, len(nodes))
    o = dict(lam=lam, block=block, lag=lag, mu=mu, typ=typ, rank=rank)
    for b in range(B):
        specs = [[_spec64(utts[b][i][k], n_fft, fsel) for k in range(K)] for i in range(3)]
        mz = _np(out["masks_z"][b])[:, :, fsel].transpose(0, 2, 1)
        mw = _np(out["mask_w"][b])[:, :, fsel].transpose(0, 2, 1)
        r0 = None if R0 is None else [tuple(r[fsel] for r in R0[b][k]) for k in range(K)]
        truth = f64_online_ragged(*specs, mz, mw, mode, "irm1", ref, o, r0)
        for nm in ("yf", "z_y", "zn", "z_s", "z_n", "sf", "nf"):
            got = _np(out[nm][b])[:, :, fsel].transpose(0, 2, 1)
            for k in range(K):
                D = chans[k] if nm in ("z_y", "zn", "z_s", "z_n") else chans[k] + K - 1
                t0 = _start(D, block, lag)
                assert t0 < got.shape[-1] - block
                e = rel_l2(got[k][..., t0:], truth[nm][k][..., t0:])
                assert e <= TOL, (nm, b, k, t0, e)


BITEXACT = [([2, 4, 2], None), ([1, 4, 1], None), ([2, 4, 6, 4], None), ([2, 4, 2], "uneven"),
            ([1, 4, 1], "uneven")]


@pytest.mark.parametrize("chans,lens", BITEXACT, ids=["%s-%s" % ("".join(map(str, c)), l) for c, l in BITEXACT])
def test_online_batch_is_bit_exact_with_even_groups(dev, chans, lens):
    """Every count group holds an even number of signals (n_C * C), so each group's STFT pairs every utterance's
    signals among themselves as a lone run does: each utterance's online outputs, filters and masks equal its lone
    run (B = 1) with torch.equal.  With uneven lengths the lone run is on the trimmed signals, and NaN past each
    length reaches no output."""
    from disco_b200.ragged import online_tango_ragged
    assert all(chans.count(C) * C % 2 == 0 for C in set(chans))
    n_fft, block = 256, 8
    hop = n_fft // 2
    lengths = [12000, 9000 + 37, 12000 - 3 * hop] if lens else [12000] * 3
    L, B = max(lengths), len(lengths)
    clean = _batch(dev, [_utterance(1100 + b + sum(chans), chans, L, gate=2000) for b in range(B)])
    batch = clean
    if lens:
        batch = []
        for a in clean:
            a = a.clone()
            for b, Lb in enumerate(lengths):
                a[b, :, Lb:] = float("nan")
            batch.append(a)
    kw = dict(block=block, lag=1, n_fft=n_fft, vads=("ivad", "irm2"), mask_for_z="distant")
    got = online_tango_ragged(batch[0], chans, s=batch[1], n=batch[2], lengths=lengths if lens else None, **kw)
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        Jb = -(-Tb // block)
        alone = online_tango_ragged(clean[0][b:b + 1, :, :Lb].contiguous(), chans, s=clean[1][b:b + 1, :, :Lb].contiguous(),
                                    n=clean[2][b:b + 1, :, :Lb].contiguous(), **kw)
        for nm, v in got.items():
            if nm == "nodes":
                assert v == alone[nm]
                continue
            pairs = [(v[C], alone[nm][C]) for C in v] if isinstance(v, dict) else [(v, alone[nm])]
            cut = Jb if nm in ("W1", "W2") else Tb
            for g, w in pairs:
                assert torch.equal(g[b, :, :cut], w[0]), (nm, b)
                assert not bool(g[b, :, cut:].any()), (nm, b, "not 0 past the end")
                assert bool(torch.isfinite(torch.view_as_real(g) if g.is_complex() else g).all()), nm


# ---- 5. scoring -----------------------------------------------------------------------------------------------------
def test_scores_match_the_adapter(dev):
    """post.to_time + post.tango_scores(..., stoi=True, lengths=) run unchanged on tango_ragged's outputs of an uneven
    batch: every score is finite and [B, K], and the spectra scored are the adapter's for each trimmed utterance within
    the parity rule."""
    from disco_b200 import post
    from disco_b200.ragged import tango_ragged
    from disco_b200.tango import offline_tango
    from test_gpu_stoi import speechlike
    fs, L, n_fft = 16000, 3 * 16000, 512
    chans = [2, 3, 1]
    K, B = len(chans), 3
    rows0 = [0, 2, 5]                                            # microphone 0 of each node
    lengths = [L, 40000, 33001]
    utts = [_utterance(1300 + b, chans, L, gate=6000) for b in range(B)]
    yd, sd, nd = (a.clone() for a in _batch(dev, utts))
    for b, Lb in enumerate(lengths):
        for a in (yd, sd, nd):
            a[b, :, Lb:] = 0
    s_dry = torch.from_numpy(np.stack([speechlike(60 + b, L + 100, period=6000, gain=0.05) for b in range(B)])).to(dev)
    n_dry = torch.from_numpy((0.02 * np.random.default_rng(5).standard_normal((B, L + 100))).astype(np.float32)).to(dev)
    out = tango_ragged(yd, chans, sd, nd, n_fft=n_fft, lengths=lengths)
    score = lambda o, sl, lens: post.tango_scores(
        yd[sl][:, rows0], sd[sl][:, rows0], nd[sl][:, rows0], s_dry[sl], n_dry[sl],
        post.to_time(o, L, n_fft=n_fft, lengths=lens), fs, stoi=True, lengths=lens)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        got = score(out, slice(None), lengths)
        for r in got:
            for key, v in r.items():
                assert v.shape[:2] == (B, K) and bool(torch.isfinite(v).all()), key
        for b, Lb in enumerate(lengths):
            trimmed = tuple([[ch[:Lb] for ch in node] for node in part] for part in utts[b])
            ad = dict(zip(NAMES, offline_tango(*trimmed, ["irm1", "irm1"], None, "local", n_fft=n_fft)))
            Tb = ad["yf"][0].shape[1]
            assert not bool(out["yf"][b, :, :, Tb:].any())
            for nm in ("yf", "sf", "nf", "z_y", "z_s", "z_n"):
                for k in range(K):
                    e = rel_l2_mag(_np(out[nm][b, k, :, :Tb]), ad[nm][k])
                    assert record_parity("ragged_scores_b%d" % b, nm, k, err_ref=e,
                                         note="reference = tango.offline_tango on the trimmed utterance"), (nm, b, k, e)
