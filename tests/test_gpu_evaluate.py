"""The evaluation driver (disco_b200/evaluate.py) on the device: files and scores against the reference's tango.main
(tests/golden/tango_main_kat.npz, oracle/make_tango_main.py), batched against alone, network masks
against the offline_tango adapter, online mode against online_tango run per RIR, and resuming."""
import os
import pickle
import shutil

import numpy as np
import pytest
import torch

from conftest import GOLDEN, record_parity, rel_l2_mag
from disco_b200 import evaluate as ev
from disco_b200 import post, wav_io
from oracle.make_tango_main import (FRAME_STEP, SAMPLE_STEP, TANGO_MAIN_NODES, TANGO_MAIN_RIRS, WAV_NAMES,
                                    make_tango_dataset, pcm_sha256, tree_digest)

pytestmark = pytest.mark.gpu

# scores that depend on the inputs alone, and the rest (of the beamformed outputs)
INPUT_SCORES = ("snr_in_cnv", "snr_in_dry", "sdr_in_cnv", "sir_in_cnv", "sdr_in_dry", "sir_in_dry", "sar_in_dry")
PCM = 1.0 / 32768


def _run(dataset, results, **kw):
    ev.main(kw.pop("vads", ["irm1", "irm1"]), "out", TANGO_MAIN_RIRS[0], "ssn", nb_rir=len(TANGO_MAIN_RIRS),
            path_to_dataset=dataset, results_root=results, **kw)
    return os.path.join(results, "living", "test", "out")


def _tree(out):
    return sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)


def _pickles(out, rir):
    res = {}
    for kind in ("tango", "mwf"):
        with open(os.path.join(out, "OIM", "results_%s_%d_ssn.p" % (kind, rir)), "rb") as fh:
            res[kind] = pickle.load(fh)
    return res


def _wav(out, rir, name, node):
    return wav_io.read(os.path.join(out, "WAV", str(rir), "%s-ssn_Node-%d.wav" % (name, node)))[0]


def _mask(out, rir, step, node):
    return np.load(os.path.join(out, "MASK", str(rir), "step%d_ssn_Node-%d.npy" % (step, node)))


def _z(out, rir, node):
    return np.load(os.path.join(out, "STFT", "z", "raw", "0-6", "%d_ssn_Node-%d.npy" % (rir, node)))


def _assert_scores(got, want, input_rtol=None, f64=None, ref=None):
    """Input-only scores within 1e-6 dB (or input_rtol relative), beamformed ones within 0.01 dB, delta STOI 1e-4.
    The beamformed outputs of step 2 are ill-conditioned here: the reference's own float32 rounding moves their
    scores by up to ~0.005 dB from the float64 oracle's.  So, as record_parity does for spectra, a beamformed score
    outside its bar passes when it is as close to the float64 scores f64 as the reference's scores ref are (25 % on
    top, plus a tenth of the bar)."""
    for kind in ("tango", "mwf"):
        for k, w in want[kind].items():
            g = got[kind][k]
            if k == "snr_in_raw":
                assert type(g) is type(w) and g == w
            elif k in INPUT_SCORES:
                if input_rtol is None:
                    # the golden's n_dry gain was applied in float64 (NumPy 2 casting), the driver's in float32 as the
                    # reference's pinned NumPy does: one-ulp differences in many samples of n_dry, which move the
                    # fw_snr of the dry pair by ~1.1e-5 dB at the fixture's ~0.01 dB
                    bar = 3e-5 if k == "snr_in_dry" else 1e-6
                    assert np.max(np.abs(g - w)) < bar, (kind, k, g, w)
                else:
                    assert np.allclose(g, w, rtol=input_rtol, atol=0), (kind, k, g, w)
            else:
                bar = 1e-4 if k.startswith("delta_stoi") else 0.01
                near = np.abs(g - w) < bar
                if f64 is not None:
                    x = f64[kind][k]
                    near |= np.abs(g - x) <= 1.25 * np.abs(ref[kind][k] - x) + bar / 10
                assert near.all(), (kind, k, g, w)


def _f64_scores(root, rir):
    """The scores of the float64 oracle's outputs (oracle/tango_f64.py, librosa's iSTFT in float64) for one RIR."""
    from oracle import librosa_np, tango_f64
    y, s, n, s_dry, n_dry, fs = _lone(root, rir)
    cpu = lambda x: x[0].cpu().numpy()
    f = tango_f64.offline_tango(cpu(y), cpu(s), cpu(n))
    L = y.shape[-1]
    times = {nm: torch.from_numpy(np.array([[librosa_np.istft(f[nm][k], hop_length=256, win_length=512, length=L,
                                                               dtype=np.float64) for k in range(4)]],
                                            dtype=np.float32)).cuda()
             for nm in ("yf", "z_y", "sf", "nf", "z_s", "z_n")}
    return _lone_scores(y, s, n, s_dry, n_dry, fs, times)


def _golden_scores(g, rir):
    return {kind: {k: g["p_%d_%s_%s" % (rir, kind, k)][()] for k in g["keys_%d_%s" % (rir, kind)]}
            for kind in ("tango", "mwf")}


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """The data set and the driver's outputs at batch 1 and 3 (irm1 / irm1, mask_z 'local')."""
    root = str(tmp_path_factory.mktemp("evaluate"))
    make_tango_dataset(root)
    g = np.load(os.path.join(GOLDEN, "tango_main_kat.npz"))
    assert tree_digest(os.path.join(root, "disco")) == str(g["dataset_sha256"])       # the generator is unchanged
    out = {b: _run(root, os.path.join(root, "res%d" % b), batch=b) for b in (1, 3)}
    f64 = {rir: _f64_scores(root, rir) for rir in TANGO_MAIN_RIRS}
    return root, out, g, f64


@pytest.mark.parametrize("batch", [1, 3])
def test_files_and_scores_match_the_reference(runs, batch):
    from oracle import tango_f64
    root, outs, g, f64 = runs
    out = outs[batch]
    assert _tree(out) == list(g["tree"])
    assert os.path.isdir(os.path.join(out, "FIG"))
    for i, rir in enumerate(TANGO_MAIN_RIRS):
        res = _pickles(out, rir)
        want = _golden_scores(g, rir)
        for kind in ("tango", "mwf"):
            assert list(res[kind]) == list(want[kind])
            for k, v in res[kind].items():
                assert np.asarray(v).dtype == want[kind][k].dtype and np.shape(v) == np.shape(want[kind][k]), k
        _assert_scores(res, want, f64=f64[rir], ref=want)
        node = int(g["wav_node_%d" % rir])
        for name in WAV_NAMES:
            x = _wav(out, rir, name, node)
            assert len(x) == int(g["wavlen_%d_%s" % (rir, name)]), name
            if name.startswith("in_"):
                assert pcm_sha256(x) == str(g["wavsha_%d_%s" % (rir, name)]), name          # byte-identical samples
            else:
                pcm = np.round(x[::SAMPLE_STEP].astype(np.float64) * 32768).astype(np.int32)
                assert np.max(np.abs(pcm - g["wav_%d_%s" % (rir, name)])) <= 1, name
        y, s, n, *_ = ev.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        o64 = tango_f64.offline_tango(np.array(y), np.array(s), np.array(n))
        for k in TANGO_MAIN_NODES:
            tag = "%d_%d" % (rir, k)
            for step in (1, 2):
                m = _mask(out, rir, step, k)
                assert str(m.dtype) == str(g["mask_meta_" + tag][step - 1])
                assert m.shape == tuple(g["mask_shape_" + tag])
                # the golden keeps step 2 only where it differs from step 1
                ref = g["mask_%d_%s" % (step, tag)] if "mask_%d_%s" % (step, tag) in g else g["mask_1_" + tag]
                # 1e-5, not test_gpu_dataset_post's 5e-6: the float32 STFT kernel's absolute error moves the mask of
                # near-silent bins of the gated target by up to 6.4e-6 from float64 here (the reference's, 1e-7)
                assert np.max(np.abs(m[:, ::FRAME_STEP] - ref)) < 1e-5, (rir, step, k)
            z = _z(out, rir, k)
            meta = g["z_meta_" + tag]
            assert str(z.dtype) == str(meta[0]) == "complex64" and z.shape == tuple(int(v) for v in meta[1:])
            z, ref, z64 = z[:, ::FRAME_STEP], g["zabs_" + tag], o64["z_y"][k - 1][:, ::FRAME_STEP]
            e_ref, e_f64, ref_f64 = rel_l2_mag(z, ref), rel_l2_mag(z, z64), rel_l2_mag(ref, z64)
            # where the reference itself is nearly 1e-5 from float64 (just under record_parity's fallback), the direct
            # distance is the sum of two such errors; it passes when ours is as close to float64 as the reference
            # (the and-rule's second clause) and the direct distance is what the two explain
            assert (record_parity("evaluate_b%d_%d" % (batch, rir), "z_y", k - 1, e_ref, e_f64, ref_f64)
                    or (e_f64 <= ref_f64 + 1e-6 and e_ref <= 1.25 * (e_f64 + ref_f64))), (rir, k, e_ref, e_f64, ref_f64)


def test_batched_equals_alone(runs):
    _, outs, g, f64 = runs
    a, b = outs[3], outs[1]
    assert _tree(a) == _tree(b)
    for rir in TANGO_MAIN_RIRS:
        # the inputs are the same samples; only the trailing zeros of the padded batch differ
        _assert_scores(_pickles(a, rir), _pickles(b, rir), input_rtol=1e-9, f64=f64[rir], ref=_golden_scores(g, rir))
        for k in range(1, 5):
            for name in WAV_NAMES:
                x, w = _wav(a, rir, name, k), _wav(b, rir, name, k)
                assert x.shape == w.shape and np.max(np.abs(x - w)) <= PCM + 1e-9, (rir, name, k)
            for step in (1, 2):
                assert np.max(np.abs(_mask(a, rir, step, k) - _mask(b, rir, step, k))) < 5e-6
            assert rel_l2_mag(_z(a, rir, k), _z(b, rir, k)) < 1e-5


def _lone(root, rir):
    """One RIR's inputs on the device: y, s, n [1, K, C, L], s_dry, n_dry [1, L_dry], fs."""
    y, s, n, s_dry, n_dry, fs, _ = ev.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
    t = lambda a: torch.from_numpy(np.array(a, dtype=np.float32)).cuda()[None]
    return t(y), t(s), t(n), t(s_dry), t(n_dry), fs


def _lone_scores(y, s, n, s_dry, n_dry, fs, times):
    """tango_scores of one RIR as the driver scores it: over [fs, min(L, L_s_dry, L_n_dry))."""
    score_len = np.array([min(y.shape[-1], s_dry.shape[-1], n_dry.shape[-1])])
    r, rz = post.tango_scores(y[:, :, 0], s[:, :, 0], n[:, :, 0], s_dry, n_dry, times, fs, stoi=True,
                              lengths=score_len)
    return {kind: {k: v[0].cpu().numpy() for k, v in d.items()} for kind, d in (("tango", r), ("mwf", rz))}


def _checkpoint(path, n_ch, seed):
    from disco_b200 import dnn_mask
    torch.manual_seed(seed)
    model = dnn_mask.build_crnn(n_ch)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    torch.save({"model_state_dict": model.state_dict()}, path)
    return path


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("z_sigs", ["zs_hat", ["zs_hat", "zn_hat"]])
def test_network_masks_match_offline_tango(runs, tmp_path, z_sigs, batch):
    """batch=1 runs the adapter's routes: masks within 5e-6 and scores as against the reference.  batch=3 pads RIRs
    11001 and 11002: their step-1 masks must still be the lone RIR's within 5e-6 (a network that saw the clamped
    padding would differ in the last 10 frames).  Its step-2 networks hear z, which the padded batch's stored-spectra
    route rounds differently from the lone fused route (~1e-6 relative); the random-weight network amplifies that,
    so those masks get 2e-3."""
    from disco_b200.tango import offline_tango
    root = runs[0]
    n2 = 4 if isinstance(z_sigs, str) else 7
    paths = [_checkpoint(str(tmp_path / "step1.pt"), 1, 1), _checkpoint(str(tmp_path / "step2.pt"), n2, 2)]
    out = _run(root, str(tmp_path / "res"), vads=["crnn", "crnn"], models=paths, z_sigs=z_sigs, batch=batch)
    mods = ev.load_models(["crnn", "crnn"], paths, [1, n2])
    for rir in TANGO_MAIN_RIRS:
        y, s, n, s_dry, n_dry, fs = _lone(root, rir)
        lists = lambda x: [[x[0, k, c].cpu().numpy() for c in range(x.shape[2])] for k in range(x.shape[1])]
        res = offline_tango(lists(y), lists(s), lists(n), ["crnn", "crnn"], mods=mods, mask_for_z="local",
                            z_sigs=z_sigs)
        outs = dict(zip(("yf", "sf", "nf", "z_y", "z_s", "z_n", "zn", "masks_z", "mask_w"), res))
        for k in range(4):
            for step, nm in ((1, "masks_z"), (2, "mask_w")):
                m = _mask(out, rir, step, k + 1)
                bar = 2e-3 if batch > 1 and step == 2 else 5e-6
                assert m.dtype == np.float32 and np.max(np.abs(m - outs[nm][k])) < bar, (rir, step, k)
        if batch > 1:
            continue
        spec = {nm: torch.from_numpy(np.array(outs[nm])).cuda()[None] for nm in ("yf", "sf", "nf", "z_y", "z_s", "z_n")}
        times = post.to_time(spec, y.shape[-1], layout="FT")
        got, want = _pickles(out, rir), _lone_scores(y, s, n, s_dry, n_dry, fs, times)
        for kind in want:
            want[kind]["snr_in_raw"] = got[kind]["snr_in_raw"]
        _assert_scores(got, want)


def test_online_matches_online_tango_per_rir(runs, tmp_path):
    from disco_b200.online import online_tango
    root = runs[0]
    out = _run(root, str(tmp_path / "res"), online=True, batch=3)
    for rir in TANGO_MAIN_RIRS:
        y, s, n, s_dry, n_dry, fs = _lone(root, rir)
        L = y.shape[-1]
        o = online_tango(y, s=s, n=n, vads=("irm1", "irm1"), mask_for_z="local", block=8, lag=1, lambda_cor=0.95)
        times = post.to_time(o, L, layout="TF")
        sig = {"yf": times["yf"], "z_y": times["z_y"], "nf": times["nf"], "sf": times["sf"]}
        for k in range(4):
            for name, t in (("out_mix", "yf"), ("mid_z", "z_y"), ("out_noi", "nf"), ("out_tar", "sf")):
                ref_path = str(tmp_path / "ref.wav")
                wav_io.write(ref_path, sig[t][0, k].cpu().numpy(), fs)
                assert np.array_equal(_wav(out, rir, name, k + 1), wav_io.read(ref_path)[0]), (rir, name, k)
            for step, nm in ((1, "masks_z"), (2, "mask_w")):
                assert np.array_equal(_mask(out, rir, step, k + 1), o[nm][0, k].T.cpu().numpy())
            assert np.array_equal(_z(out, rir, k + 1), o["z_y"][0, k].T.cpu().numpy())
        got, want = _pickles(out, rir), _lone_scores(y, s, n, s_dry, n_dry, fs, times)
        for kind in want:
            for key, w in want[kind].items():
                assert np.allclose(got[kind][key], w, rtol=1e-9, atol=0), (rir, kind, key)


def test_resume_skips_finished_rirs(runs, tmp_path, monkeypatch, capsys):
    root, outs = runs[:2]
    res = str(tmp_path / "res")
    shutil.copytree(os.path.dirname(os.path.dirname(os.path.dirname(outs[3]))), res)
    out = os.path.join(res, "living", "test", "out")
    calls = []
    real = ev.tango_batched

    def spy(y, *a, **k):
        calls.append(y.shape[0])
        return real(y, *a, **k)
    monkeypatch.setattr(ev, "tango_batched", spy)
    stamp = lambda: {p: os.stat(os.path.join(out, p)).st_mtime_ns for p in _tree(out)}
    before = stamp()
    _run(root, res, batch=3)
    assert calls == [] and stamp() == before
    assert capsys.readouterr().out.count("already processed") == 3
    redo = TANGO_MAIN_RIRS[1]
    os.remove(os.path.join(out, "OIM", "results_mwf_%d_ssn.p" % redo))
    _run(root, res, batch=3)
    assert calls == [1]
    after = stamp()
    assert set(after) == set(before)
    changed = {p for p in after if after[p] != before[p]}
    assert changed and all(str(redo) in p for p in changed)
    assert len([p for p in changed if p.startswith("WAV")]) == 28
