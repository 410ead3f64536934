"""The z-signal driver (disco_b200/get_z.py) on the device: files against the reference's get_z_signals.main
(tests/golden/get_z_kat.npz, oracle/make_get_z.py; zs_hat against tango_main_kat.npz), batched against alone, every
mask route against the per-RIR adapter compat.get_z_signals.offline_tango + save_z_signals, the command line,
resuming and a failing writer."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, record_parity, rel_l2, rel_l2_mag
from disco_b200 import get_z as gz
from disco_b200.dataset_post import save_z_signals
from oracle.make_get_z import FRAME_STEP, GET_Z_NODES, file_name, raw_name
from oracle.make_tango_main import FRAME_STEP as TANGO_FRAME_STEP
from oracle.make_tango_main import TANGO_MAIN_NODES, TANGO_MAIN_RIRS, make_tango_dataset, tree_digest

pytestmark = pytest.mark.gpu


def _out(root, save_dir):
    return os.path.join(root, "disco", "living", "test", "stft_z", save_dir)


def _run(root, save_dir, vad="irm1", **kw):
    gz.main(vad, save_dir, TANGO_MAIN_RIRS[0], "ssn", nb_rir=len(TANGO_MAIN_RIRS), path_to_dataset=root, **kw)
    return _out(root, save_dir)


def _tree(out):
    return sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)


def _load(out, sub, kind, rir, node):
    return np.load(os.path.join(out, file_name(sub, kind, rir, node)))


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    """The data set and the driver's outputs at batch 1 and 3 (irm1, mask_z 'local')."""
    root = str(tmp_path_factory.mktemp("get_z"))
    make_tango_dataset(root)
    g = np.load(os.path.join(GOLDEN, "get_z_kat.npz"))
    assert tree_digest(os.path.join(root, "disco")) == str(g["dataset_sha256"])       # the generator is unchanged
    out = {b: _run(root, "b%d" % b, batch=b) for b in (1, 3)}
    return root, out, g


def _parity(case, output, node, z, ref, z64):
    """test_gpu_evaluate's rule for z: record_parity, or, where the reference itself is nearly 1e-5 from float64,
    as close to float64 as the reference and a direct distance the two explain."""
    e_ref, e_f64, ref_f64 = rel_l2_mag(z, ref), rel_l2_mag(z, z64), rel_l2_mag(ref, z64)
    assert (record_parity(case, output, node, e_ref, e_f64, ref_f64)
            or (e_f64 <= ref_f64 + 1e-6 and e_ref <= 1.25 * (e_f64 + ref_f64))), (case, output, node, e_ref, e_f64,
                                                                                   ref_f64)


@pytest.mark.parametrize("batch", [1, 3])
def test_files_match_the_reference(runs, batch):
    from oracle import tango_f64
    root, outs, g = runs
    out = outs[batch]
    tree = _tree(out)
    assert tree == list(g["tree"])
    for rel, dtype, shape in zip(tree, g["dtype"], g["shape"]):
        a = np.load(os.path.join(out, rel))
        assert str(a.dtype) == str(dtype) and a.shape == tuple(shape), rel
    # the reference saves np.abs of the array it saved raw; so does the driver, bit for bit
    assert list(g["abs_files"]) == [rel for rel in tree if rel.startswith("normed")] and not g["abs_dev"].any()
    for rel in g["abs_files"]:
        a, raw = np.load(os.path.join(out, rel)), np.load(os.path.join(out, raw_name(rel)))
        assert np.array_equal(a, np.abs(raw)), rel
    kat = np.load(os.path.join(GOLDEN, "tango_main_kat.npz"))
    for rir in TANGO_MAIN_RIRS:
        y, s, n = gz.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        o64 = tango_f64.offline_tango(np.array(y), np.array(s), np.array(n))
        # zs_hat is tango's step-1 z_y, pinned by tango_main_kat.npz (oracle/make_get_z.py checks it is the same)
        for k in TANGO_MAIN_NODES:
            z = _load(out, "raw", "zs_hat", rir, k)[:, ::TANGO_FRAME_STEP]
            _parity("get_z_b%d_%d" % (batch, rir), "zs_hat", k - 1, z, kat["zabs_%d_%d" % (rir, k)],
                    o64["z_y"][k - 1][:, ::TANGO_FRAME_STEP])
        for k in GET_Z_NODES:
            z = _load(out, "raw", "zn_hat", rir, k)[:, ::FRAME_STEP]
            _parity("get_z_b%d_%d" % (batch, rir), "zn_hat", k - 1, z, g["znabs_%d_%d" % (rir, k)],
                    o64["zn"][k - 1][:, ::FRAME_STEP])


def test_batched_equals_alone(runs):
    """batch=3 pads RIRs 11001 and 11002 and passes their lengths: test_gpu_evaluate's bar for z."""
    _, outs, _ = runs
    a, b = outs[3], outs[1]
    assert _tree(a) == _tree(b)
    for rir in TANGO_MAIN_RIRS:
        for k in range(1, 5):
            for kind in ("zs_hat", "zn_hat"):
                x, w = _load(a, "raw", kind, rir, k), _load(b, "raw", kind, rir, k)
                assert x.shape == w.shape and rel_l2_mag(x, w) < 1e-5, (rir, k, kind)


def _checkpoint(path, seed):
    from disco_b200 import dnn_mask
    torch.manual_seed(seed)
    model = dnn_mask.build_crnn(1)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.normal_(0, 0.1)
            m.running_var.uniform_(0.5, 1.5)
    torch.save({"model_state_dict": model.state_dict()}, path)
    return path


@pytest.mark.parametrize("vad, mask_z", [("irm1", "local"), ("ibm1", "local"), ("ivad", "local"),
                                         ("irm1", "use_oracle_refs"), ("crnn", "local")])
def test_matches_the_per_rir_adapter(runs, tmp_path, monkeypatch, vad, mask_z):
    """Each RIR of a padded batch of 3 against compat.get_z_signals.offline_tango on that RIR alone, saved by
    save_z_signals: the same files; the step-1 masks of the batch's one tango_step1 call are the lone RIR's over its
    frames and 0 after them, so a network never saw the clamped padding.  The oracle masks come from spectra of other
    STFT groupings (the driver transforms the reference microphones alone, padded; the adapter every microphone of the
    lone RIR), so they get 2e-5: the float32 STFT moves near-silent bins of the gated target's mask by up to 6.4e-6 from
    float64 (test_gpu_evaluate), and two groupings measured 1.1e-5 apart here.  The 0/1 masks may differ in at most
    1e-4 of the bins, where those spectra tip a threshold.  z within 2e-5 relative as complex spectra: the padded
    batch's stored-spectra route and the lone fused route each sit up to ~1.3e-5 from float64 here, as the reference
    does.  Where the two are further apart, the conditioning of the masks' statistics has amplified that rounding (the
    random-weight network's masks took them 2.4e-3 apart), and ours must be as close to the float64 step 1 with the
    adapter's masks as the adapter's is."""
    from disco_b200.compat.get_z_signals import offline_tango
    from oracle import tango_f64
    root = runs[0]
    weights = _checkpoint(str(tmp_path / "sc.pt"), 3) if vad == "crnn" else None
    masks, real = [], gz.tango_step1

    def spy(y, mask, *a, **k):
        masks.append(mask.transpose(-1, -2).cpu().numpy())          # [B, K, F, T]
        return real(y, mask, *a, **k)
    monkeypatch.setattr(gz, "tango_step1", spy)
    out = _run(root, "%s_%s" % (vad, mask_z), vad, mask_z=mask_z, weights_sc=weights, batch=3)
    assert len(masks) == 1 and masks[0].shape[0] == 3
    mods = gz.load_models([weights])
    ref = str(tmp_path / "adapter")
    for b, rir in enumerate(TANGO_MAIN_RIRS):
        y, s, n = gz.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        z_y, _, _, zn, mz = offline_tango(y, s, n, vad, mods=mods, mask_for_z=mask_z)
        save_z_signals(z_y, zn, ref, "0-6", rir, "ssn")
        T = z_y[0].shape[1]
        got = masks[0][b]
        assert not got[..., T:].any(), rir
        for k in range(4):
            if vad in ("ibm1", "ivad"):
                assert np.mean(got[k, :, :T] != mz[k]) <= 1e-4, (rir, k)
            else:
                assert np.max(np.abs(got[k, :, :T] - mz[k])) < 2e-5, (rir, k)
        f64 = None
        for k in range(1, 5):
            for kind, lst in (("zs_hat", z_y), ("zn_hat", zn)):
                x, w = _load(out, "raw", kind, rir, k), lst[k - 1]
                if rel_l2(x, w) < 2e-5:
                    continue
                assert mask_z == "local", (rir, k, kind, rel_l2(x, w))
                if f64 is None:
                    m = np.array(mz, np.float64)
                    f64 = tango_f64.offline_tango(np.array(y), masks=(m, m))
                z64 = f64["z_y" if kind == "zs_hat" else "zn"][k - 1]
                assert rel_l2(x, z64) <= 1.25 * rel_l2(w, z64) + 1e-6, (rir, k, kind, rel_l2(x, w), rel_l2(x, z64),
                                                                        rel_l2(w, z64))
    assert _tree(out) == _tree(ref)
    for rel in _tree(ref):
        x, w = np.load(os.path.join(out, rel)), np.load(os.path.join(ref, rel))
        assert x.dtype == w.dtype and x.shape == w.shape, rel


def test_command_line_writes_the_reference_tree(runs, tmp_path):
    """python -m disco_b200.get_z with the reference's defaults (-vt irm1, --noise fs, -mz local, -msc './') on a
    make_tango_dataset tree of 'fs' noise: the golden tree under the other noise name; a second call skips all three
    RIRs and writes nothing."""
    g = runs[2]
    root = str(tmp_path)
    make_tango_dataset(root, noise="fs")
    cmd = [sys.executable, "-m", "disco_b200.get_z", "-vt", "irm1", "-sd", "out", "--rir", "11001", "--nb_rir", "3",
           "--dataset", root]
    first = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert first.returncode == 0, first.stderr
    out = _out(root, "out")
    assert _tree(out) == [rel.replace("_ssn_", "_fs_") for rel in g["tree"]]
    stamp = {p: os.stat(os.path.join(out, p)).st_mtime_ns for p in _tree(out)}
    second = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True)
    assert second.returncode == 0, second.stderr
    assert second.stdout.splitlines() == ["Conf %d with fs noise already processed" % r for r in TANGO_MAIN_RIRS]
    assert {p: os.stat(os.path.join(out, p)).st_mtime_ns for p in _tree(out)} == stamp


def test_resume_redoes_only_unfinished_rirs(runs, monkeypatch, capsys):
    root, outs, _ = runs
    out = _out(root, "resume")
    shutil.copytree(outs[1], out)           # computed one RIR per call, as a redone RIR alone is
    calls = []
    real = gz.tango_step1

    def spy(y, *a, **k):
        calls.append(y.shape[0])
        return real(y, *a, **k)
    monkeypatch.setattr(gz, "tango_step1", spy)
    stamp = lambda: {p: os.stat(os.path.join(out, p)).st_mtime_ns for p in _tree(out)}
    before = stamp()
    content = {p: open(os.path.join(out, p), "rb").read() for p in before}
    capsys.readouterr()
    _run(root, "resume", batch=3)
    assert calls == [] and stamp() == before
    assert capsys.readouterr().out.count("already processed") == 3
    redo = TANGO_MAIN_RIRS[1]
    os.remove(os.path.join(out, file_name("normed", "zn_hat", redo, 4)))
    _run(root, "resume", batch=3)
    assert calls == [1]
    after = stamp()
    assert set(after) == set(before)
    changed = {p for p in after if after[p] != before[p]}
    assert changed == {p for p in after if "%d_ssn" % redo in p} and len(changed) == 16
    for p in after:
        with open(os.path.join(out, p), "rb") as fh:
            assert fh.read() == content[p], p


def test_writer_failure_raises_from_main(runs):
    """A file where the stft_z/<save_dir> directory should be: the writer thread's error is raised by main."""
    root = runs[0]
    with open(_out(root, "blocked"), "w") as fh:
        fh.write("not a directory")
    with pytest.raises((FileExistsError, NotADirectoryError)):
        _run(root, "blocked", batch=2)
