"""The z-signal driver (disco_b200/get_z.py) without a GPU: signatures, command line, data-set paths, the resume plan,
input reading and the errors raised before any device work."""
import importlib
import inspect
import json
import os

import numpy as np
import pytest
import torch

from disco_b200 import get_z as gz
from disco_b200 import wav_io

REF = "disco_theque/speech_enhancement/get_z_signals.py:"
NAMES = ("main", "get_input_signals", "load_models", "get_dset", "get_directory_name")


def test_signatures_match_the_reference(golden_dir):
    """Same rule as test_compat_cpu.test_adapter_signatures_match_the_reference, over
    tests/golden/reference_signatures_get_z.json; compat.get_z_signals re-exports the same functions."""
    ref = json.load(open(os.path.join(golden_dir, "reference_signatures_get_z.json")))
    assert set(ref) == {REF + k for k in NAMES}
    compat = importlib.import_module("disco_b200.compat.get_z_signals")
    for name in NAMES:
        fn = getattr(gz, name)
        assert getattr(compat, name) is fn
        ours = list(inspect.signature(fn).parameters.values())
        want_all = ref[REF + name]["params"]
        for i, want in enumerate(want_all):
            got = ours[i]
            assert got.name == want["name"], (name, i, got.name)
            assert got.kind in (got.POSITIONAL_OR_KEYWORD, got.POSITIONAL_ONLY), (name, got.name)
            if want["has_default"]:
                assert got.default is not inspect.Parameter.empty and got.default == want["default"], (name, got.name)
            else:
                assert got.default is inspect.Parameter.empty, (name, got.name)
        for extra in ours[len(want_all):]:
            assert extra.kind == extra.KEYWORD_ONLY, (name, extra.name)
    assert callable(compat.offline_tango)


def test_cli_parses_the_reference_flags():
    args, kw = gz.parse_args(["-sd", "out", "--rir", "11001"])
    assert args == ("irm1", "out", 11001, "fs")           # -vt defaults to 'irm1', --noise to 'fs' (:366-383)
    assert kw == dict(scenario="living", mask_z="local", weights_sc="./", nb_rir=1, batch=8,
                      path_to_dataset=gz.PATH_TO_DATASET)
    args, kw = gz.parse_args(["--vad_type", "crnn", "--sav_dir", "x", "--rir", "3", "--scenario", "meeting",
                              "--noise", "ssn", "--mask_z", "use_oracle_refs", "--mod_sc", "sc.pt", "--nb_rir", "20",
                              "--batch", "4", "--dataset", "/d"])
    assert args == ("crnn", "x", 3, "ssn")
    assert kw == dict(scenario="meeting", mask_z="use_oracle_refs", weights_sc="sc.pt", nb_rir=20, batch=4,
                      path_to_dataset="/d")
    _, kw = gz.parse_args(["-vt", "ivad", "-scene", "random", "-mz", "None", "-msc", "None"])
    assert kw["mask_z"] is None and kw["weights_sc"] is None and kw["scenario"] == "random"
    for mz in ("local", "distant", "compressed", "use_oracle_refs", "use_oracle_zs"):
        assert gz.parse_args(["-mz", mz])[1]["mask_z"] == mz
    for bad in (["--noise", "wind"], ["-scene", "office"], ["-mz", "global"], ["-vt", "irm1", "irm1"]):
        with pytest.raises(SystemExit):
            gz.parse_args(bad)


def test_dset_and_directory_names():
    assert [gz.get_dset(r) for r in (1, 11000, 11001, 12000)] == ["train", "train", "test", "test"]
    for r in (0, 12001):
        with pytest.raises(AssertionError, match="between 1 and 12000"):
            gz.get_dset(r)
    assert gz.get_directory_name([[0, 6]]) == "0-6"
    assert gz.get_directory_name([[3, 6], [5, 15]]) == "3-6_5-15"
    assert gz._save_root("/d", "living", 11000, "out") == os.path.join("/d", "disco", "living", "train", "stft_z",
                                                                        "out", "")
    assert gz._save_root("/d", "meeting", 11001, "o") == os.path.join("/d", "disco", "meeting", "test", "stft_z", "o",
                                                                       "")


def _files(root, rir, nodes, noise="ssn", save_dir="out"):
    """Writes the z files of nodes `nodes` of one RIR in the order save_z_signals writes them."""
    base = gz._save_root(root, "living", rir, save_dir)
    for k in nodes:
        for sub in (("raw",), ("normed", "abs")):
            for kind in ("zs_hat", "zn_hat"):
                d = os.path.join(base, *sub, "0-6", kind)
                os.makedirs(d, exist_ok=True)
                np.save(os.path.join(d, "%d_%s_Node-%d.npy" % (rir, noise, k)), np.zeros((2, 2), np.float32))


def test_batch_plan_skips_finished_rirs(tmp_path, capsys):
    root = str(tmp_path)
    _files(root, 10999, range(1, 5))        # finished
    _files(root, 11001, range(1, 4))        # interrupted before node 4: redone
    _files(root, 11003, range(1, 5))
    plan = gz._batch_plan(10998, 8, 3, "ssn", "living", "out", root, 4)
    assert plan == [[10998, 11000, 11001], [11002, 11004, 11005]]
    out = capsys.readouterr().out
    assert "Conf 10999 with ssn noise already processed" in out and "Conf 11003 with ssn noise already processed" in out
    assert "11001" not in out
    # the last file alone decides, as the reference's check would if it had the '.npy'
    os.remove(os.path.join(gz._save_root(root, "living", 11003, "out"), "raw", "0-6", "zs_hat", "11003_ssn_Node-1.npy"))
    assert gz._batch_plan(11003, 1, 8, "ssn", "living", "out", root, 4) == []
    os.remove(os.path.join(gz._save_root(root, "living", 11003, "out"), "normed", "abs", "0-6", "zn_hat",
                           "11003_ssn_Node-4.npy"))
    assert gz._batch_plan(11003, 1, 8, "ssn", "living", "out", root, 4) == [[11003]]
    assert gz._batch_plan(10999, 1, 8, "fs", "living", "out", root, 4) == [[10999]]        # other noise
    assert gz._batch_plan(10999, 1, 8, "ssn", "living", "other", root, 4) == [[10999]]     # other save_dir
    assert gz._batch_plan(11001, 1, 8, "ssn", "living", "out", root, 3) == []              # three nodes: done
    assert gz._batch_plan(10998, 3, 0, "ssn", "living", "out", root, 4) == [[10998], [11000]]


def test_get_input_signals_structure(tmp_path):
    from oracle.make_tango_main import make_tango_dataset
    root = str(tmp_path)
    make_tango_dataset(root)
    base = os.path.join(root, "disco", "living", "test", "wav_processed", "0-6")
    for rir, L in ((11001, 41000), (11002, 47513), (11003, 55300)):
        out = gz.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        assert isinstance(out, tuple) and len(out) == 3
        for lst in out:
            assert isinstance(lst, list) and len(lst) == 4 and all(isinstance(node, list) and len(node) == 4
                                                                   for node in lst)
            assert all(ch.dtype == np.float32 and ch.shape == (L,) for node in lst for ch in node)
        y, s, n = out
        for lst, name in ((y, "mixture/%d_ssn_Ch-7.wav"), (s, "target/%d_Ch-7.wav"), (n, "noise/%d_ssn_Ch-7.wav")):
            want = wav_io.read(os.path.join(base, name % rir), dtype="float32")[0]
            assert np.array_equal(lst[1][2], want)                               # Ch-7 = node 2, microphone 3
    y, _, _ = gz.get_input_signals(11001, path_to_dataset=root, nb_ch=(2, 2))       # the first 4 microphones
    assert [len(node) for node in y] == [2, 2]
    # the driver's batch: zero-padded to the longest, each RIR's own length kept
    data = gz._read_batch([11001, 11002, 11003], "living", "ssn", root, (4, 4, 4, 4))
    assert data["sig"].shape == (3, 3, 4, 4, 55300) and list(data["lengths"]) == [41000, 47513, 55300]
    assert not data["sig"][:, 0, ..., 41000:].any()
    assert np.array_equal(data["sig"][0, 1, 1, 2, :47513], gz.get_input_signals(11002, path_to_dataset=root)[0][1][2])


@pytest.fixture
def no_device(monkeypatch):
    """A driver whose device stage, and the loading of a network, fail the test if reached."""
    def reached(*a, **k):
        raise AssertionError("device work was started")
    monkeypatch.setattr(gz, "_compress", reached)
    monkeypatch.setattr(gz, "tango_step1", reached)
    monkeypatch.setattr(gz, "load_models", reached)


def _run(root, vad="irm1", **kw):
    kw.setdefault("nb_rir", 3)
    kw.setdefault("batch", 3)
    gz.main(vad, "out", 11001, "ssn", path_to_dataset=root, device="cpu", **kw)


def test_argument_errors_before_any_file_is_read(tmp_path, no_device, monkeypatch):
    def read(*a, **k):
        raise AssertionError("a file was read")
    monkeypatch.setattr(gz, "_read_batch", read)
    monkeypatch.setattr(gz, "_batch_plan", read)
    root = str(tmp_path)
    with pytest.raises(TypeError, match="NoneType"):
        _run(root, mask_z=None)
    for vad in ("crnn", "rnn"):
        with pytest.raises(ValueError, match="weights_sc"):
            _run(root, vad=vad)
    with pytest.raises(ValueError, match="Unknown value for `mask_type`"):
        _run(root, vad="irm")
    with pytest.raises(ValueError, match="same number of microphones"):
        _run(root, nb_ch=(4, 4, 2, 4))
    assert os.listdir(root) == []


def test_weights_are_loaded_for_networks_only(tmp_path, monkeypatch):
    """weights_sc (the command line's default './' included) is not loaded for oracle masks; a network loads the
    single-channel CRNN once."""
    loaded = []
    monkeypatch.setattr(gz, "load_models", lambda w, device=None: loaded.append((list(w), device)) or [None])
    monkeypatch.setattr(gz, "_batch_plan", lambda *a: [])
    for vad in ("irm1", "ibm2", "iam1", "ivad"):
        _run(str(tmp_path), vad=vad, weights_sc="./")
    assert loaded == []
    _run(str(tmp_path), vad="crnn", weights_sc="sc.pt")
    assert loaded == [(["sc.pt"], torch.device("cpu"))]


def test_load_models_builds_the_single_channel_crnn(tmp_path):
    from disco_b200 import dnn_mask
    torch.manual_seed(0)
    path = str(tmp_path / "sc.pt")
    torch.save({"model_state_dict": dnn_mask.build_crnn(1).state_dict()}, path)
    mods = gz.load_models([path, None], device="cpu")
    assert len(mods) == 1 and not mods[0].training
    want = torch.load(path)["model_state_dict"]
    got = mods[0].state_dict()
    assert set(got) == set(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert gz.load_models([None]) == [None]


def test_input_errors_before_device_work(tmp_path, no_device):
    from oracle.make_tango_main import make_tango_dataset
    root = str(tmp_path)
    make_tango_dataset(root)
    proc = os.path.join(root, "disco", "living", "test", "wav_processed", "0-6")
    # a channel of another length
    bad = os.path.join(proc, "noise", "11002_ssn_Ch-5.wav")
    x, fs = wav_io.read(bad)
    wav_io.write(bad, x[:-10], fs)
    with pytest.raises(ValueError, match="11002_ssn_Ch-5.wav"):
        _run(root)
    wav_io.write(bad, x, fs)
    # a channel at another rate
    bad = os.path.join(proc, "mixture", "11003_ssn_Ch-9.wav")
    wav_io.write(bad, wav_io.read(bad)[0], 8000)
    with pytest.raises(ValueError, match="11003_ssn_Ch-9.wav"):
        _run(root)
    # a missing file
    os.remove(os.path.join(proc, "target", "11001_Ch-16.wav"))
    with pytest.raises(FileNotFoundError, match="11001_Ch-16.wav"):
        _run(root)
    assert not os.path.exists(os.path.join(root, "disco", "living", "test", "stft_z"))


def test_pipeline_writes_cut_spectra_and_surfaces_writer_errors(tmp_path, monkeypatch):
    """The reader / device / writer pipeline with a stand-in device stage (z_y = frame index + i * RIR, zn = -z_y):
    each RIR's files hold its own T_b = 1 + L_b // 256 frames as C-ordered (F, T_b) arrays, and an error on the
    writer thread is raised by main."""
    from oracle.make_tango_main import make_tango_dataset
    root = str(tmp_path)
    make_tango_dataset(root)

    def fake(data, vad, mods, mask_for_z, dev):
        B, K, C, L = data["sig"][0].shape
        t = torch.arange(gz.ops.n_frames(L), dtype=torch.float32).view(1, 1, -1, 1).expand(B, K, -1, 257)
        z = torch.complex(t, torch.tensor(data["rirs"], dtype=torch.float32).view(B, 1, 1, 1).expand_as(t))
        return {"z_y": z.contiguous(), "zn": -z}
    monkeypatch.setattr(gz, "_compress", fake)
    _run(root, batch=2)
    base = gz._save_root(root, "living", 11001, "out")
    for rir, L in ((11001, 41000), (11002, 47513), (11003, 55300)):
        for k in range(1, 5):
            z = np.load(os.path.join(base, "raw", "0-6", "zs_hat", "%d_ssn_Node-%d.npy" % (rir, k)))
            assert z.dtype == np.complex64 and z.shape == (257, 1 + L // 256) and z.flags.c_contiguous
            assert np.array_equal(z.real[0], np.arange(1 + L // 256)) and (z.imag == rir).all()
            zn = np.load(os.path.join(base, "normed", "abs", "0-6", "zn_hat", "%d_ssn_Node-%d.npy" % (rir, k)))
            assert zn.dtype == np.float32 and np.array_equal(zn, np.abs(-z))
    # an unwritable stft_z tree: the writer thread's error comes out of main
    import shutil
    shutil.rmtree(os.path.join(root, "disco", "living", "test", "stft_z"))
    with open(os.path.join(root, "disco", "living", "test", "stft_z"), "w") as fh:
        fh.write("not a directory")
    with pytest.raises((FileExistsError, NotADirectoryError)):
        _run(root, batch=2)
