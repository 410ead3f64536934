"""The evaluation driver (disco_b200/evaluate.py) without a GPU: signatures, command line, data-set paths, the batch plan,
input reading and the errors raised before any device work."""
import importlib
import inspect
import json
import os
import pickle

import numpy as np
import pytest
import torch

from disco_b200 import evaluate as ev
from disco_b200 import wav_io

REF = "disco_theque/speech_enhancement/tango.py:"
OURS = {name: "disco_b200.evaluate:" + name
        for name in ("main", "get_input_signals", "load_models", "get_dset", "get_directory_name")}


def test_signatures_match_the_reference(golden_dir):
    """Same rule as test_compat_cpu.test_adapter_signatures_match_the_reference, over
    tests/golden/reference_signatures_main.json; compat.tango re-exports the same functions."""
    ref = json.load(open(os.path.join(golden_dir, "reference_signatures_main.json")))
    assert set(ref) == {REF + k for k in OURS}
    compat = importlib.import_module("disco_b200.compat.tango")
    for name, target in OURS.items():
        mod, attr = target.split(":")
        fn = getattr(importlib.import_module(mod), attr)
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


def test_cli_parses_the_reference_flags():
    args, kw = ev.parse_args(["-vt", "irm1", "ibm2", "-sd", "out", "--rir", "11001"])
    assert args == (["irm1", "ibm2"], "out", 11001, "fs")              # --noise defaults to 'fs' (tango.py:664)
    assert kw["scenario"] == "living" and kw["mask_z"] == "local" and kw["z_sigs"] == "zs_hat"
    assert kw["models"] == [None, None]
    assert (kw["nb_rir"], kw["batch"], kw["results_root"], kw["online"], kw["block"], kw["lag"]) == \
        (1, 8, "results", False, 8, 1)
    assert kw["path_to_dataset"] == ev.PATH_TO_DATASET
    args, kw = ev.parse_args(["--vad_type", "crnn", "crnn", "--sav_dir", "x", "--rir", "3", "-scene", "meeting",
                              "--noise", "ssn", "-mz", "None", "-m", "a.pt", "None", "-zs", "zs_hat", "zn_hat",
                              "--nb_rir", "20", "--batch", "4", "--dataset", "/d", "--results", "/r", "--online",
                              "--block", "4", "--lag", "2"])
    assert args == (["crnn", "crnn"], "x", 3, "ssn")
    assert kw["mask_z"] is None and kw["models"] == ["a.pt", None] and kw["z_sigs"] == ["zs_hat", "zn_hat"]
    assert kw["scenario"] == "meeting"
    assert (kw["nb_rir"], kw["batch"], kw["path_to_dataset"], kw["results_root"], kw["online"], kw["block"],
            kw["lag"]) == (20, 4, "/d", "/r", True, 4, 2)
    assert ev.parse_args(["-m", "None", "None"])[1]["models"] == [None, None]
    assert ev.parse_args(["-zs", "zn_hat"])[1]["z_sigs"] == "zn_hat"
    for bad in (["--noise", "wind"], ["-scene", "office"], ["-mz", "global"], ["-vt", "irm1"]):
        with pytest.raises(SystemExit):
            ev.parse_args(bad)


def test_dset_and_directory_names():
    assert [ev.get_dset(r) for r in (1, 11000, 11001, 12000)] == ["train", "train", "test", "test"]
    for r in (0, 12001, -5):
        with pytest.raises(AssertionError, match="between 1 and 12000"):
            ev.get_dset(r)
    assert ev.get_directory_name([[0, 6]]) == "0-6"
    assert ev.get_directory_name([[3, 6], [5, 15]]) == "3-6_5-15"


def _pickle(root, rir, kind, save_dir="out", noise="ssn"):
    d = os.path.join(root, "living", ev.get_dset(rir), save_dir, "OIM")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "results_%s_%d_%s.p" % (kind, rir, noise)), "wb") as fh:
        pickle.dump({}, fh)


def test_batch_plan_skips_finished_rirs(tmp_path, capsys):
    root = str(tmp_path)
    _pickle(root, 10999, "tango")
    _pickle(root, 10999, "mwf")             # finished
    _pickle(root, 11001, "tango")           # interrupted between the two pickles: redone
    _pickle(root, 11003, "mwf")
    plan = ev._batch_plan(10998, 8, 3, "ssn", "living", "out", root)
    assert plan == [[10998, 11000, 11001], [11002, 11004, 11005]]
    out = capsys.readouterr().out
    assert "Conf 10999 with ssn noise already processed" in out and "Conf 11003 with ssn noise already processed" in out
    assert ev._batch_plan(10999, 1, 8, "ssn", "living", "out", root) == []
    assert ev._batch_plan(10999, 1, 8, "fs", "living", "out", root) == [[10999]]        # other noise: not done


def test_get_input_signals_structure(tmp_path):
    from oracle.make_tango_main import make_tango_dataset
    root = str(tmp_path)
    make_tango_dataset(root)
    for rir, L, dry in ((11001, 41000, (40300, 40700)), (11002, 47513, (48413, 48013)), (11003, 55300, (55300, 55300))):
        y, s, n, s_dry, n_dry, fs, snr = ev.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        assert fs == 16000
        for lst in (y, s, n):
            assert isinstance(lst, list) and len(lst) == 4 and all(isinstance(node, list) and len(node) == 4
                                                                   for node in lst)
            assert all(ch.dtype == np.float32 and ch.shape == (L,) for node in lst for ch in node)
        assert s_dry.dtype == n_dry.dtype == np.float32 and (len(s_dry), len(n_dry)) == dry
        base = os.path.join(root, "disco", "living", "test")
        want = np.load(os.path.join(base, "log", "snrs", "dry", "0-6", "%d_ssn.npy" % rir), allow_pickle=True)[0]
        assert type(snr) is type(want) and snr == want
        raw = wav_io.read(os.path.join(base, "wav_original", "dry", "noise", "%d_S-2_ssn.wav" % rir), dtype="float32")[0]
        assert np.array_equal(n_dry, raw * np.float32(10 ** (-want / 20)))      # float32 product
        mix = wav_io.read(os.path.join(base, "wav_processed", "0-6", "mixture", "%d_ssn_Ch-7.wav" % rir))[0]
        assert np.array_equal(y[1][2], mix)                                      # Ch-7 = node 2, microphone 3
    y, *_ = ev.get_input_signals(11001, path_to_dataset=root, nb_ch=(2, 2))     # the first 4 microphones
    assert [len(node) for node in y] == [2, 2]


@pytest.fixture
def no_device(monkeypatch):
    """tango_batched / online_tango that fail the test if reached."""
    def reached(*a, **k):
        raise AssertionError("device work was started")
    monkeypatch.setattr(ev, "tango_batched", reached)
    monkeypatch.setattr(ev, "online_tango", reached)


def _run(root, **kw):
    kw.setdefault("nb_rir", 3)
    kw.setdefault("batch", 3)
    ev.main(["irm1", "irm1"], "out", 11001, "ssn", path_to_dataset=root, results_root=os.path.join(root, "res"),
            device="cpu", **kw)


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
    # a batch of two rates: every file of RIR 11003 at 8 kHz
    for dirpath, _, files in os.walk(os.path.join(root, "disco")):
        for f in files:
            if f.startswith("11003") and f.endswith(".wav"):
                p = os.path.join(dirpath, f)
                wav_io.write(p, wav_io.read(p)[0], 8000)
    with pytest.raises(ValueError, match="11003_Ch-1.wav"):
        _run(root)
    # a missing file
    missing = os.path.join(proc, "mixture", "11001_ssn_Ch-16.wav")
    os.remove(missing)
    with pytest.raises(FileNotFoundError, match="11001_ssn_Ch-16.wav"):
        _run(root)
    os.remove(os.path.join(root, "disco", "living", "test", "log", "snrs", "dry", "0-6", "11001_ssn.npy"))
    with pytest.raises(FileNotFoundError, match="11001_ssn.npy"):
        _run(root)
    assert not any("OIM" in d for d, _, _ in os.walk(os.path.join(root, "res")))


def test_online_rejects_network_masks(tmp_path, no_device):
    with pytest.raises(ValueError, match="not causal"):
        ev.main(["crnn", "irm1"], "out", 11001, "ssn", path_to_dataset=str(tmp_path), online=True, device="cpu")


def test_one_host_copy_round_trips_every_dtype():
    g = torch.Generator().manual_seed(0)
    t = {"a": torch.rand((2, 3, 5), generator=g), "b": torch.rand((2, 3), generator=g, dtype=torch.float64),
         "c": torch.complex(torch.rand((2, 4, 3), generator=g), torch.rand((2, 4, 3), generator=g)).transpose(1, 2)}
    h = ev._to_host(t)
    for k, v in t.items():
        assert h[k].dtype == v.numpy().dtype and np.array_equal(h[k], v.numpy())
