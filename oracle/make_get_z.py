"""Golden files of the z-signal driver (disco_b200/get_z.py) from the UNMODIFIED reference -- TEST INFRASTRUCTURE.

Run where the reference is mounted:

    python oracle/make_get_z.py

writes tests/golden/get_z_kat.npz (the reference's get_z_signals.main, get_z_signals.py:320-360, on
oracle.make_tango_main.make_tango_dataset, run through oracle/ref_shim.py) and
tests/golden/reference_signatures_get_z.json (the signatures of main and the helpers it calls, extracted from the
reference source as oracle/make_signatures.py extracts the others).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden")

GET_Z_NODES = (1, 3)          # nodes whose |zn_hat| the golden keeps
FRAME_STEP = 4                # every FRAME_STEP-th frame of them, as tango_main_kat keeps |z|
KINDS = ("zs_hat", "zn_hat")


def get_z_kat(ref):
    """Files of the reference's get_z_signals.main on make_tango_dataset, RIRs TANGO_MAIN_RIRS, 'irm1', mask_z 'local'.
    Substituted:
      * soundfile -> disco_b200.wav_io (an absent third-party package);
      * the module globals path_to_dataset (the temporary data set), nb_ch = [4, 4, 4, 4] and ref_mics = [0, 0, 0, 0]
        (their defaults, set again so that the run does not depend on an earlier import);
      * load_models -> a two-argument function that returns [None]: main calls load_models(vad_type, weights)
        (get_z_signals.py:343) but load_models takes one argument (:95), so the unmodified main raises TypeError
        for every mask type.  With oracle masks the models are not used.

    Kept: the file tree under stft_z/out/; each file's dtype and shape; |zn_hat| of nodes GET_Z_NODES, every
    FRAME_STEP-th frame, float32; per normed/abs file the largest |abs file - |raw file||.  zs_hat is step 1's z_y,
    which tests/golden/tango_main_kat.npz already pins: the generator checks that it is bit for bit the |z| stored
    there instead of storing it twice."""
    import importlib
    from disco_b200 import wav_io
    from oracle.make_tango_main import FRAME_STEP as TANGO_FRAME_STEP
    from oracle.make_tango_main import TANGO_MAIN_NODES, TANGO_MAIN_RIRS, make_tango_dataset, tree_digest
    import tempfile
    sfm = sys.modules["soundfile"]
    sfm.read, sfm.write = wav_io.read, wav_io.write
    gz = importlib.import_module("disco_theque.speech_enhancement.get_z_signals")
    gz.load_models = lambda vad_type, weights: [None]
    kat = np.load(os.path.join(OUT, "tango_main_kat.npz"))
    blob = {}
    with tempfile.TemporaryDirectory() as root:
        make_tango_dataset(root)
        blob["dataset_sha256"] = np.array(tree_digest(os.path.join(root, "disco")))
        assert str(blob["dataset_sha256"]) == str(kat["dataset_sha256"])
        gz.path_to_dataset, gz.nb_ch, gz.ref_mics = root, np.array([4, 4, 4, 4]), [0, 0, 0, 0]
        for rir in TANGO_MAIN_RIRS:
            gz.main("irm1", "out", rir, "ssn", mask_z="local")
        out = os.path.join(root, "disco", "living", "test", "stft_z", "out")
        tree = sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out) for f in fs)
        blob["tree"] = np.array(tree)
        arrays = {rel: np.load(os.path.join(out, rel)) for rel in tree}
        blob["dtype"] = np.array([str(arrays[rel].dtype) for rel in tree])
        blob["shape"] = np.array([arrays[rel].shape for rel in tree], dtype=np.int64)
        normed = [rel for rel in tree if rel.startswith("normed")]
        blob["abs_files"] = np.array(normed)
        blob["abs_dev"] = np.array([np.max(np.abs(arrays[rel] - np.abs(arrays[raw_name(rel)]))) for rel in normed],
                                   dtype=np.float64)
        for rir in TANGO_MAIN_RIRS:
            for node in GET_Z_NODES:
                blob["znabs_%d_%d" % (rir, node)] = np.abs(arrays[file_name("raw", "zn_hat", rir, node)])[:, ::FRAME_STEP]
            for node in TANGO_MAIN_NODES:
                zs = arrays[file_name("raw", "zs_hat", rir, node)]
                assert np.array_equal(np.abs(zs)[:, ::TANGO_FRAME_STEP], kat["zabs_%d_%d" % (rir, node)]), (rir, node)
    np.savez_compressed(os.path.join(OUT, "get_z_kat.npz"), **blob)
    print("get_z_signals.main KATs written (%d files in the tree)" % len(tree))


def file_name(sub, kind, rir, node, noise="ssn", dirry="0-6"):
    """Path of one z file relative to stft_z/<save_dir>/ (get_z_signals.py:352-359); sub 'raw' or 'normed'."""
    parts = ("raw",) if sub == "raw" else ("normed", "abs")
    return os.path.join(*parts, dirry, kind, "%d_%s_Node-%d.npy" % (rir, noise, node))


def raw_name(rel):
    """The raw file a normed/abs file is the magnitude of."""
    return os.path.join("raw", os.path.relpath(rel, os.path.join("normed", "abs")))


FUNCTIONS_GET_Z = {
    "disco_theque/speech_enhancement/get_z_signals.py": ["main", "get_input_signals", "load_models", "get_dset",
                                                         "get_directory_name"],
}


def signatures_get_z():
    """tests/golden/reference_signatures_get_z.json, by the extraction of oracle/make_signatures.py run on
    FUNCTIONS_GET_Z (its module globals name the table and the output file)."""
    from oracle import make_signatures as ms
    saved = ms.FUNCTIONS, ms.OUT
    ms.FUNCTIONS, ms.OUT = FUNCTIONS_GET_Z, os.path.join(OUT, "reference_signatures_get_z.json")
    try:
        ms.main()
    finally:
        ms.FUNCTIONS, ms.OUT = saved


if __name__ == "__main__":
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    from oracle import ref_shim
    get_z_kat(ref_shim.load())
    signatures_get_z()
