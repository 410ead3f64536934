"""Golden files of the evaluation driver (disco_b200/evaluate.py) from the UNMODIFIED reference -- TEST INFRASTRUCTURE.

Run where the reference is mounted:

    python -m oracle.make_tango_main

writes tests/golden/tango_main_kat.npz (the reference's tango.main, tango.py:460-641, on make_tango_dataset, run
through oracle/ref_shim.py) and tests/golden/reference_signatures_main.json (the signatures of main and the helpers it
calls, extracted from the reference source as oracle/make_signatures.py extracts the others).
"""
import hashlib
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

TANGO_MAIN_RIRS = (11001, 11002, 11003)


def make_tango_dataset(root, seed=41, rirs=TANGO_MAIN_RIRS, lengths=(41000, 47513, 55300),
                       dry_extra=((-700, -300), (900, 500), (0, 0)), noise="ssn", scene="living", processed=True):
    """A tiny data set in the layout tango.get_input_signals reads (tango.py:74-109) under root/disco/<scene>/<set>/:
    per RIR 16 microphones (4 nodes x 4) of a gated target and a stationary noise, each convolved with its own decaying
    random response and cut to the RIR's length, the noise with sensor noise added (wav_original/cnv/), and the two
    dry sources, whose lengths differ from the convolved ones by dry_extra (wav_original/dry/).  processed=True also mixes them as PostGenerator does
    (post_generator.py:99-118: one SNR in [0, 6] dB per RIR, the noise scaled in float32, the mixture summed in
    float64) into wav_processed/0-6/ and log/snrs/dry/0-6/; processed=False leaves that to PostGenerator.
    16-bit PCM at 16 kHz.  Shared by the golden generator, the tests and scripts/evaluate_bench.py."""
    from disco_b200 import wav_io
    rng = np.random.default_rng(seed)
    fs = 16000
    for rir, L, (d_t, d_n) in zip(rirs, lengths, dry_extra):
        base = os.path.join(root, "disco", scene, "train" if rir < 11001 else "test")
        j = lambda *p: os.path.join(base, *p)
        for d in ("wav_original/dry/target", "wav_original/dry/noise", "wav_original/cnv/target",
                  "wav_original/cnv/noise"):
            os.makedirs(j(d), exist_ok=True)
        colour = np.exp(-np.arange(24) / 4.0) * rng.standard_normal(24)
        on = (np.arange(L + d_t) % 12000) < 8000                       # speech-like on / off pattern
        s_dry = np.convolve(rng.standard_normal(L + d_t + 23), colour, "valid") * on
        n_dry = rng.standard_normal(L + d_n)
        s_dry, n_dry = 0.3 * s_dry / np.abs(s_dry).max(), 0.3 * n_dry / np.abs(n_dry).max()
        wav_io.write(j("wav_original/dry/target", "%d_S-1.wav" % rir), s_dry, fs)
        wav_io.write(j("wav_original/dry/noise", "%d_S-2_%s.wav" % (rir, noise)), n_dry, fs)
        fit = lambda x: np.pad(x, (0, max(0, L - len(x))))[:L]
        for ch in range(1, 17):
            decay = np.exp(-np.arange(64) / 12.0)
            h_s, h_n = rng.standard_normal(64) * decay, rng.standard_normal(64) * decay
            h_s[0], h_n[0] = 2.0, 2.0
            wav_io.write(j("wav_original/cnv/target", "%d_S-1_Ch-%d.wav" % (rir, ch)),
                         0.5 * np.convolve(fit(s_dry), h_s)[:L] / np.linalg.norm(h_s), fs)
            # plus an independent sensor noise 20 dB below the source's: the noise field is not rank one, as in a
            # room, so the step-2 statistics are well conditioned
            cnv = np.convolve(fit(n_dry), h_n)[:L] / np.linalg.norm(h_n)
            wav_io.write(j("wav_original/cnv/noise", "%d_S-2_%s_Ch-%d.wav" % (rir, noise, ch)),
                         0.5 * (cnv + 0.1 * np.std(cnv) * rng.standard_normal(L)), fs)
        if not processed:
            continue
        snr = rng.uniform(0, 6)
        gain = np.float32(10 ** (-snr / 20))
        for d in ("target", "noise", "mixture"):
            os.makedirs(j("wav_processed", "0-6", d), exist_ok=True)
        os.makedirs(j("log", "snrs", "dry", "0-6"), exist_ok=True)
        for ch in range(1, 17):
            t = wav_io.read(j("wav_original/cnv/target", "%d_S-1_Ch-%d.wav" % (rir, ch)))[0]
            n = wav_io.read(j("wav_original/cnv/noise", "%d_S-2_%s_Ch-%d.wav" % (rir, noise, ch)))[0] * gain
            wav_io.write(j("wav_processed", "0-6", "target", "%d_Ch-%d.wav" % (rir, ch)), t, fs)
            wav_io.write(j("wav_processed", "0-6", "noise", "%d_%s_Ch-%d.wav" % (rir, noise, ch)), n, fs)
            wav_io.write(j("wav_processed", "0-6", "mixture", "%d_%s_Ch-%d.wav" % (rir, noise, ch)),
                         t.astype(np.float64) + n.astype(np.float64), fs)
        np.save(j("log", "snrs", "dry", "0-6", "%d_%s" % (rir, noise)), np.array([snr]))


def tree_digest(root):
    """sha256 over the relative paths and bytes of every file under root, in sorted order."""
    h = hashlib.sha256()
    for rel in sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs):
        h.update(rel.encode())
        with open(os.path.join(root, rel), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


TANGO_MAIN_NODES = (1, 3)           # nodes whose MASK and STFT/z arrays the golden keeps
# every FRAME_STEP-th frame of those arrays and every SAMPLE_STEP-th sample of the out_* / mid_z WAVs are kept, which
# holds the fixture to the size of the repository's other golden files
FRAME_STEP, SAMPLE_STEP = 4, 4
WAV_NAMES = ("in_mix", "out_mix", "mid_z", "in_noi", "out_noi", "in_tar", "out_tar")


def pcm_sha256(x):
    """sha256 of the 16-bit samples of a signal wav_io.read returned."""
    return hashlib.sha256(np.round(np.asarray(x, np.float64) * 32768).astype("<i2").tobytes()).hexdigest()


def tango_main_kat(ref):
    """Files of the reference's tango.main (tango.py:460-641) on make_tango_dataset, 'irm1' / 'irm1', mask_z 'local'.
    Substituted: soundfile -> disco_b200.wav_io, the names tango.py bound at import bss -> oracle.bss_np and stoi ->
    oracle.stoi_np (both absent third-party packages), save_conf -> no-op (a matplotlib figure).  main writes
    results/ under the working directory, so it runs in a temporary one.

    Kept: the file tree; both pickles; of nodes TANGO_MAIN_NODES the step-1 masks, the step-2 masks where they differ
    from step 1, and |z| (the parity metric reads magnitudes only), every FRAME_STEP-th frame, with each file's dtype and
    shape; of one node per RIR the sha256 of the in_* WAV samples and every SAMPLE_STEP-th sample of out_* and mid_z."""
    import pickle
    import sys
    import tempfile
    from disco_b200 import wav_io
    from oracle import bss_np, stoi_np
    sfm = sys.modules["soundfile"]
    sfm.read, sfm.write = wav_io.read, wav_io.write
    t = ref.tango
    t.bss, t.stoi, t.save_conf = bss_np.bss_eval_sources, stoi_np.stoi, lambda *a, **k: None
    blob = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as root:
        make_tango_dataset(root)
        blob["dataset_sha256"] = np.array(tree_digest(os.path.join(root, "disco")))
        t.path_to_dataset, t.nb_ch, t.ref_mics = root, np.array([4, 4, 4, 4]), [0, 0, 0, 0]
        try:
            os.chdir(root)
            for rir in TANGO_MAIN_RIRS:
                t.main(["irm1", "irm1"], "out", rir, "ssn")
        finally:
            os.chdir(cwd)
        out = os.path.join(root, "results", "living", "test", "out")
        blob["tree"] = np.array(sorted(os.path.relpath(os.path.join(d, f), out) for d, _, fs in os.walk(out)
                                       for f in fs))
        for i, rir in enumerate(TANGO_MAIN_RIRS):
            for kind in ("tango", "mwf"):
                with open(os.path.join(out, "OIM", "results_%s_%d_ssn.p" % (kind, rir)), "rb") as fh:
                    res = pickle.load(fh)
                blob["keys_%d_%s" % (rir, kind)] = np.array(list(res))
                for k, v in res.items():
                    blob["p_%d_%s_%s" % (rir, kind, k)] = np.asarray(v)
            for node in TANGO_MAIN_NODES:
                masks = [np.load(os.path.join(out, "MASK", str(rir), "step%d_ssn_Node-%d.npy" % (step, node)))
                         for step in (1, 2)]
                z = np.load(os.path.join(out, "STFT", "z", "raw", "0-6", "%d_ssn_Node-%d.npy" % (rir, node)))
                tag = "%d_%d" % (rir, node)
                blob["mask_1_" + tag] = masks[0][:, ::FRAME_STEP]
                if not np.array_equal(masks[0], masks[1]):
                    blob["mask_2_" + tag] = masks[1][:, ::FRAME_STEP]
                blob["mask_meta_" + tag] = np.array([str(masks[0].dtype), str(masks[1].dtype)])
                blob["mask_shape_" + tag] = np.array(masks[0].shape)
                blob["zabs_" + tag] = np.abs(z)[:, ::FRAME_STEP]
                blob["z_meta_" + tag] = np.array([str(z.dtype)] + [str(v) for v in z.shape])
            node = i % 4 + 1
            blob["wav_node_%d" % rir] = np.array(node)
            for name in WAV_NAMES:
                x = wav_io.read(os.path.join(out, "WAV", str(rir), "%s-ssn_Node-%d.wav" % (name, node)))[0]
                blob["wavlen_%d_%s" % (rir, name)] = np.array(len(x))
                if name.startswith("in_"):
                    blob["wavsha_%d_%s" % (rir, name)] = np.array(pcm_sha256(x))
                else:
                    blob["wav_%d_%s" % (rir, name)] = np.round(x[::SAMPLE_STEP].astype(np.float64) * 32768).astype(np.int16)
    np.savez_compressed(os.path.join(OUT, "tango_main_kat.npz"), **blob)
    print("tango.main KATs written (%d files in the tree)" % len(blob["tree"]))


FUNCTIONS_MAIN = {
    "disco_theque/speech_enhancement/tango.py": ["main", "get_input_signals", "load_models", "get_dset",
                                                 "get_directory_name"],
}


def signatures_main():
    """tests/golden/reference_signatures_main.json, by the extraction of oracle/make_signatures.py run on
    FUNCTIONS_MAIN (its module globals name the table and the output file)."""
    from oracle import make_signatures as ms
    saved = ms.FUNCTIONS, ms.OUT
    ms.FUNCTIONS, ms.OUT = FUNCTIONS_MAIN, os.path.join(OUT, "reference_signatures_main.json")
    try:
        ms.main()
    finally:
        ms.FUNCTIONS, ms.OUT = saved


if __name__ == "__main__":
    from oracle import ref_shim
    tango_main_kat(ref_shim.load())
    signatures_main()
