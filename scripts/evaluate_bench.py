"""Time the evaluation driver (disco_b200/evaluate.py) on a synthetic data set, against the per-RIR loop a user writes
today from the reference-signature adapters.

N RIRs of 4 nodes x 4 microphones, 7-11 s at 16 kHz, are generated from a seed into a temporary directory that is
deleted at exit: make_tango_dataset's convolved and dry sources, mixed into wav_processed/ by PostGenerator.  Then

  main      evaluate.main(irm1, irm1, mask_z 'local') over the N RIRs at each --batches value, into a fresh results
            tree each time; RIRs/s over the whole call, and per batch the host read (in its background thread), the
            device work (CUDA events around beamforming, time signals, scores and the device-to-host copy) and the
            host write
  loop      per RIR, the calls of tango.main (tango.py:490-593) through the adapters: get_input_signals,
            offline_tango, 6 x 4 my_istft, and per node the 6 compat.separation, 6 compat.stoi, 4 compat.metrics.fw_snr
            and 4 fw_sd calls; files are not written.  Timed on the first --loop RIRs

One untimed call of each way first.  Prints the card's name and power limit and one JSON line.

    python scripts/evaluate_bench.py [--rirs 64] [--batches 1 8 32] [--loop 8] [--seed 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200 import evaluate as ev  # noqa: E402
from disco_b200.dataset_post import PostGenerator  # noqa: E402
from oracle.make_tango_main import make_tango_dataset  # noqa: E402

FIRST = 11001            # the 'test' set of get_dset / PostGenerator


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def make_data(root, n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(7 * 16000, 11 * 16000 + 1, size=n)
    make_tango_dataset(root, seed=seed, rirs=range(FIRST, FIRST + n), lengths=lengths, dry_extra=[(0, 0)] * n,
                       processed=False)
    np.random.seed(seed)
    PostGenerator(FIRST, n, "living", "ssn", [0, 6], os.path.join(root, "disco"), batch=8).post_process()
    return lengths


class Timed:
    """Wraps the driver's read, device and write stages to time each batch."""

    def __init__(self):
        self.read, self.device, self.write = [], [], []
        self._orig = (ev._read_batch, ev._beamform, ev._to_host, ev._write_batch)

    def __enter__(self):
        read, beam, host, write = self._orig

        def t_read(*a, **k):
            t0 = time.perf_counter()
            out = read(*a, **k)
            self.read.append(time.perf_counter() - t0)
            return out

        def t_beam(*a, **k):
            self._ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self._ev[0].record()
            return beam(*a, **k)

        def t_host(*a, **k):
            out = host(*a, **k)
            self._ev[1].record()
            self._ev[1].synchronize()
            self.device.append(self._ev[0].elapsed_time(self._ev[1]) / 1e3)
            return out

        def t_write(*a, **k):
            t0 = time.perf_counter()
            write(*a, **k)
            self.write.append(time.perf_counter() - t0)
        ev._read_batch, ev._beamform, ev._to_host, ev._write_batch = t_read, t_beam, t_host, t_write
        return self

    def __exit__(self, *exc):
        ev._read_batch, ev._beamform, ev._to_host, ev._write_batch = self._orig


def run_main(root, n, batch, tag):
    results = os.path.join(root, "results_" + tag)
    with Timed() as t:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.main(["irm1", "irm1"], "out", FIRST, "ssn", nb_rir=n, batch=batch, path_to_dataset=root,
                results_root=results)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    stat = lambda x: {"sum_s": round(float(np.sum(x)), 3), "median_s": round(float(np.median(x)), 4)}
    return {"batch": batch, "rirs": n, "wall_s": round(wall, 3), "rirs_per_s": round(n / wall, 2),
            "read": stat(t.read), "device": stat(t.device), "write": stat(t.write)}


def adapter_loop(root, rirs):
    """tango.main's per-RIR calls through the adapters (no files written)."""
    from disco_b200.compat import metrics, separation, stoi
    from disco_b200.compat.math_utils import my_istft
    from disco_b200.tango import offline_tango
    for rir in rirs:
        y, s, n, s_dry, n_dry, fs, _ = ev.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        sh, s_f, n_f, z_sh, z_s, z_n, _, _, _ = offline_tango(y, s, n, ["irm1", "irm1"], mods=[None, None],
                                                               mask_for_z="local")
        L = len(s[0][0])
        for k in range(len(y)):
            sh_t, szh_t, sf_t, nf_t, szf_t, nzf_t = (my_istft(x[k], L) for x in (sh, z_sh, s_f, n_f, z_s, z_n))
            m = min(L, len(sh_t), len(s_dry), len(n_dry))
            c = lambda x: x[fs:m]
            refs_dry, refs = np.vstack((c(s_dry), c(n_dry))), np.vstack((c(s[k][0]), c(n[k][0])))
            for ests in (np.vstack((c(sh_t), c(y[k][0]) - c(sh_t))), np.vstack((c(szh_t), c(y[k][0]) - c(szh_t))),
                         np.vstack((c(y[k][0]), c(y[k][0]) - c(sh_t)))):
                separation.bss_eval_sources(refs_dry, ests, compute_permutation=False)
                separation.bss_eval_sources(refs, ests, compute_permutation=False)
            for clean in (c(s[k][0]), c(s_dry)):
                for deg in (c(y[k][0]), c(sh_t), c(szh_t)):
                    stoi.stoi(clean, deg, fs)
            for a, b in ((sf_t, nf_t), (s[k][0], n[k][0]), (s_dry, n_dry), (szf_t, nzf_t)):
                metrics.fw_snr(c(a), c(b), fs)
            for a, b in ((sf_t, s[k][0]), (sf_t, s_dry), (szf_t, s[k][0]), (szf_t, s_dry)):
                metrics.fw_sd(c(a), c(b), fs)
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rirs", type=int, default=64)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--loop", type=int, default=8, help="RIRs timed in the per-RIR adapter loop")
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("evaluate_bench needs a CUDA device")
    gpu = card()
    print("card:", gpu, flush=True)
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        lengths = make_data(root, a.rirs, a.seed)
        print("data set: %d RIRs, mean %.2f s, max %.2f s (%.1f s to generate)"
              % (a.rirs, lengths.mean() / 16000, lengths.max() / 16000, time.perf_counter() - t0), flush=True)
        run_main(root, min(a.rirs, max(a.batches)), max(a.batches), "warmup")
        adapter_loop(root, [FIRST])
        rows = []
        for b in a.batches:
            rows.append(run_main(root, a.rirs, b, "b%d" % b))
            print(json.dumps(rows[-1]), flush=True)
        n_loop = min(a.loop, a.rirs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        adapter_loop(root, range(FIRST, FIRST + n_loop))
        loop_s = time.perf_counter() - t0
    print(json.dumps({"card": gpu, "rirs": a.rirs, "mean_len_s": round(float(lengths.mean()) / 16000, 3),
                      "main": rows, "adapter_loop": {"rirs": n_loop, "wall_s": round(loop_s, 3),
                                                     "rirs_per_s": round(n_loop / loop_s, 3)}}))


if __name__ == "__main__":
    main()
