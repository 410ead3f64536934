"""Time the z-signal driver (disco_b200/get_z.py) on a synthetic data set, against the per-RIR loop a user writes
today from the reference-signature adapters.

N RIRs of 4 nodes x 4 microphones, 9-11 s at 16 kHz, are generated from a seed into a temporary directory that is
deleted at exit: make_tango_dataset's convolved sources, mixed into wav_processed/ by PostGenerator.  Then

  main      get_z.main('irm1', mask_z 'local') over the N RIRs at each --batches value, into a fresh stft_z/ tree each
            time (deleted after the run); RIRs/s over the whole call and what share of that wall time went to the host
            read (reader thread), the device work (CUDA events around the masks, step 1 and the device-to-host copy)
            and the host write (writer thread).  The same again with the writes made in the main thread
            ('serial_write') tells whether the writer thread pays
  loop      per RIR, what get_z_signals.main does through the adapters: get_input_signals,
            compat.get_z_signals.offline_tango and save_z_signals.  Timed on the first --loop RIRs

One untimed call of each way first.  Prints the card's name and power limit and one JSON line.

    python scripts/get_z_bench.py [--rirs 64] [--batches 1 8 32] [--loop 8] [--seed 5]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import Future

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200 import get_z as gz  # noqa: E402
from disco_b200.dataset_post import PostGenerator, save_z_signals  # noqa: E402
from oracle.make_tango_main import make_tango_dataset  # noqa: E402

FIRST = 11001            # the 'test' set of get_dset / PostGenerator


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def make_data(root, n, seed):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(9 * 16000, 11 * 16000 + 1, size=n)
    make_tango_dataset(root, seed=seed, rirs=range(FIRST, FIRST + n), lengths=lengths, dry_extra=[(0, 0)] * n,
                       processed=False)
    np.random.seed(seed)
    PostGenerator(FIRST, n, "living", "ssn", [0, 6], os.path.join(root, "disco"), batch=8).post_process()
    return lengths


class Inline:
    """An executor that runs what it is given at once, in the calling thread."""

    def __init__(self, max_workers=None):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def submit(self, fn, *a, **k):
        f = Future()
        try:
            f.set_result(fn(*a, **k))
        except BaseException as e:          # noqa: B902 - handed to the caller through the future, as a pool would
            f.set_exception(e)
        return f


class Timed:
    """Wraps the driver's read, device and write stages to time each batch; serial_write=True makes main's second
    executor (the writer's) an Inline one."""

    def __init__(self, serial_write=False):
        self.read, self.device, self.write = [], [], []
        self.serial_write = serial_write
        self._orig = (gz._read_batch, gz._compress, gz._to_host, gz._write_batch, gz.ThreadPoolExecutor)

    def __enter__(self):
        read, compress, host, write, pool = self._orig

        def t_read(*a, **k):
            t0 = time.perf_counter()
            out = read(*a, **k)
            self.read.append(time.perf_counter() - t0)
            return out

        def t_compress(*a, **k):
            self._ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            self._ev[0].record()
            return compress(*a, **k)

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
        made = []

        def executor(max_workers=None):
            made.append(None)
            return Inline() if self.serial_write and len(made) % 2 == 0 else pool(max_workers=max_workers)
        gz._read_batch, gz._compress, gz._to_host, gz._write_batch = t_read, t_compress, t_host, t_write
        gz.ThreadPoolExecutor = executor
        return self

    def __exit__(self, *exc):
        gz._read_batch, gz._compress, gz._to_host, gz._write_batch, gz.ThreadPoolExecutor = self._orig


def run_main(root, n, batch, tag, serial_write=False):
    with Timed(serial_write) as t:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        gz.main("irm1", tag, FIRST, "ssn", nb_rir=n, batch=batch, path_to_dataset=root)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    shutil.rmtree(gz._save_root(root, "living", FIRST, tag))
    share = lambda x: {"sum_s": round(float(np.sum(x)), 3), "median_s": round(float(np.median(x)), 4),
                       "share_of_wall": round(float(np.sum(x)) / wall, 3)}
    return {"batch": batch, "writer": "main thread" if serial_write else "writer thread", "rirs": n,
            "wall_s": round(wall, 3), "rirs_per_s": round(n / wall, 2), "read": share(t.read),
            "device": share(t.device), "write": share(t.write)}


def adapter_loop(root, rirs, save_dir):
    """get_z_signals.main's per-RIR calls through the adapters, files written."""
    from disco_b200.compat.get_z_signals import offline_tango
    for rir in rirs:
        y, s, n = gz.get_input_signals(rir, "living", "ssn", path_to_dataset=root)
        z_sh, _, _, z_nh, _ = offline_tango(y, s, n, "irm1", mods=[None], mask_for_z="local")
        save_z_signals(z_sh, z_nh, gz._save_root(root, "living", rir, save_dir), "0-6", rir, "ssn")
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rirs", type=int, default=64)
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--loop", type=int, default=8, help="RIRs timed in the per-RIR adapter loop")
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("get_z_bench needs a CUDA device")
    gpu = card()
    print("card:", gpu, flush=True)
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        lengths = make_data(root, a.rirs, a.seed)
        print("data set: %d RIRs, mean %.2f s, max %.2f s (%.1f s to generate)"
              % (a.rirs, lengths.mean() / 16000, lengths.max() / 16000, time.perf_counter() - t0), flush=True)
        run_main(root, min(a.rirs, max(a.batches)), max(a.batches), "warmup")
        adapter_loop(root, [FIRST], "warmup_loop")
        shutil.rmtree(gz._save_root(root, "living", FIRST, "warmup_loop"))
        rows = []
        for b in a.batches:
            for serial in (False, True):
                rows.append(run_main(root, a.rirs, b, "b%d%s" % (b, "s" if serial else ""), serial))
                print(json.dumps(rows[-1]), flush=True)
        n_loop = min(a.loop, a.rirs)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        adapter_loop(root, range(FIRST, FIRST + n_loop), "loop")
        loop_s = time.perf_counter() - t0
        shutil.rmtree(gz._save_root(root, "living", FIRST, "loop"))
    print(json.dumps({"card": gpu, "rirs": a.rirs, "mean_len_s": round(float(lengths.mean()) / 16000, 3),
                      "main": rows, "adapter_loop": {"rirs": n_loop, "wall_s": round(loop_s, 3),
                                                     "rirs_per_s": round(n_loop / loop_s, 3)}}))


if __name__ == "__main__":
    main()
