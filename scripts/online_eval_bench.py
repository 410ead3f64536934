"""Time what evaluating online (recursive) Tango from the clean components costs over the bare deployment step:

  masks     online_tango(y, (mask_z, mask_w)): the masks given, five outputs
  eval      online_tango(y, s=s, n=n, vads=("irm1", "irm2")): the masks built from s, n, and the diagnostics z_s, z_n,
            sf, nf (four more filter_sum_blocks passes and the two clean STFTs)
  no_diag   the same with diagnostics=False: the masks built from s, n, no filtered images

64 utterances x 4 nodes x 4 mics x 10 s at 16 kHz, n_fft 512, block 8, lag 1; the masks of `masks` are those `eval`
builds (irm1 / irm2 of the images, made once outside the timing).  CUDA events around each call, `--warmup` untimed
calls of each way, then `--runs` rounds that time each way once in turn; prints one JSON line with min / median in ms,
the card and its power limit, and writes nothing.

    python scripts/online_eval_bench.py [--utts 64] [--runs 5] [--warmup 2]
"""
import argparse
import datetime
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200.online import online_tango  # noqa: E402
from disco_b200.synth import make_batch  # noqa: E402


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fs", type=int, default=16000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, K, C, L, n_fft, block = args.utts, 4, 4, 10 * args.fs, 512, 8
    y, s, n = (torch.from_numpy(a).to(dev) for a in make_batch(B, K, C, L, seed0=1))
    kw = dict(block=block, lag=1, n_fft=n_fft)
    vads = ("irm1", "irm2")
    first = online_tango(y, s=s, n=n, vads=vads, diagnostics=False, **kw)
    masks = (first["masks_z"], first["mask_w"])
    del first
    ways = {
        "masks": lambda: online_tango(y, masks, **kw),
        "eval": lambda: online_tango(y, s=s, n=n, vads=vads, **kw),
        "no_diag": lambda: online_tango(y, s=s, n=n, vads=vads, diagnostics=False, **kw),
    }
    for f in ways.values():
        for _ in range(args.warmup):
            f()
    torch.cuda.synchronize()
    ts = {w: [] for w in ways}
    for _ in range(args.runs):
        for w, f in ways.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            torch.cuda.synchronize()
            ts[w].append(a.elapsed_time(b))
    res = {w: {"min_ms": round(min(t), 3), "median_ms": round(float(np.median(t)), 3)} for w, t in ts.items()}
    print(json.dumps({"utts": B, "K": K, "C": C, "seconds": L / args.fs, "n_fft": n_fft, "block": block, **res,
                      "gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(),
                      "session": datetime.datetime.now(datetime.timezone.utc).isoformat(timespec="seconds")}))


if __name__ == "__main__":
    main()
