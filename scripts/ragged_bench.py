"""Time Tango on a batch of ragged arrays three ways (oracle irm1 masks from s, n; mask_for_z 'local'; n_fft 512):

  ragged    one ragged.tango_ragged call on the packed batch, geometry [2, 4, 6, 4] (step 2 at D = 5 .. 9)
  loop      tango.offline_tango once per utterance on the same data (NumPy lists in, NumPy lists out)
  uniform   tango_batched on the uniform geometry [4, 4, 4, 4]: the same 16 microphones, the same bytes

64 utterances x 10 s at 16 kHz.  `--warmup` untimed rounds, then `--runs` rounds, each timing the three ways in turn
with CUDA events and a final synchronise; prints min / median in ms with the card's name and power limit, and writes
nothing.

    python scripts/ragged_bench.py [--utts 64] [--seconds 10] [--runs 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200.ragged import tango_ragged  # noqa: E402
from disco_b200.synth import make_batch  # noqa: E402
from disco_b200.tango import offline_tango, tango_batched  # noqa: E402

RAGGED = [2, 4, 6, 4]
UNIFORM = [4, 4, 4, 4]


def _timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        q = "%s, power limit not readable" % torch.cuda.get_device_name(0)
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fs", type=int, default=16000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, L, n_fft = args.utts, int(args.seconds * args.fs), 512
    K, cmax = len(RAGGED), max(RAGGED)
    # one set of signals: the ragged geometry takes the first C_k microphones of each node, the uniform one 4
    y, s, n = make_batch(B, K, cmax, L, seed0=1)
    pack = lambda a, chans: np.ascontiguousarray(np.concatenate([a[:, k, :c] for k, c in enumerate(chans)], axis=1))
    yr, sr, nr = (torch.from_numpy(pack(a, RAGGED)).to(dev) for a in (y, s, n))
    yu, su, nu = (torch.from_numpy(np.ascontiguousarray(a[:, :, :4])).to(dev) for a in (y, s, n))
    lists = [tuple([[a[b, k, c] for c in range(C)] for k, C in enumerate(RAGGED)] for a in (y, s, n))
             for b in range(B)]
    ways = {
        "ragged": lambda: tango_ragged(yr, RAGGED, sr, nr, n_fft=n_fft),
        "loop": lambda: [offline_tango(*u, "irm1", None, "local", n_fft=n_fft) for u in lists],
        "uniform": lambda: tango_batched(yu, su, nu, n_fft=n_fft),
    }
    for _ in range(args.warmup):
        for fn in ways.values():
            fn()
    torch.cuda.synchronize()
    ts = {w: [] for w in ways}
    for _ in range(args.runs):
        for w, fn in ways.items():
            ts[w].append(_timed(fn))
    res = {w: {"min_ms": round(min(v), 3), "median_ms": round(float(np.median(v)), 3)} for w, v in ts.items()}
    print(json.dumps({"utts": B, "seconds": args.seconds, "n_fft": n_fft, "ragged": RAGGED, "uniform": UNIFORM,
                      "card": _card(), **res}))


if __name__ == "__main__":
    main()
