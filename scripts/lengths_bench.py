"""Time a dataset-like batch of utterances of different lengths three ways (tango_batched with oracle irm1 masks):

  lengths   one tango_batched(..., lengths=) call on the batch zero-padded to its longest utterance
  loop      one tango_batched call per utterance, each on its own length
  uniform   the batch of the same count at the longest length, every utterance that long (the fused routes)

64 utterances with lengths drawn uniformly from 7-11 s at 16 kHz, at 1 node x 4 mics and 4 nodes x 4 mics.
CUDA events around each way, `--warmup` untimed calls, then `--runs` timed calls; prints min / median in ms and
writes nothing.

    python scripts/lengths_bench.py [--utts 64] [--runs 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200.synth import make_batch  # noqa: E402
from disco_b200.tango import tango_batched  # noqa: E402


def _time(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return {"min_ms": round(min(ts), 3), "median_ms": round(float(np.median(ts)), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fs", type=int, default=16000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    B = args.utts
    lengths = rng.integers(7 * args.fs, 11 * args.fs + 1, size=B)
    L = int(lengths.max())
    for K, C in ((1, 4), (4, 4)):
        y, s, n = make_batch(B, K, C, L, seed0=1)
        for b, Lb in enumerate(lengths):
            for a in (y, s, n):
                a[b, ..., Lb:] = 0
        yd, sd, nd = (torch.from_numpy(a).to(dev) for a in (y, s, n))
        solo = [tuple(t[b:b + 1, ..., :Lb].contiguous() for t in (yd, sd, nd)) for b, Lb in enumerate(lengths)]
        ways = {
            "lengths": lambda: tango_batched(yd, sd, nd, lengths=lengths),
            "loop": lambda: [tango_batched(*u) for u in solo],
            "uniform": lambda: tango_batched(yd, sd, nd),
        }
        res = {w: _time(f, args.runs, args.warmup) for w, f in ways.items()}
        print(json.dumps({"K": K, "C": C, "utts": B, "L_max": L, "mean_len_s": round(float(lengths.mean()) / args.fs, 3),
                          "gpu": torch.cuda.get_device_name(0), **res}))
        del yd, sd, nd, solo
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
