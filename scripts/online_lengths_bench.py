"""Time online (recursive) Tango on a dataset-like batch of utterances of different lengths three ways:

  lengths   one online_tango(..., lengths=) call on the batch zero-padded to its longest utterance
  loop      one online_tango call per utterance, each on its own length
  uniform   the batch of the same count at the longest length, every utterance that long

64 utterances with lengths drawn uniformly from 7-11 s at 16 kHz, at 1 node x 4 mics, 4 nodes x 4 mics and 8 nodes x
2 mics (step 2 at D = 9, the staged wide scan); block 8, lag 1, n_fft 512, irm1 / irm2 masks of the images (made
once, outside the timing).  CUDA events around each way, `--warmup` untimed calls, then `--runs` timed calls; prints
min / median in ms and writes nothing.

    python scripts/online_lengths_bench.py [--utts 64] [--runs 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200 import ops  # noqa: E402
from disco_b200.online import online_tango  # noqa: E402
from disco_b200.synth import make_batch  # noqa: E402
from lengths_bench import _time  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--fs", type=int, default=16000)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    B, n_fft = args.utts, 512
    lengths = rng.integers(7 * args.fs, 11 * args.fs + 1, size=B)
    L = int(lengths.max())
    frames = ops.n_frames(lengths, n_fft)
    for K, C in ((1, 4), (4, 4), (8, 2)):
        y, s, n = make_batch(B, K, C, L, seed0=1)
        for b, Lb in enumerate(lengths):
            for a in (y, s, n):
                a[b, ..., Lb:] = 0
        yd = torch.from_numpy(y).to(dev)
        S = ops.stft_lengths(torch.from_numpy(s[:, :, 0]).to(dev), lengths, n_fft)
        N = ops.stft_lengths(torch.from_numpy(n[:, :, 0]).to(dev), lengths, n_fft)
        masks = (ops.tf_mask(S, N, "irm1"), ops.tf_mask(S, N, "irm2"))
        del S, N
        solo = [(yd[b:b + 1, ..., :Lb].contiguous(), tuple(m[b:b + 1, :, :Tb].contiguous() for m in masks))
                for b, (Lb, Tb) in enumerate(zip(lengths, frames))]
        ways = {
            "lengths": lambda: online_tango(yd, masks, lengths=lengths),
            "loop": lambda: [online_tango(u, mu) for u, mu in solo],
            "uniform": lambda: online_tango(yd, masks),
        }
        res = {w: _time(f, args.runs, args.warmup) for w, f in ways.items()}
        print(json.dumps({"K": K, "C": C, "utts": B, "L_max": L,
                          "mean_len_s": round(float(lengths.mean()) / args.fs, 3),
                          "gpu": torch.cuda.get_device_name(0), **res}))
        del yd, masks, solo
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
