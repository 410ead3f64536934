"""Times STOI on the device against the float64 NumPy oracle on the host and prints one JSON line.

    python scripts/stoi_bench.py [--utts 64] [--nodes 4] [--seconds 10] [--reps 5]

GPU: post.tango_scores(stoi=True) minus post.tango_scores(stoi=False) at the cfg-3 shape (utts x nodes utterances of
`seconds` s at 16 kHz, gated speech-like signals from synth.make_utterance so that the silent-frame removal has pauses
to drop; 6 STOI pairs per node), and one stoi call of tango.main's per-node shape (2 cleans x 3 degraded signals, six
pairs, `seconds` - 1 s), CUDA events, median of `reps`.  CPU: the oracle (oracle/stoi_np.py) on one pair of that
shape.  The card name and its power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bss_bench import card, gpu_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--nodes", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=3)
    args = ap.parse_args()
    from disco_b200 import post, stoi
    from disco_b200.synth import make_utterance
    from oracle import stoi_np
    dev = torch.device("cuda:0")
    fs = 16000
    L = int(args.seconds * fs)
    B, K = args.utts, args.nodes
    gate = fs // 2
    y, s, n = (torch.from_numpy(np.stack(a)[:, :, 0]).to(dev)
               for a in zip(*[make_utterance(b, K, 1, L, gate_period=gate) for b in range(B)]))
    g = torch.Generator(device=dev).manual_seed(0)
    times = {k: s + 0.3 * torch.randn(B, K, L, device=dev, generator=g) for k in ("yf", "z_y", "sf", "nf", "z_s", "z_n")}
    s_dry = torch.from_numpy(np.stack([make_utterance(1000 + b, 1, 1, L, gate_period=gate)[1][0, 0]
                                       for b in range(B)])).to(dev)
    n_dry = 0.05 * torch.randn(B, L, device=dev, generator=g)
    t_with = gpu_ms(lambda: post.tango_scores(y, s, n, s_dry, n_dry, times, fs, stoi=True), args.reps)
    t_without = gpu_ms(lambda: post.tango_scores(y, s, n, s_dry, n_dry, times, fs), args.reps)
    Ln = L - fs
    cleans = torch.stack((s[0, 0, fs:], s_dry[0, fs:]))
    degraded = torch.stack((y[0, 0, fs:], times["yf"][0, 0, fs:], times["z_y"][0, 0, fs:]))
    pairs = torch.tensor([(c, e) for c in range(2) for e in range(3)], dtype=torch.int32, device=dev)
    t_call = gpu_ms(lambda: stoi.stoi_pairs(cleans, degraded, pairs, fs), args.reps)
    x, e = cleans[0].cpu().numpy(), degraded[0].cpu().numpy()
    ts = []
    for _ in range(args.cpu_reps):
        t0 = time.perf_counter()
        stoi_np.stoi(x, e, fs)
        ts.append(time.perf_counter() - t0)
    name, power = card()
    print(json.dumps({
        "metric": "stoi", "card": name, "power_limit": power,
        "tango_scores_stoi_ms": round(t_with, 3), "tango_scores_no_stoi_ms": round(t_without, 3),
        "stoi_part_ms": round(t_with - t_without, 3), "tango_scores_shape": [B, K, L],
        "stoi_node_call_ms": round(t_call, 3), "node_call_shape": [2, 3, Ln],
        "oracle_cpu_s_per_call": round(float(np.median(ts)), 4), "oracle_call_samples": Ln,
    }))


if __name__ == "__main__":
    main()
