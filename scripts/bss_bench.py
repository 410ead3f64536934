"""Times BSS-eval on the device against the float64 NumPy oracle on the host and prints one JSON line.

    python scripts/bss_bench.py [--utts 64] [--nodes 4] [--seconds 10] [--reps 5]

GPU: post.tango_scores at the cfg-3 shape (utts x nodes utterances of `seconds` s at 16 kHz: the dry reference set of
each utterance and the convolved one of each node, three estimate sets each), and bss_eval_sources at tango.main's
per-node shape (2 references x 2 estimates, 144 000 samples), CUDA events, median of `reps`.  CPU: the oracle
(oracle/bss_np.py, mir_eval's algorithm) on one call of the per-node shape, single-threaded BLAS unless the
environment says otherwise.  The card name and its power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def gpu_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--nodes", type=int, default=4)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cpu-reps", type=int, default=1)
    args = ap.parse_args()
    from disco_b200 import bss_eval, post
    from oracle import bss_np
    dev = torch.device("cuda:0")
    fs = 16000
    L = int(args.seconds * fs)
    B, K = args.utts, args.nodes
    g = torch.Generator(device=dev).manual_seed(0)
    rnd = lambda *s: 0.1 * torch.randn(*s, device=dev, generator=g)
    s, n = rnd(B, K, L), rnd(B, K, L)
    y = s + n
    times = {k: rnd(B, K, L) for k in ("yf", "z_y", "sf", "nf", "z_s", "z_n")}
    s_dry, n_dry = rnd(B, L), rnd(B, L)
    t_scores = gpu_ms(lambda: post.tango_scores(y, s, n, s_dry, n_dry, times, fs), args.reps)
    Ln = L - fs
    refs, ests = rnd(2, Ln), rnd(2, Ln)
    t_call = gpu_ms(lambda: bss_eval.bss_eval_sources(refs, ests, compute_permutation=False), args.reps)
    r64, e64 = refs.double().cpu().numpy(), ests.double().cpu().numpy()
    ts = []
    for _ in range(args.cpu_reps):
        t0 = time.perf_counter()
        bss_np.bss_eval_sources(r64, e64, compute_permutation=False)
        ts.append(time.perf_counter() - t0)
    name, power = card()
    print(json.dumps({
        "metric": "bss_eval", "card": name, "power_limit": power,
        "tango_scores_ms": round(t_scores, 3), "tango_scores_shape": [B, K, L],
        "bss_eval_call_ms": round(t_call, 3), "call_shape": [2, 2, Ln],
        "oracle_cpu_s_per_call": round(float(np.median(ts)), 4),
        "oracle_cpu_threads": os.environ.get("OMP_NUM_THREADS", "default"),
    }))


if __name__ == "__main__":
    main()
