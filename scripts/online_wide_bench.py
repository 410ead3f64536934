"""Time the online (recursive) statistics at D = C + K - 1 >= 9 and the whole online_tango call at the MEETIT
geometry (8 nodes x 2 mics, step 2 at D = 9).

  scm        ops.scm_recursive alone: 16 utterances x 8 nodes x 2 mics x 10 s with Z of all nodes (D = 9) and
             32 x 1 node x 16 mics (D = 16), block 8, frame-major masks.  CUDA events around --launches launches,
             --runs times after warm-up; min and median per launch, algorithmic bytes (in 8DFT + 4FT per group, out
             16JFD^2 per group, 16FD^2 more in with R0) and their share of 3.35 TB/s.
  ab         with --ab-lib PATH (a build of the same ABI that runs D = 9 on the one-thread-per-(bin, block) template
             plus scm_combine): both libraries on the D = 9 input, alternated run by run in this process, and
             whether their matrices are bit-identical.
  tango      online.online_tango on 16 utterances x 8 nodes x 2 mics x 10 s (block 8, lag 1): the whole call timed,
             then the per-kernel split from torch.profiler in a separate run.

Prints one JSON line per measurement, with the card's name and power limit read in the same run; writes nothing.

    python scripts/online_wide_bench.py [--runs 5] [--launches 20] [--ab-lib PATH] [--skip-tango]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from disco_b200 import _lib, online, ops  # noqa: E402

HBM = 3.35e12       # H100 SXM data-sheet HBM3 bandwidth, bytes/s
N_FFT, HOP, FS = 512, 256, 16000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(), "unknown"


def per_launch_ms(fn, runs, launches):
    """min and median over `runs` of the mean time of `launches` back-to-back calls (CUDA events)."""
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / launches)
    return ts


def scm_bytes(n_grp, D, T, F, J, r0=False):
    """Algorithmic bytes of one scm_recursive call: every input read once, every output matrix written once."""
    per = 8 * D * F * T + 4 * F * T + 16 * J * F * D * D + (16 * F * D * D if r0 else 0)
    return n_grp * per


def make_input(dev, B, K, C, T, F, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    cplx = lambda *s: torch.view_as_complex(torch.randn(*s, 2, device=dev, generator=g))
    Y = cplx(B, K, C, T, F)
    Z = cplx(B, K, T, F) if K > 1 else None
    m = torch.rand(B, K, T, F, device=dev, generator=g)
    return Y, Z, m


def call_lib(lib, Y, Z, m, Rss, Rnn, lam, block, K, C, T):
    B = Y.shape[0]
    _lib.check(lib.disco_scm_recursive(ops._ptr(Y), ops._ptr(Z), ops._ptr(m), None, None, ops._ptr(Rss), ops._ptr(Rnn),
                                       lam, block, 2, B, K, C, T, N_FFT, None, 0, ops._stream()))


def bench_scm(dev, args, meta):
    T, F, block, lam = 1 + 10 * FS // HOP, N_FFT // 2 + 1, 8, 0.95
    J = (T + block - 1) // block
    for name, B, K, C in (("cfg5_step2_D9", 16, 8, 2), ("array16_D16", 32, 1, 16)):
        D = C + K - 1
        Y, Z, m = make_input(dev, B, K, C, T, F, 1)
        fn = lambda: ops.scm_recursive(Y, m, Z, lam, block, 2)
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = per_launch_ms(fn, args.runs, args.launches)
        nb = scm_bytes(B * K, D, T, F, J)
        print(json.dumps({"what": "scm_recursive", "shape": name, "B": B, "K": K, "C": C, "D": D, "T": T, "block": block,
                          "min_ms": round(min(ts), 4), "median_ms": round(float(np.median(ts)), 4),
                          "algo_GB": round(nb / 1e9, 3), "hbm_frac_at_min": round(nb / (min(ts) * 1e-3) / HBM, 3),
                          **meta}), flush=True)
        if args.ab_lib and D == 9:
            bench_ab(Y, Z, m, lam, block, K, C, T, args, meta)
        del Y, Z, m
        torch.cuda.empty_cache()


def bench_ab(Y, Z, m, lam, block, K, C, T, args, meta):
    """The in-tree library against --ab-lib on the same input, alternated run by run."""
    old = ctypes.CDLL(os.path.abspath(args.ab_lib))
    res, argt = _lib.SIGNATURES["disco_scm_recursive"]
    old.disco_scm_recursive.restype, old.disco_scm_recursive.argtypes = res, argt
    new = _lib.load()
    B, F, D = Y.shape[0], Y.shape[-1], C + K - 1
    J = (T + block - 1) // block
    outs = {}
    for tag, lib in (("new", new), ("old", old)):
        Rss = torch.empty((B, K, J, F, D, D), dtype=torch.complex64, device=Y.device)
        Rnn = torch.empty_like(Rss)
        outs[tag] = (lib, Rss, Rnn)
        for _ in range(3):
            call_lib(lib, Y, Z, m, Rss, Rnn, lam, block, K, C, T)
    torch.cuda.synchronize()
    same = all(torch.equal(outs["new"][i], outs["old"][i]) for i in (1, 2))
    times = {"new": [], "old": []}
    for _ in range(args.runs):
        for tag in ("new", "old"):
            lib, Rss, Rnn = outs[tag]
            times[tag] += per_launch_ms(lambda: call_lib(lib, Y, Z, m, Rss, Rnn, lam, block, K, C, T), 1, args.launches)
    print(json.dumps({"what": "ab_D9", "bit_identical": same,
                      **{"%s_%s_ms" % (tag, s): round(f(times[tag]), 4) for tag in times
                         for s, f in (("min", min), ("median", lambda x: float(np.median(x))))}, **meta}), flush=True)
    del outs


def bench_tango(dev, args, meta):
    B, K, C, L, block = 16, 8, 2, 10 * FS, 8
    g = torch.Generator(device=dev).manual_seed(2)
    y = torch.randn(B, K, C, L, device=dev, generator=g)
    T, F = 1 + L // HOP, N_FFT // 2 + 1
    mz = torch.rand(B, K, T, F, device=dev, generator=g)
    mw = torch.rand(B, K, T, F, device=dev, generator=g)
    fn = lambda: online.online_tango(y, (mz, mw), lambda_cor=0.95, block=block, lag=1, n_fft=N_FFT)
    fn()
    torch.cuda.synchronize()
    ts = per_launch_ms(fn, args.runs, 1)
    print(json.dumps({"what": "online_tango", "B": B, "K": K, "C": C, "seconds": L // FS, "block": block,
                      "min_ms": round(min(ts), 3), "median_ms": round(float(np.median(ts)), 3), **meta}), flush=True)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = getattr(e, "cuda_time_total", 0.0)
        if us > 0:
            rows.append((e.key, e.count, us))
    rows.sort(key=lambda r: -r[2])
    print(json.dumps({"what": "online_tango_profile", "kernels": [
        {"name": k[:90], "calls": c, "ms": round(us / 1e3, 3)} for k, c, us in rows[:14]], **meta}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--ab-lib", default=None)
    ap.add_argument("--skip-tango", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("online_wide_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    name, power = card()
    meta = {"card": name, "power_limit": power}
    bench_scm(dev, args, meta)
    if not args.skip_tango:
        bench_tango(dev, args, meta)


if __name__ == "__main__":
    main()
