"""Latency of the online Tango stream (disco_b200/stream.py) on the GPU, next to the whole-signal online_tango.

    python scripts/stream_latency.py [--seconds 10] [--runs 3]

B streams of K nodes x C microphones at 16 kHz, n_fft 512, block 8, lag 1, pushed in chunks of 8 hops (2048 samples,
128 ms); masks are slices of fixed device tensors.  Per configuration it prints one JSON line:
  push_ms          CUDA-event time of one push (the host waits for its outputs after every push, as a caller that
                   consumes them does): median over the pushes of a run, then median and min-max over the runs
  rtf              real-time factor of the whole batch, B x 0.128 s of audio per push over push_ms
  launches_push    kernels one steady-state push runs (torch.profiler, a run of its own)
  offline_ms, offline_frames_per_s   the same audio through online_tango on the whole signal (median of the runs)
The first line names the GPU and its power limit."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from disco_b200 import ops
from disco_b200.online import online_tango
from disco_b200.stream import OnlineTangoStream

FS, N_FFT, BLOCK, CHUNK = 16000, 512, 8, 2048


def gpu_info():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl or "unknown"}


def session(y, mz, mw, times=None):
    """Push y chunk by chunk, then flush; with `times`, append the CUDA-event time (ms) of every full push."""
    B, K, C, L = y.shape
    s = OnlineTangoStream(B, K, C, n_fft=N_FFT, block=BLOCK, lag=1, device=y.device)
    fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for p in range(0, L, CHUNK):
        ev[0].record()
        s.push(y[..., p:p + CHUNK], fn)
        ev[1].record()
        ev[1].synchronize()
        if times is not None and p + CHUNK <= L:
            times.append(ev[0].elapsed_time(ev[1]))
    s.flush(fn)
    torch.cuda.synchronize()


def launches_per_push(y, mz, mw):
    """Kernels of one steady-state push (the 5th), counted in a profiled run of its own."""
    B, K, C, L = y.shape
    s = OnlineTangoStream(B, K, C, n_fft=N_FFT, block=BLOCK, lag=1, device=y.device)
    fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]])
    for p in range(0, 4 * CHUNK, CHUNK):
        s.push(y[..., p:p + CHUNK], fn)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        s.push(y[..., 4 * CHUNK:5 * CHUNK], fn)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(kern), sorted({e.name for e in kern})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_latency.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    for B, K, C in ((256, 1, 4), (64, 4, 4)):
        L = int(args.seconds * FS)
        rng = np.random.default_rng(0)
        y = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
        T, F = ops.n_frames(L, N_FFT), N_FFT // 2 + 1
        mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        session(y, mz, mw)                                   # warm-up
        run_ms = []
        for _ in range(args.runs):
            times = []
            session(y, mz, mw, times)
            run_ms.append(float(np.median(times)))
        n_launch, names = launches_per_push(y, mz, mw)
        online_tango(y, (mz, mw), block=BLOCK, lag=1, n_fft=N_FFT)
        torch.cuda.synchronize()
        off = []
        for _ in range(args.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            online_tango(y, (mz, mw), block=BLOCK, lag=1, n_fft=N_FFT)
            e1.record()
            e1.synchronize()
            off.append(e0.elapsed_time(e1))
        med = float(np.median(run_ms))
        off_ms = float(np.median(off))
        print(json.dumps({
            "B": B, "K": K, "C": C, "n_fft": N_FFT, "block": BLOCK, "lag": 1, "chunk": CHUNK, "seconds": L / FS,
            "runs": args.runs, "push_ms": round(med, 4), "push_ms_min": round(min(run_ms), 4),
            "push_ms_max": round(max(run_ms), 4), "rtf": round(B * CHUNK / FS / (med / 1e3), 1),
            "launches_push": n_launch, "kernels": names,
            "offline_ms": round(off_ms, 3), "offline_frames_per_s": round(B * K * T / (off_ms / 1e3))}), flush=True)


if __name__ == "__main__":
    main()
