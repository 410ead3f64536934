"""Latency of the online Tango stream and pool on a ragged array (disco_b200/stream.py with per-node channel counts),
next to the array of equal counts with the same microphones and bytes.

    python scripts/ragged_stream_latency.py [--seconds 10] [--runs 3]

The method of scripts/stream_options_latency.py: 64 streams at 16 kHz, n_fft 512, block 8, lag 1, pushed in chunks
of 8 hops (2048 samples, 128 ms), masks sliced from fixed device tensors by mask_fn.  Four configurations, timed in
one process and alternating run by run after one warm-up session each:
  stream  64 x [2, 4, 6, 4]   three channel-count groups (D = 5, 7, 9)
  stream  64 x [4, 4, 4, 4]   one group (D = 7): the calls of the int-C stream
  pool    64 slots of [2, 4, 6, 4], every slot pushed 2048 samples per push
  pool    64 slots of [4, 4, 4, 4]
Per configuration one JSON line:
  push_ms          CUDA-event time of one push (the host waits for its outputs after every push): median over the
                   pushes of a run, then median and min-max over the runs
  rtf              real-time factor of the whole batch, 64 x 0.128 s of audio per push over push_ms
  launches_push    kernels one steady-state push runs (torch.profiler, a run of its own)
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
from disco_b200.stream import OnlineTangoPool, OnlineTangoStream

FS, N_FFT, BLOCK, CHUNK, B = 16000, 512, 8, 2048, 64
GEOMETRIES = ([2, 4, 6, 4], [4, 4, 4, 4])


def gpu_info():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl or "unknown"}


class Config:
    """One measured shape: packed signals [B, M, L], masks [B, K, T, F], and a stream or a pool that takes them."""

    def __init__(self, kind, channels, L, dev):
        rng = np.random.default_rng(0)
        K, M = len(channels), sum(channels)
        T, F = ops.n_frames(L, N_FFT), N_FFT // 2 + 1
        self.kind, self.channels, self.L, self.dev = kind, channels, L, dev
        self.y = torch.from_numpy(rng.standard_normal((B, M, L)).astype(np.float32)).to(dev)
        mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
        self.fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + z.shape[2]], mw[:, :, t0:t0 + z.shape[2]])
        # every slot of the pool stands at the same frame, so slot s's masks are row s of the same slice
        self.pfn = lambda t0, n_fr, Y, z, zn: self.fn(int(t0.max()), Y, z, zn)

    def name(self):
        return "%s %d x %s" % (self.kind, B, self.channels)

    def open(self):
        kw = dict(n_fft=N_FFT, block=BLOCK, lag=1, device=self.dev)
        K = len(self.channels)
        if self.kind == "stream":
            return OnlineTangoStream(B, K, self.channels, wide=True, **kw)
        pool = OnlineTangoPool(B, K, self.channels, **kw)
        pool.open(list(range(B)))
        return pool

    def push(self, st, p):
        x = self.y[..., p:p + CHUNK]
        if self.kind == "stream":
            return st.push(x, self.fn)
        return st.push(x, np.full(B, x.shape[-1], dtype=np.int64), self.pfn)

    def close(self, st):
        return st.flush(self.fn) if self.kind == "stream" else st.close(list(range(B)), self.pfn)


def session(cfg, times=None):
    """Push the signals chunk by chunk, then end the streams; with `times`, append the CUDA-event time (ms) of every
    full push."""
    st = cfg.open()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for p in range(0, cfg.L, CHUNK):
        ev[0].record()
        cfg.push(st, p)
        ev[1].record()
        ev[1].synchronize()
        if times is not None and p + CHUNK <= cfg.L:
            times.append(ev[0].elapsed_time(ev[1]))
    cfg.close(st)
    torch.cuda.synchronize()


def launches_per_push(cfg):
    """Kernels of one steady-state push (the 5th), counted in a profiled run of its own."""
    st = cfg.open()
    for p in range(0, 4 * CHUNK, CHUNK):
        cfg.push(st, p)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        cfg.push(st, 4 * CHUNK)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return len(kern), sorted({e.name for e in kern})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "ragged_stream_latency.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    L = int(args.seconds * FS)
    cfgs = [Config(kind, ch, L, dev) for kind in ("stream", "pool") for ch in GEOMETRIES]
    for cfg in cfgs:
        session(cfg)                                         # warm-up
    run_ms = {cfg.name(): [] for cfg in cfgs}
    for _ in range(args.runs):
        for cfg in cfgs:
            times = []
            session(cfg, times)
            run_ms[cfg.name()].append(float(np.median(times)))
    for cfg in cfgs:
        ms = run_ms[cfg.name()]
        n_launch, names = launches_per_push(cfg)
        med = float(np.median(ms))
        K = len(cfg.channels)
        print(json.dumps({
            "kind": cfg.kind, "B": B, "channels": cfg.channels, "groups": len(set(cfg.channels)),
            "D": sorted({c + K - 1 for c in cfg.channels}), "n_fft": N_FFT, "block": BLOCK, "lag": 1, "chunk": CHUNK,
            "seconds": L / FS, "runs": args.runs, "push_ms": round(med, 4), "push_ms_min": round(min(ms), 4),
            "push_ms_max": round(max(ms), 4), "rtf": round(B * CHUNK / FS / (med / 1e3), 1),
            "launches_push": n_launch, "kernels": names}), flush=True)


if __name__ == "__main__":
    main()
