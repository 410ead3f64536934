"""Latency of the online Tango stream (disco_b200/stream.py) at the shapes its options opened, next to the whole-signal
online_tango with the same options.

    python scripts/stream_options_latency.py [--seconds 10] [--runs 3]

The method of scripts/stream_latency.py: B streams at 16 kHz, n_fft 512, block 8, lag 1, pushed in chunks of 8 hops
(2048 samples, 128 ms).  Two configurations:
  64 x (8 nodes x 2 mics)   D = 9 in step 2 (the MEETIT geometry), masks sliced from fixed device tensors
  64 x (4 nodes x 4 mics)   with clean components: s, n pushed next to y, oracle masks vads = ("irm1", "irm1") built
                            by the stream, and the outputs z_s, z_n, sf, nf and the six time signals
Per configuration one JSON line:
  push_ms          CUDA-event time of one push (the host waits for its outputs after every push): median over the
                   pushes of a run, then median and min-max over the runs
  rtf              real-time factor of the whole batch, B x 0.128 s of audio per push over push_ms
  launches_push    kernels one steady-state push runs (torch.profiler, a run of its own)
  offline_ms       the same audio through online_tango on the whole signal, same options (median of the runs)
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
VADS = ("irm1", "irm1")


def gpu_info():
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return {"gpu": torch.cuda.get_device_name(0), "power_limit": pl or "unknown"}


class Config:
    """One measured shape: its signals and how a stream and the whole-signal run take them."""

    def __init__(self, B, K, C, clean, L, dev):
        rng = np.random.default_rng(0)
        T, F = ops.n_frames(L, N_FFT), N_FFT // 2 + 1
        self.B, self.K, self.C, self.clean = B, K, C, clean
        if clean:
            self.s = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
            self.n = torch.from_numpy(0.5 * rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
            self.y = self.s + self.n
            self.fn = None
        else:
            self.y = torch.from_numpy(rng.standard_normal((B, K, C, L)).astype(np.float32)).to(dev)
            mz = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
            mw = torch.from_numpy(rng.uniform(0.05, 0.95, (B, K, T, F)).astype(np.float32)).to(dev)
            self.masks = (mz, mw)
            self.fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]])

    def stream(self):
        return OnlineTangoStream(self.B, self.K, self.C, n_fft=N_FFT, block=BLOCK, lag=1, device=self.y.device,
                                 vads=VADS if self.clean else None, wide=True)

    def push(self, st, p):
        sn = dict(s_chunk=self.s[..., p:p + CHUNK], n_chunk=self.n[..., p:p + CHUNK]) if self.clean else {}
        return st.push(self.y[..., p:p + CHUNK], self.fn, **sn)

    def whole(self):
        if self.clean:
            return online_tango(self.y, None, block=BLOCK, lag=1, n_fft=N_FFT, s=self.s, n=self.n, vads=VADS)
        return online_tango(self.y, self.masks, block=BLOCK, lag=1, n_fft=N_FFT)


def session(cfg, times=None):
    """Push the signals chunk by chunk, then flush; with `times`, append the CUDA-event time (ms) of every full push."""
    L = cfg.y.shape[-1]
    st = cfg.stream()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for p in range(0, L, CHUNK):
        ev[0].record()
        cfg.push(st, p)
        ev[1].record()
        ev[1].synchronize()
        if times is not None and p + CHUNK <= L:
            times.append(ev[0].elapsed_time(ev[1]))
    st.flush(cfg.fn)
    torch.cuda.synchronize()


def launches_per_push(cfg):
    """Kernels of one steady-state push (the 5th), counted in a profiled run of its own."""
    st = cfg.stream()
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
    assert torch.cuda.is_available(), "stream_options_latency.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    L = int(args.seconds * FS)
    for B, K, C, clean in ((64, 8, 2, False), (64, 4, 4, True)):
        cfg = Config(B, K, C, clean, L, dev)
        session(cfg)                                         # warm-up
        run_ms = []
        for _ in range(args.runs):
            times = []
            session(cfg, times)
            run_ms.append(float(np.median(times)))
        n_launch, names = launches_per_push(cfg)
        cfg.whole()
        torch.cuda.synchronize()
        off = []
        for _ in range(args.runs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            cfg.whole()
            e1.record()
            e1.synchronize()
            off.append(e0.elapsed_time(e1))
        med = float(np.median(run_ms))
        print(json.dumps({
            "B": B, "K": K, "C": C, "D": C + K - 1, "clean": clean, "vads": VADS if clean else None,
            "n_fft": N_FFT, "block": BLOCK, "lag": 1, "chunk": CHUNK, "seconds": L / FS, "runs": args.runs,
            "push_ms": round(med, 4), "push_ms_min": round(min(run_ms), 4), "push_ms_max": round(max(run_ms), 4),
            "rtf": round(B * CHUNK / FS / (med / 1e3), 1), "launches_push": n_launch, "kernels": names,
            "offline_ms": round(float(np.median(off)), 3)}), flush=True)
        del cfg
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
