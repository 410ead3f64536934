"""Latency of the pool of independent online Tango streams (disco_b200/stream.py OnlineTangoPool) on the GPU, alternated
in the same run with the lockstep OnlineTangoStream on audio of the same shape.

    python scripts/pool_latency.py [--seconds 6] [--runs 3]

S slots of K nodes x C microphones at 16 kHz, n_fft 512, block 8, lag 1, pushes of 2048 samples (128 ms, one block).
Slot s opens at push s mod 8 and its first push carries (s mod 8 + 1) hops, so the slots' frames sit at every offset
within a block: their block closes spread over the pushes, and a push runs two rounds (one where the offset is 0).
Masks are gathered from fixed device tensors.  Per configuration one JSON line:
  pool_push_ms     CUDA-event time of one push once every slot is open (the host waits for its outputs after every
                   push): median over the pushes of a run, then median and min-max over the runs
  lockstep_push_ms the same for OnlineTangoStream(S, K, C) pushing all slots in lockstep, runs alternated with the pool's
  pool_launches_push / lockstep_launches_push   kernels of one steady-state push (torch.profiler, a run of its own)
  pool_rounds_push the pool's rounds in that push
The first line names the GPU and its power limit, read in the same run."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np
import torch

from disco_b200 import ops
from disco_b200.stream import OnlineTangoPool, OnlineTangoStream
from stream_latency import gpu_info

FS, N_FFT, BLOCK, CHUNK, STAGGER = 16000, 512, 8, 2048, 8


class PoolSession:
    def __init__(self, y, mz, mw):
        self.y, self.mz, self.mw = y, mz, mw
        S, K, C, L = y.shape
        self.pool = OnlineTangoPool(S, K, C, n_fft=N_FFT, block=BLOCK, lag=1, device=y.device)
        self.rounds = 0

    def fn(self, t0, n_fr, Y, z, zn):
        """The masks of frames [t0[s], t0[s] + n_fr[s]) of every slot: one gather from the fixed tensors."""
        self.rounds += 1
        f, S = z.shape[2], z.shape[0]
        t = torch.from_numpy(np.minimum(t0[:, None] + np.arange(f), self.mz.shape[2] - 1)).to(self.y.device)
        idx = t[:, None, :, None].expand(S, z.shape[1], f, z.shape[3])
        return torch.gather(self.mz, 2, idx), torch.gather(self.mw, 2, idx)

    def run(self, pushes, times=None, profile_at=None):
        """`pushes` pushes; slot s opens at push s mod STAGGER and receives the signal from its own start."""
        S, K, C, L = self.y.shape
        pos = np.zeros(S, dtype=np.int64)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        prof = None
        for p in range(pushes):
            opening = [s for s in range(S) if s % STAGGER == p]
            if opening:
                self.pool.open(opening)
            is_open = np.array([self.pool.is_open(s) for s in range(S)])
            first = np.array([(s % STAGGER + 1) * (N_FFT // 2) if s in opening else CHUNK for s in range(S)])
            n = np.where(is_open, np.minimum(first, L - pos), 0)
            chunk = torch.zeros((S, K, C, CHUNK), device=self.y.device)
            for s in np.nonzero(n)[0]:
                chunk[s, ..., :n[s]] = self.y[s, ..., pos[s]:pos[s] + n[s]]
            torch.cuda.synchronize()
            self.rounds = 0
            if p == profile_at:
                prof = torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                                          torch.profiler.ProfilerActivity.CUDA])
                prof.__enter__()
            ev[0].record()
            self.pool.push(chunk, n, self.fn)
            ev[1].record()
            ev[1].synchronize()
            if prof is not None and p == profile_at:
                prof.__exit__(None, None, None)
                kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
                return len(kern), self.rounds
            if times is not None and p >= STAGGER:
                times.append(ev[0].elapsed_time(ev[1]))
            pos += n
        return None


def lockstep(y, mz, mw, pushes, times=None):
    S, K, C, L = y.shape
    s = OnlineTangoStream(S, K, C, n_fft=N_FFT, block=BLOCK, lag=1, device=y.device)
    fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]])
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for p in range(pushes):
        ev[0].record()
        s.push(y[..., p * CHUNK:(p + 1) * CHUNK], fn)
        ev[1].record()
        ev[1].synchronize()
        if times is not None and p >= STAGGER:
            times.append(ev[0].elapsed_time(ev[1]))
    return s


def lockstep_launches(y, mz, mw):
    s = lockstep(y, mz, mw, STAGGER)
    fn = lambda t0, Y, z, zn: (mz[:, :, t0:t0 + Y.shape[3]], mw[:, :, t0:t0 + Y.shape[3]])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                            torch.profiler.ProfilerActivity.CUDA]) as prof:
        s.push(y[..., STAGGER * CHUNK:(STAGGER + 1) * CHUNK], fn)
        torch.cuda.synchronize()
    return len([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=6.0)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "pool_latency.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    for S, K, C in ((256, 1, 4), (64, 4, 4)):
        L = int(args.seconds * FS) // CHUNK * CHUNK
        pushes = L // CHUNK
        rng = np.random.default_rng(0)
        y = torch.from_numpy(rng.standard_normal((S, K, C, L)).astype(np.float32)).to(dev)
        T, F = ops.n_frames(L, N_FFT), N_FFT // 2 + 1
        mz = torch.from_numpy(rng.uniform(0.05, 0.95, (S, K, T, F)).astype(np.float32)).to(dev)
        mw = torch.from_numpy(rng.uniform(0.05, 0.95, (S, K, T, F)).astype(np.float32)).to(dev)
        PoolSession(y, mz, mw).run(pushes)                       # warm-up
        lockstep(y, mz, mw, pushes)
        pool_ms, lock_ms = [], []
        for _ in range(args.runs):                               # alternated
            t = []
            PoolSession(y, mz, mw).run(pushes, t)
            pool_ms.append(float(np.median(t)))
            t = []
            lockstep(y, mz, mw, pushes, t)
            lock_ms.append(float(np.median(t)))
        n_pool, rounds = PoolSession(y, mz, mw).run(pushes, profile_at=STAGGER + 1)
        n_lock = lockstep_launches(y, mz, mw)
        pm, lm = float(np.median(pool_ms)), float(np.median(lock_ms))
        print(json.dumps({
            "S": S, "K": K, "C": C, "n_fft": N_FFT, "block": BLOCK, "lag": 1, "chunk": CHUNK, "seconds": L / FS,
            "runs": args.runs, "pool_push_ms": round(pm, 4), "pool_push_ms_min": round(min(pool_ms), 4),
            "pool_push_ms_max": round(max(pool_ms), 4), "lockstep_push_ms": round(lm, 4),
            "lockstep_push_ms_min": round(min(lock_ms), 4), "lockstep_push_ms_max": round(max(lock_ms), 4),
            "pool_over_lockstep": round(pm / lm, 3), "pool_launches_push": n_pool, "pool_rounds_push": rounds,
            "lockstep_launches_push": n_lock}), flush=True)


if __name__ == "__main__":
    main()
