"""Cost of saving and moving live online Tango sessions (disco_b200/stream_state.py) on the GPU.

    python scripts/stream_state_cost.py [--slots 64] [--runs 3]

Per geometry, a pool of S slots is opened and pushed in chunks of 2048 samples (128 ms) until every slot has closed
more than `lag` blocks.  Then, slot by slot, the session is exported (release=True), written with torch.save to a
memory buffer, read back with torch.load(weights_only=True) and restored into the same slot of a second pool.  Each
step is timed on the host clock around work that ends with the device idle (export copies to host memory and waits
for the copy; restore is followed by torch.cuda.synchronize): median over the slots of a run, then median and min-max
over the runs after a warm-up run, as in scripts/stream_latency.py.  Each line also gives the state's bytes, counted
from its tensors and from the formula of DESIGN §4.5.  The first line names the GPU and its power limit."""
import argparse
import io
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from disco_b200 import stream_state
from disco_b200.stream import OnlineTangoPool

from stream_latency import gpu_info

CHUNK = 2048
# (K, C or channels, n_fft, block, lag)
GEOMETRIES = [(4, 4, 512, 8, 1), (4, [2, 4, 6, 4], 512, 8, 1), (8, 2, 512, 8, 2), (2, 4, 1024, 64, 1),
              (4, 4, 256, 1, 2)]


def formula_bytes(K, C, n_fft, block, lag, closed, B=1):
    """The bytes of a state without clean components (DESIGN §4.5)."""
    counts = [C] * K if isinstance(C, int) else list(C)
    F, H, M, P = n_fft // 2 + 1, n_fft // 2, sum(counts), block
    nw = min(closed, lag)
    per = 4 * M * n_fft + 8 * M * P * F + 2 * 4 * K * P * F + (8 * K * P * F if K > 1 else 0) + 4 * K * H
    for c in counts:
        D = c + K - 1
        per += 2 * 8 * F * (c * c + D * D) + 8 * nw * F * (c + D)
    return B * per


def fill(K, C, n_fft, block, lag, S, dev, rng):
    """A pool of S open slots, each past lag + 1 blocks and mid-block."""
    pool = OnlineTangoPool(S, K, C, n_fft=n_fft, block=block, lag=lag, device=dev)
    lead = pool._lead(S)
    F, H = n_fft // 2 + 1, n_fft // 2
    pool.open(range(S))
    need = ((lag + 2) * block + block // 2 + 1) * H
    fn = lambda t0, n_fr, Y, z, zn: (torch.full(z.shape, 0.6, device=dev), torch.full(z.shape, 0.3, device=dev))
    while pool.samples_in.min() < need:
        y = torch.from_numpy(rng.standard_normal(lead + (CHUNK,)).astype(np.float32)).to(dev)
        pool.push(y, np.full(S, CHUNK, dtype=np.int64), fn)
    torch.cuda.synchronize()
    return pool


def one_run(geo, S, dev, rng):
    K, C, n_fft, block, lag = geo
    src = fill(K, C, n_fft, block, lag, S, dev, rng)
    dst = OnlineTangoPool(S, K, C, n_fft=n_fft, block=block, lag=lag, device=dev)
    t = {"export": [], "save": [], "load": [], "restore": []}
    nbytes = file_bytes = closed = None
    for s in range(S):
        t0 = time.perf_counter()
        st = src.export(s, release=True)
        t1 = time.perf_counter()
        buf = io.BytesIO()
        torch.save(st, buf)
        t2 = time.perf_counter()
        buf.seek(0)
        back = torch.load(buf, weights_only=True)
        t3 = time.perf_counter()
        dst.restore(s, back)
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        for k, a, b in (("export", t0, t1), ("save", t1, t2), ("load", t2, t3), ("restore", t3, t4)):
            t[k].append((b - a) * 1e3)
        nbytes, file_bytes, closed = stream_state.nbytes(st), buf.getbuffer().nbytes, st["closed"]
    return {k: float(np.median(v)) for k, v in t.items()}, nbytes, file_bytes, closed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_state_cost.py measures on a CUDA device"
    dev = torch.device("cuda:0")
    print(json.dumps(gpu_info()), flush=True)
    rng = np.random.default_rng(0)
    for geo in GEOMETRIES:
        one_run(geo, min(args.slots, 4), dev, rng)                       # warm-up
        runs = [one_run(geo, args.slots, dev, rng) for _ in range(args.runs)]
        K, C, n_fft, block, lag = geo
        line = {"K": K, "C": C, "n_fft": n_fft, "block": block, "lag": lag, "slots": args.slots, "runs": args.runs,
                "state_bytes": runs[0][1], "formula_bytes": formula_bytes(K, C, n_fft, block, lag, runs[0][3]),
                "file_bytes": runs[0][2]}
        for k in ("export", "save", "load", "restore"):
            v = [r[0][k] for r in runs]
            line[k + "_ms"] = round(float(np.median(v)), 4)
            line[k + "_ms_min"] = round(min(v), 4)
            line[k + "_ms_max"] = round(max(v), 4)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
