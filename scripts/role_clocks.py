"""Where the warp roles of the fused STFT+SCM kernel spend their cycles: busy, or waiting on which mbarrier.

    python scripts/role_clocks.py [--build] [what ...]

Builds the library with -DDISCO_ROLE_CLOCKS into build/role_clocks/ (once; --build rebuilds), loads it in place of
the in-tree library (DISCO_B200_LIB), runs each kernel once to warm up and once measured, and prints per role (loader,
FFT warps, SCM / filter consumer warps) the share of its cycles spent working and waiting on samp_full, samp_empty,
spec_full and spec_empty, averaged over the warps of that role in every CTA.

what: stft_scm2_noY (<512,4,2,OUT_NONE>, 64 x 4 mics x 10 s; the default) | stft_scm2 (<512,4,2>) |
      stft_scm1 (<512,4,1>) | stft_filter_dual (<512,4,0,OUT_FILTER>) | stft_scm_c8 (<512,8,1>, 128 x 8 mics) | all
"""
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from disco_b200 import build as _build  # noqa: E402

VARIANT = os.path.join(ROOT, "build", "role_clocks")
LIB = os.path.join(VARIANT, "libdisco_b200.so")
ROLES = {1: "loader", 2: "fft", 3: "consumer"}
WAITS = ("samp_full", "samp_empty", "spec_full", "spec_empty")
TARGETS = ("stft_scm2_noY", "stft_scm2", "stft_scm1", "stft_filter_dual", "stft_scm_c8")


def table(buf):
    """buf: uint64 [max CTAs, 32 warps, slots] (disco_role_clocks_layout)
    -> rows of (role, warps, tiles/warp, jobs/warp, cycles, busy, waits)."""
    rows = []
    n_cta = int((buf[:, :, 0] != 0).any(axis=1).sum())
    for code, name in ROLES.items():
        sel = buf[buf[:, :, 0] == code].astype(np.float64)
        if not len(sel):
            continue
        total = sel[:, 3].sum()
        waits = sel[:, 4:8].sum(axis=0) / total
        rows.append((name, len(sel) / max(n_cta, 1), sel[:, 1].mean(), sel[:, 2].mean(), sel[:, 3].mean(),
                     1.0 - waits.sum(), waits))
    return n_cta, rows


def main(argv):
    force = "--build" in argv
    what = [a for a in argv if not a.startswith("--")] or ["stft_scm2_noY"]
    if what == ["all"]:
        what = list(TARGETS)
    if force or not os.path.exists(LIB):
        _build.build(force=force, defines=("DISCO_ROLE_CLOCKS",), lib=LIB, obj=os.path.join(VARIANT, "obj"))
    os.environ["DISCO_B200_LIB"] = LIB
    import torch
    from disco_b200 import _lib, ops

    lib = _lib.load()
    lib.disco_role_clocks.restype = ctypes.c_longlong
    lib.disco_role_clocks.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    lib.disco_role_clocks_layout.restype = None
    lib.disco_role_clocks_layout.argtypes = [ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    max_ctas, slots = ctypes.c_int(), ctypes.c_int()
    lib.disco_role_clocks_layout(ctypes.byref(max_ctas), ctypes.byref(slots))
    if slots.value != 8:
        raise RuntimeError("role-clock slots: the library records %d per warp, this script reads 8" % slots.value)
    buf = np.zeros((max_ctas.value, 32, slots.value), np.uint64)

    def read(reset):
        n = lib.disco_role_clocks(buf.ctypes.data, buf.nbytes, reset)
        if n < 0:
            raise RuntimeError("disco_role_clocks: CUDA error")
        if n != buf.nbytes:
            raise RuntimeError("disco_role_clocks copied %d bytes, the layout has %d" % (n, buf.nbytes))

    dev = torch.device("cuda:0")
    print(torch.cuda.get_device_name(dev))
    g = torch.Generator().manual_seed(0)
    L = 160000
    T, F = 1 + L // 256, 257
    rnd = lambda *s: torch.rand(s, generator=g).to(dev)
    cplx = lambda *s: torch.complex(torch.randn(s, generator=g), torch.randn(s, generator=g)).to(dev)
    ops.init(512)
    x4 = torch.randn((64, 4, L), generator=g).to(dev)
    m, m2 = rnd(64, T, F), rnd(64, T, F)
    runs = {
        "stft_scm2_noY": ("stft_scm_kernel<512,4,2,OUT_NONE>", lambda: ops.stft_scm2(x4, m, m2, want_Y=False)),
        "stft_scm2": ("stft_scm_kernel<512,4,2,OUT_Y>", lambda: ops.stft_scm2(x4, m, m2)),
        "stft_scm1": ("stft_scm_kernel<512,4,1,OUT_Y>", lambda: ops.stft_scm(x4, m, keep_partials=True)),
        "stft_filter_dual": ("stft_scm_kernel<512,4,0,OUT_FILTER>",
                             lambda: ops.stft_filter_dual(x4, cplx(64, F, 4), cplx(64, F, 4))),
    }
    if "stft_scm_c8" in what:
        x8, m8 = torch.randn((128, 8, L), generator=g).to(dev), rnd(128, T, F)
        runs["stft_scm_c8"] = ("stft_scm_kernel<512,8,1,OUT_Y>", lambda: ops.stft_scm(x8, m8, keep_partials=True))
    for w in what:
        name, fn = runs[w]
        fn()
        read(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        read(1)
        n_cta, rows = table(buf)
        print("\n%s (%s): %d CTAs, call %.1f us (instrumented)" % (name, w, n_cta, e0.elapsed_time(e1) * 1e3))
        print("%-9s %5s %7s %6s %9s %6s %s" % ("role", "warps", "tiles", "jobs", "cycles", "busy",
                                               " ".join("%10s" % k for k in WAITS)))
        for role, warps, tiles, jobs, cyc, busy, waits in rows:
            print("%-9s %5.0f %7.1f %6.1f %9.0f %6.3f %s" % (role, warps, tiles, jobs, cyc, busy,
                                                            " ".join("%10.3f" % v for v in waits)))


if __name__ == "__main__":
    main(sys.argv[1:])
