"""Build libdisco_b200.so (hand-written sm_90a CUDA kernels + C ABI) in-tree with nvcc.

    python -m disco_b200.build [-v] [--force]

nvcc cross-compiles without a GPU.  The shared library lands next to this file so that it
travels with the source tree to the GPU box; objects go to build/ (git-ignored).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(HERE, "libdisco_b200.so")
SOURCES = ["api.cu", "stft_scm.cu", "scm.cu", "scm_wide.cu", "solve.cu", "solve_small.cu", "filter_sum.cu", "filter_sum_multi.cu", "filter_dual.cu", "mid_multi.cu", "istft.cu", "filterbank.cu", "online.cu", "online_wide.cu", "misc.cu", "stream.cu", "bss.cu", "stoi.cu", "lengths.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _deps_mtime():
    newest = 0.0
    for dirpath in (CSRC, os.path.join(ROOT, "include")):
        for fn in os.listdir(dirpath):
            if fn.endswith((".cuh", ".h")):
                newest = max(newest, os.path.getmtime(os.path.join(dirpath, fn)))
    return newest


def build(verbose=False, force=False, defines=(), lib=LIB, obj=OBJ):
    """defines: extra -D macros (a measurement variant such as DISCO_ROLE_CLOCKS); such a variant goes to its own
    lib and obj directory so that it never replaces the in-tree library."""
    os.makedirs(obj, exist_ok=True)
    hdr = _deps_mtime()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(obj, src.replace(".cu", ".o"))
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr):
            cmd = ([NVCC] + FLAGS + ["-D" + d for d in defines] + (["-Xptxas", "-v"] if verbose else []) +
                   ["-c", s, "-o", o])
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for cmd, r in ex.map(run, jobs):
            if verbose or r.returncode != 0:
                sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr + "\n")
            if r.returncode != 0:
                raise RuntimeError("nvcc failed for %s" % cmd[-3])
    objs = [os.path.join(obj, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or not os.path.exists(lib):
        cmd = [NVCC, "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return lib


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="--force" in sys.argv))
