"""Compare the machine code of the kernels of one CUDA source at two git revisions, function by function.

    python scripts/sass_diff.py disco_b200/csrc/stream.cu [--rev HEAD]

Compiles the source as it stands in the working tree and as it was at `rev` with the flags of disco_b200/build.py
(no GPU needed), then compares `cuobjdump -sass` of every function both objects define: instruction text only, with
the offsets, the encodings and the file-name header left out.  Prints one line per function (same / DIFF n lines,
new, removed) and exits 1 if a common function differs."""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from disco_b200 import build  # noqa: E402

CUOBJDUMP = os.path.join(os.path.dirname(build.NVCC), "cuobjdump")


def sass(obj):
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            # a function in an anonymous namespace carries a hash of the source's path, which differs between the trees
            cur = funcs.setdefault(re.sub(r"_GLOBAL__N__[0-9a-f]+_", "_GLOBAL__N__", m.group(1)), [])
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", line)
        if cur is not None and m:
            cur.append(" ".join(m.group(1).split()))
    return funcs


def compile_obj(src_dir, rel, out):
    subprocess.run([build.NVCC] + build.FLAGS + ["-c", os.path.join(src_dir, rel), "-o", out], check=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("source", help="path of the .cu file, relative to the repository root")
    ap.add_argument("--rev", default="HEAD")
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        old_tree = os.path.join(tmp, "old")
        os.makedirs(old_tree)
        tar = subprocess.run(["git", "-C", ROOT, "archive", args.rev, "disco_b200/csrc", "include"],
                             capture_output=True, check=True).stdout
        subprocess.run(["tar", "-x", "-C", old_tree], input=tar, check=True)
        compile_obj(old_tree, args.source, os.path.join(tmp, "old.o"))
        compile_obj(ROOT, args.source, os.path.join(tmp, "new.o"))
        old, new = sass(os.path.join(tmp, "old.o")), sass(os.path.join(tmp, "new.o"))
    bad = 0
    for name in sorted(set(old) | set(new)):
        if name not in new:
            print("removed", name)
        elif name not in old:
            print("new    ", name)
        elif old[name] == new[name]:
            print("same   ", name, "(%d instructions)" % len(old[name]))
        else:
            n = sum(a != b for a, b in zip(old[name], new[name])) + abs(len(old[name]) - len(new[name]))
            print("DIFF   ", name, "(%d lines)" % n)
            bad += 1
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
