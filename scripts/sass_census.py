"""Static instruction census of the fused STFT kernel's roles: which warp role each SASS instruction belongs to, and
what kind of work it is.

    python scripts/sass_census.py [--obj build/obj/stft_scm.o] [--src stft_scm.cu] [--lines N] [kernel ...]

kernel: <N,C,NM,OUT> template arguments as in stft_scm.cu, e.g. 512,4,2,1 (the two-mask statistics pass without Y,
the default set also has 512,4,0,2 (filter pass), 512,4,2,0 and 512,4,1,0).  --obj: another build's object, with
--src the stft_scm.cu it was compiled from.  The instructions of the roles must add up to the function's: the
script stops if they do not.

Disassembles the kernels of the object (nvdisasm -gi, line info of -lineinfo builds; no GPU needed) and attributes
each instruction to the line of stft_scm_kernel it was inlined into.  The role is the branch of the kernel that line
lies in (setup, loader + Nyquist bin, FFT warps, SCM / filter consumer warps); the kind is
    fp32   FFMA FADD FMUL (and their two-lane forms, on architectures that have them)
    smem   LDS STS (and shared-memory atomics / barriers on mbarriers: SYNCS)
    gmem   LDG STG LDC and TMA copies
    int    IADD3 IMAD LEA SHF LOP3 ISETP SEL IABS PRMT ... and their uniform-datapath forms
    move   MOV UMOV S2R S2UR R2UR CS2R ...
    ctrl   BRA BSSY BSYNC EXIT CALL RET WARPSYNC NOP and predicate logic
    bar    BAR (named barriers)
With --lines N it also prints the N source lines with the most non-fp32 instructions per role: where the address
arithmetic, moves and branches are.  The counts are static (instructions in the code), not issued instructions: each
fully unrolled loop appears once per unrolled trip, a run-time loop body once.
"""
import argparse
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from disco_b200 import build  # noqa: E402

BIN = os.path.dirname(build.NVCC)
SRC = os.path.join(ROOT, "disco_b200", "csrc", "stft_scm.cu")
KINDS = ("fp32", "smem", "gmem", "int", "move", "ctrl", "bar", "other")
DEFAULT = ("512,4,2,1", "512,4,0,2", "512,4,2,0", "512,4,1,0")


def kind(op):
    base = op.split(".")[0]
    b = base[1:] if base.startswith("U") and base not in ("UMOV",) else base
    if b in ("FFMA", "FADD", "FMUL", "FMUL2", "FFMA2", "FADD2"):
        return "fp32"
    if b in ("FMNMX", "HFMA2", "FSEL", "FSETP"):
        return "move" if b == "HFMA2" else "int"
    if b in ("LDS", "STS", "LDSM", "ATOMS", "SYNCS"):
        return "smem"
    if b in ("LDG", "STG", "LDC", "LDL", "STL", "UBLKCP", "BLKCP", "UTMALDG", "LD", "ST", "RED", "ATOMG"):
        return "gmem"
    if b in ("BAR",):
        return "bar"
    if b in ("MOV", "UMOV", "S2R", "S2UR", "R2UR", "CS2R", "SHFL", "MOV32I", "F2I", "I2F"):
        return "move"
    if b in ("BRA", "BSSY", "BSYNC", "EXIT", "CALL", "RET", "WARPSYNC", "NOP", "PLOP3", "VOTE", "VOTEU", "ELECT",
             "BREAK", "YIELD", "SETMAXREG", "USETMAXREG", "ACQBULK", "JMP", "BMOV", "ARRIVES"):
        return "ctrl"
    if b in ("IADD3", "IMAD", "LEA", "SHF", "LOP3", "ISETP", "SEL", "IABS", "PRMT", "IMNMX", "POPC", "FLO", "BREV",
             "LEA_HI", "IDP", "IADD", "SGXT", "BMSK", "IMUL", "ISCADD", "P2R", "R2P", "FCHK", "MUFU"):
        return "int"
    return "other"


def kernel_roles(src):
    """(first, last) line of each role's branch in stft_scm_kernel, found from the role banners of the source."""
    lines = open(src).read().splitlines()
    at = lambda pat: next(i + 1 for i, l in enumerate(lines) if re.search(pat, l))
    k0 = at(r"stft_scm_kernel\(typename")
    ld, ff, sc = at(r"=+ LOADER"), at(r"=+ FFT warps"), at(r"=+ SCM warps")
    k1 = next(i + 1 for i in range(sc, len(lines)) if lines[i].startswith("}"))
    return k0, [("loader", ld - 2, ff - 3), ("fft", ff - 2, sc - 3), ("consumer", sc - 2, k1)]


def census(obj, names, src=SRC):
    """-> {function: {role: Counter(kind -> count, ("line", line, kind) -> count)}, plus "_all": Counter("n")}"""
    obj = os.path.abspath(obj)
    with tempfile.TemporaryDirectory() as tmp:
        subprocess.run([os.path.join(BIN, "cuobjdump"), "-xelf", "all", obj], cwd=tmp, check=True, capture_output=True)
        cubin = next(os.path.join(tmp, f) for f in os.listdir(tmp) if f.endswith(".cubin") and "sm_90" in f)
        text = subprocess.run([os.path.join(BIN, "nvdisasm"), "-gi", "-c", cubin], capture_output=True, text=True,
                              check=True).stdout
    k0, roles = kernel_roles(src)
    out = {}
    fn, loc = None, None
    for line in text.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", line)
        if m:
            fn = m.group(1) if m.group(1) in names else None
            loc = None
            if fn:
                out[fn] = collections.defaultdict(collections.Counter)
            continue
        if line.startswith("//---"):   # the banner of the next section
            fn = None
        if fn is None:
            continue
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)(.*)', line)
        if m:
            # the outermost frame of the chain is the kernel line everything else was inlined into
            chain = re.findall(r'"([^"]+)", line (\d+)', line)
            f, ln = chain[-1]
            loc = int(ln) if f.endswith("stft_scm.cu") else None
            continue
        if re.match(r"\s+/\*[0-9a-f]{4,}\*/", line):
            out[fn]["_all"]["n"] += 1   # every instruction line, whatever its form: the check of the roles' sum
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m:
            role = "setup"
            if loc is not None:
                for name, a, b in roles:
                    if a <= loc <= b:
                        role = name
            k = kind(m.group(2))
            out[fn][role][k] += 1
            out[fn][role][("line", loc, k)] += 1
    return out


def mangled(spec):
    n, c, nm, o = (int(v) for v in spec.split(","))
    return "_ZN5disco15stft_scm_kernelILi%dELi%dELi%dELi%dEEEvNS_9StftParamIXT2_EE4typeE" % (n, c, nm, o)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("kernels", nargs="*", default=list(DEFAULT))
    ap.add_argument("--obj", default=os.path.join(build.OBJ, "stft_scm.o"))
    ap.add_argument("--src", default=SRC, help="the stft_scm.cu the object was compiled from (its line numbers)")
    ap.add_argument("--lines", type=int, default=0)
    args = ap.parse_args()
    names = {mangled(k): k for k in args.kernels}
    res = census(args.obj, set(names), args.src)
    for fn, spec in names.items():
        if fn not in res:
            print("stft_scm<%s>: not in %s" % (spec, args.obj))
            continue
        roles_sum = sum(res[fn][r][k] for r in ("setup", "loader", "fft", "consumer") for k in KINDS)
        if roles_sum != res[fn]["_all"]["n"]:
            raise SystemExit("stft_scm<%s>: the roles hold %d instructions, the function %d" %
                             (spec, roles_sum, res[fn]["_all"]["n"]))
        print("stft_scm<%s>: %d instructions" % (spec, roles_sum))
        print("  %-9s" % "role" + "".join("%7s" % k for k in KINDS) + "%8s" % "total")
        for role in ("setup", "loader", "fft", "consumer"):
            c = res[fn][role]
            tot = sum(c[k] for k in KINDS)
            print("  %-9s" % role + "".join("%7d" % c[k] for k in KINDS) + "%8d" % tot)
        if args.lines:
            for role in ("fft", "consumer"):
                c = res[fn][role]
                per = collections.Counter()
                for key, v in c.items():
                    if isinstance(key, tuple) and key[2] not in ("fp32", "smem"):
                        per[key[1]] += v
                src = open(args.src).read().splitlines()
                for ln, v in per.most_common(args.lines):
                    text = src[ln - 1].strip()[:80] if ln else "?"
                    print("    %-8s line %4s: %4d  %s" % (role, ln, v, text))


if __name__ == "__main__":
    main()
