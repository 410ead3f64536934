"""The instantiation table of tests/test_gpu_stft_instances.py covers exactly the fused-STFT kernels and the
partial-sum consumers the launchers dispatch to (the sets are parsed out of the CUDA sources), and the workspace the
ABI sizes holds every slot the segment contract of kernels.h writes, for every reserved-SM setting."""
import re

import pytest
import torch

import test_gpu_stft_instances as gpu
from test_kernel_instances_cpu import _function, _src

N_FFTS = (256, 512, 1024)


def _eval_c(expr, **env):
    """A C condition or integer expression of the launchers, in Python."""
    py = expr.replace("&&", " and ").replace("||", " or ").replace("/", "//").replace("true", "True")
    return eval(py, {}, env)


def _supported():
    """(n_fft, C, n_mask) for which `bool stft_scm_supported(int n_fft, int C, int n_mask)` holds."""
    body = _function(_src("stft_scm.cu"), "bool stft_scm_supported(")
    body = re.sub(r"//[^\n]*", "", body)
    py = ["def f(n_fft, C, n_mask):"]
    for stmt in (s.strip() for s in body.split(";") if s.strip()):
        stmt = stmt.replace("&&", " and ").replace("||", " or ").replace("true", "True").replace("false", "False")
        m = re.fullmatch(r"if\s*\((.*)\)\s*return\s+(.*)", stmt, re.S)
        if m:
            py.append("    if %s: return %s" % (m.group(1), m.group(2)))
        else:
            m = re.fullmatch(r"return\s+(.*)", stmt, re.S)
            assert m, "unexpected statement in stft_scm_supported: " + stmt
            py.append("    return " + m.group(1))
    ns = {}
    exec("\n".join(py), ns)
    return {(n, c, k) for n in (128, 256, 512, 1024, 2048) for c in range(0, 10) for k in range(-1, 4)
            if ns["f"](n, c, k)}


def _blocks(body):
    """[(condition or None, text)]: the `if constexpr (cond) { ... }` blocks of a launcher and the rest."""
    out, rest, i = [], "", 0
    for m in re.finditer(r"if constexpr \((.*?)\)\s*\{", body):
        if m.start() < i:
            continue
        rest += body[i:m.start()]
        depth, j = 0, m.end() - 1
        for j in range(m.end() - 1, len(body)):
            depth += {"{": 1, "}": -1}.get(body[j], 0)
            if depth == 0:
                break
        out.append((m.group(1), body[m.end():j]))
        i = j + 1
    out.append((None, rest + body[i:]))
    return out


def _compiled():
    """{(kind, n_fft, C)} of the stft_scm_kernel instantiations launch_stft_scm and launch_stft_filter_dual reach."""
    src = _src("stft_scm.cu")
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_c<(\d+)>", _function(src, "cudaError_t launch_stft_scm("))
    assert found and all(a == b for a, b in found)
    nffts = {int(a) for a, _ in found}
    cs = []                                 # (condition on N, C)
    for cond, text in _blocks(_function(src, "static cudaError_t launch_c(")):
        cs += [(cond, int(c)) for c, c2 in re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_nm<N,\s*(\d+)>", text)
               if c == c2]
    nms = []                                # (condition on N, C; nm, OUT)
    for cond, text in _blocks(_function(src, "static cudaError_t launch_nm(")):
        for stmt in re.findall(r"if \(nm == (\d)\) return (.*?);", text):
            nm, call = int(stmt[0]), stmt[1]
            outs = re.findall(r"launch_one<N,\s*C,\s*\d(?:,\s*(OUT_\w+))?>", call)
            assert outs, call
            for out in outs:
                nms.append((cond, nm, out or "OUT_Y"))
    kind = {(0, "OUT_Y"): "stft", (1, "OUT_Y"): "stft_scm", (2, "OUT_Y"): "stft_scm2", (2, "OUT_NONE"): "stft_scm2_none"}
    got = set()
    for n in nffts:
        for ccond, c in cs:
            if ccond and not _eval_c(ccond, N=n):
                continue
            for ncond, nm, out in nms:
                if ncond and not _eval_c(ncond, N=n, C=c):
                    continue
                got.add((kind[(nm, out)], n, c))
    for n, c in re.findall(r"DISCO_SFD\((\d+),\s*(\d+)\)", _function(src, "cudaError_t launch_stft_filter_dual(")):
        got.add(("stft_filter_dual", int(n), int(c)))
    return got, nffts


def _table():
    return {(k, n, c) for k in gpu.NM_OF for n, cs in gpu.INSTANCES[k].items() for c in cs}


def test_stft_scm_kernel_instances():
    got, nffts = _compiled()
    assert nffts == set(N_FFTS)
    assert _table() == got, _table() ^ got
    # what the ABI admits is what is compiled: every (n_fft, C, n_mask) the support predicate accepts has a kernel
    supported = _supported()
    assert supported == {(n, c, gpu.NM_OF[k]) for k, n, c in got}, supported ^ {(n, c, gpu.NM_OF[k]) for k, n, c in got}
    # the filter pass covers the two-mask set
    assert {(n, c) for k, n, c in got if k == "stft_filter_dual"} == {(n, c) for k, n, c in got if k == "stft_scm2"}


def test_plain_stft_row_is_disco_stft_grouping():
    """disco_stft groups its signals by min(4, n_sig): the n_mask = 0 row must be exactly C 1..4 at every n_fft."""
    body = _function(_src("api.cu"), "int disco_stft(")
    m = re.search(r"const int C = n_sig >= (\d+) \? (\d+) : n_sig;", body)
    assert m and m.group(1) == m.group(2)
    cmax = int(m.group(1))
    assert all(set(cs) == set(range(1, cmax + 1)) for cs in gpu.INSTANCES["stft"].values())
    assert set(gpu.INSTANCES["stft"]) == set(N_FFTS)


def test_consumer_instances():
    src = _src("stft_scm.cu")
    fin = {int(c) for c in re.findall(r"DISCO_FIN\((\d+)\)", _function(src, "cudaError_t launch_scm_finalize("))}
    assert set(gpu.INSTANCES["scm_finalize"]["C"]) == fin
    body = _function(_src("filter_dual.cu"), "cudaError_t launch_filter_dual(")
    cases = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_c<(\d+)>", body)
    assert cases and all(a == b for a, b in cases)
    assert set(gpu.INSTANCES["filter_dual"]["C"]) == {int(a) for a, _ in cases}
    # the workspace solve: D <= 4 (solve_workspace of api.cu), one or two mask sets
    sw = _function(_src("api.cu"), "static int solve_workspace(")
    m = re.search(r"C < 1 \|\| C > (\d+) \|\| n_set < 1 \|\| n_set > (\d+)", sw)
    assert m, "solve_workspace's argument check moved"
    assert set(gpu.INSTANCES["solve_workspace"]["C"]) == set(range(1, int(m.group(1)) + 1))
    assert set(gpu.INSTANCES["solve_workspace"]["n_set"]) == set(range(1, int(m.group(2)) + 1))


def test_tile_frames_matches_source():
    m = re.search(r"int stft_tile_frames\(int n_fft, int C\) \{ return (.*?); \}", _src("stft_scm.cu"))
    assert m
    for n in N_FFTS:
        for c in range(1, 9):
            assert gpu.tile_frames(n, c) == _eval_c(m.group(1), n_fft=n, C=c)


def test_geometry_cases_cover_every_class():
    """The shape list of the GPU geometry tests reaches every launch-geometry class for the CTA counts of every
    reserved setting (the device's SM count, or the library's fallback of 132 without a device)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    for r in (0, 16, 64):
        s = sms - r
        shapes = gpu.geometry_shapes(s)
        assert all(sh is not None for sh in shapes), s
        got = set().union(*(gpu.geometry_classes(g, tp, s) for g, tp in shapes))
        assert got == gpu.ALL_CLASSES, (s, gpu.ALL_CLASSES - got)


@pytest.fixture(scope="module")
def lib():
    from disco_b200 import build, _lib
    build.build()
    return _lib.load()


def test_workspace_holds_every_written_slot(lib):
    """disco_stft_scm_workspace / scm2_workspace over n_fft, C 1..8, group counts, lengths and reserved SMs: the slot
    count it sizes (bytes / (G n_mask 2 C^2 F 4)) is at least the largest n_slot of the segment contract, and the
    sweep contains cases where it is exactly that (the bound is tight)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    tight = {}
    try:
        for r in (0, 16, 64):
            assert lib.disco_set_reserved_sms(r) == 0
            s = sms - r
            tight[r] = 0
            for n_fft in N_FFTS:
                hop, F = n_fft // 2, n_fft // 2 + 1
                for C in range(1, 9):
                    tt = gpu.tile_frames(n_fft, C)
                    for tp in (1, 2, 3, 4, 5, 7, 13, 20, 33, 100):
                        for L in {tp * tt * hop - hop, (tp - 1) * tt * hop + 1 + hop}:
                            if L <= hop:
                                L = hop + 1
                            T = 1 + L // hop
                            tpl = -(-T // tt)
                            for G in (1, 2, 3, 5, 7, 13, 20, 33, 64, s - 1, s, s + 1, 3 * s + 1):
                                n_cta, _, _, n_slot = gpu.segments(G, tpl, s)
                                for nm, fn in ((1, lib.disco_stft_scm_workspace), (2, lib.disco_stft_scm2_workspace)):
                                    nbytes = fn(G, C, L, n_fft)
                                    per_slot = G * nm * 2 * C * C * F * 4
                                    assert nbytes % per_slot == 0
                                    spg = nbytes // per_slot
                                    assert spg >= n_slot.max(), (r, n_fft, C, G, L, spg, int(n_slot.max()))
                                    tight[r] += int(spg == n_slot.max())
    finally:
        assert lib.disco_set_reserved_sms(0) == 0
    assert all(v > 0 for v in tight.values()), tight
