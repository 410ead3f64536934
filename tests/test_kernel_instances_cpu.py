"""The instantiation table of tests/test_gpu_kernel_instances.py covers exactly the kernels the launchers dispatch to:
the sets are parsed out of the CUDA sources, so a kernel instantiated later without a test fails here, on CPU."""
import os
import re

import test_gpu_kernel_instances as gpu

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "disco_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as fh:
        return fh.read()


def _function(src, signature):
    """Body of the function whose definition starts with `signature` (up to the matching brace)."""
    start = src.index(signature)
    i = src.index("{", start)
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i + 1:j]
    raise ValueError("unbalanced braces after " + signature)


def _cases(body, launcher):
    """The D of every `case D: return launcher<D>(...)` in a switch."""
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+%s<(\d+)>" % re.escape(launcher), body)
    assert found and all(a == b for a, b in found), launcher
    return {int(a) for a, _ in found}


def _supported_pairs(body):
    """Evaluate the body of `bool tango_mid_supported(int C, int K)` -- `if (cond) return expr;` lines and a final
    `return expr;` -- for every C, K in 1..16."""
    py = ["def f(C, K):"]
    for stmt in (s.strip() for s in body.split(";") if s.strip()):
        stmt = stmt.replace("&&", " and ").replace("||", " or ").replace("true", "True").replace("false", "False")
        m = re.fullmatch(r"if\s*\((.*)\)\s*return\s+(.*)", stmt, re.S)
        if m:
            py.append("    if %s: return %s" % (m.group(1), m.group(2)))
        else:
            m = re.fullmatch(r"return\s+(.*)", stmt, re.S)
            assert m, "unexpected statement in tango_mid_supported: " + stmt
            py.append("    return " + m.group(1))
    ns = {}
    exec("\n".join(py), ns)
    return {(c, k) for c in range(1, 17) for k in range(1, 17) if ns["f"](c, k)}


def test_masked_scm_instances():
    body = _function(_src("scm.cu"), "cudaError_t launch_masked_scm(")
    assert set(gpu.INSTANCES["masked_scm"]["D"]) == _cases(body, "launch_d")
    # the fused z (W1 given) exists at every D of scm.cu
    assert "if (a.W1 != nullptr) return launch_dz<D, true>(a, st);" in _src("scm.cu")
    assert set(gpu.INSTANCES["masked_scm"]["zf_D"]) == _cases(body, "launch_d")


def test_masked_scm_wide_instances():
    src = _src("scm_wide.cu")
    wide = _cases(_function(src, "cudaError_t launch_masked_scm_wide("), "launch_wide_d")
    assert set(gpu.INSTANCES["masked_scm_wide"]["D"]) == wide
    zf_max = int(re.search(r"if \(D > (\d+)\) return cudaErrorInvalidValue;", _function(src, "launch_wide_d(")).group(1))
    assert set(gpu.INSTANCES["masked_scm_wide"]["zf_D"]) == {d for d in wide if d <= zf_max}


def test_filter_sum_instances():
    body = _function(_src("filter_sum.cu"), "cudaError_t launch_filter_sum(")
    assert set(gpu.INSTANCES["filter_sum"]["D"]) == _cases(body, "launch_d")


def test_online_instances():
    src = _src("online.cu")
    assert set(gpu.INSTANCES["online"]["D"]) == _cases(_function(src, "cudaError_t launch_scm_recursive("),
                                                       "launch_blocks_d")
    assert set(gpu.INSTANCES["online"]["D"]) == _cases(_function(src, "cudaError_t launch_filter_sum_blocks("),
                                                       "launch_filter_d")


def test_filter_sum_multi_instances():
    body = _function(_src("filter_sum_multi.cu"), "cudaError_t launch_filter_sum_multi(")
    pairs = {(int(c), int(k)) for c, k in re.findall(r"FSM_CASE\((\d+),\s*(\d+)\)", body)}
    assert pairs and set(gpu.INSTANCES["filter_sum_multi"]["CK"]) == pairs


def test_tango_mid_instances():
    src = _src("mid_multi.cu")
    supported = _supported_pairs(_function(src, "bool tango_mid_supported("))
    assert set(gpu.INSTANCES["tango_mid"]["CK"]) == supported
    launched = {(int(c), int(k)) for c, k in
                re.findall(r"MID_CASE\((\d+),\s*(\d+)\)", _function(src, "cudaError_t launch_tango_mid("))}
    assert launched == supported
