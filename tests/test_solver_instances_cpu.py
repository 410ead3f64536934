"""The instantiation table and geometry mirror of tests/test_gpu_solver_instances.py match the solver sources: the
dispatch sets of `launch_mwf_solve` (solve.cu) and `launch_mwf_solve_small` (solve_small.cu), the `SolveGeom`
expressions for G and WARPS, and the 64-thread launch of solve_small.cu are parsed out of the CUDA sources, so a solver
instantiated later without a test, or a geometry change the tests do not follow, fails here, on CPU."""
import re

import test_gpu_solver_instances as gpu
from test_kernel_instances_cpu import _cases, _function, _src


def _geom_expr(src, name):
    m = re.search(r"static constexpr int %s = ([^;]+);" % name, _function(src, "struct SolveGeom"))
    assert m, name
    return m.group(1)


def test_solve_instances():
    src = _src("solve.cu")
    body = _function(src, "cudaError_t launch_mwf_solve(const SolveArgs& a, cudaStream_t st) {")
    assert set(gpu.INSTANCES["solve"]) == _cases(body, "launch_d")
    # everything below the cooperative solver's first D goes to solve_small.cu
    small_max = int(re.search(r"if \(a\.D <= (\d+)\) return launch_mwf_solve_small\(a, st\);", body).group(1))
    assert small_max == max(gpu.INSTANCES["solve_small"]) == min(gpu.INSTANCES["solve"]) - 1


def test_solve_small_instances():
    body = _function(_src("solve_small.cu"), "cudaError_t launch_mwf_solve_small(")
    assert set(gpu.INSTANCES["solve_small"]) == _cases(body, "small::launch_d")


def test_solve_geometry():
    src = _src("solve.cu")
    g_expr, w_expr = _geom_expr(src, "G"), _geom_expr(src, "WARPS")
    assert _geom_expr(src, "MPW") == "32 / G" and _geom_expr(src, "MPB").startswith("MPW * WARPS")
    assert "const int blocks = (a.n_mat + SG::MPB - 1) / SG::MPB;" in src
    # the expressions as they stand, restated below in Python: a change to either must be followed here
    assert g_expr == "D <= 2 ? 2 : (D <= 4 ? 4 : (D <= 8 ? 8 : 16))", g_expr
    assert w_expr == "D <= 8 ? 4 : 2", w_expr
    for D in gpu.INSTANCES["solve"]:
        G = 2 if D <= 2 else (4 if D <= 4 else (8 if D <= 8 else 16))
        warps = 4 if D <= 8 else 2
        assert gpu.geometry(D) == (G, 32 // G, warps, (32 // G) * warps), D
        assert D <= G, D


def test_solve_small_geometry():
    src = _src("solve_small.cu")
    launches = re.findall(r"<<<\(a\.n_mat \+ (\d+)\) / (\d+), (\d+), 0, st>>>", _function(src, "launch_d("))
    assert len(launches) == 2, launches
    for up, div, threads in launches:
        assert int(up) + 1 == int(div) == int(threads) == gpu.SMALL_THREADS
    assert re.search(r"__launch_bounds__\((\d+), MINB\)", src).group(1) == str(gpu.SMALL_THREADS)
    for D in gpu.INSTANCES["solve_small"]:
        assert gpu.geometry(D) == (1, 32, gpu.SMALL_THREADS // 32, gpu.SMALL_THREADS), D

