"""The dispatch sets and launch-plan constants that tests/test_gpu_post_instances.py mirrors, parsed out of the CUDA
sources: a retuned launcher fails here, on CPU, instead of quietly moving the GPU cases off their plan edges."""
import re

import test_gpu_post_instances as gpu
from test_kernel_instances_cpu import _function, _src


def _int_const(src, pattern):
    m = re.search(pattern, src)
    assert m, pattern
    return int(m.group(1))


def test_istft_dispatch_set():
    body = _function(_src("istft.cu"), "cudaError_t launch_istft(")
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_n<(\d+)>", body)
    assert found and all(a == b for a, b in found)
    assert {int(a) for a, _ in found} == set(gpu.ISTFT_NFFTS)


def test_istft_plan_constants():
    src = _src("istft.cu")
    assert _int_const(src, r"static constexpr int ITEMS = (\d+);") == gpu.ISTFT_ITEMS
    plan = _function(src, "static cudaError_t launch_n(")
    # the doubling rule and the rounding of fpc, as istft_plan restates them
    m = re.search(r"while \(pairs \* chunks < sm_count\(\) \* (\d+) && \(T_eff \+ chunks - 1\) / chunks > (\d+) \* G::ITEMS\)"
                  r" chunks \*= 2;", plan)
    assert m, "launch_n's chunk doubling changed"
    assert int(m.group(1)) == gpu.ISTFT_CTAS_PER_SM and int(m.group(2)) == gpu.ISTFT_MIN_TILES
    assert "a.j_end = min(a.j_end, (a.L + N + H - 1) / H);" in plan
    assert "a.fpc = ((T_eff + chunks - 1) / chunks + G::ITEMS - 1) / G::ITEMS * G::ITEMS;" in plan
    assert "chunks = (T_eff + a.fpc - 1) / a.fpc;" in plan


def test_band_stats_dispatch_set():
    body = _function(_src("filterbank.cu"), "cudaError_t launch_band_stats(")
    found = re.findall(r"case\s+(\d+)\s*:\s*band_stats_kernel<(\d+)>", body)
    assert found and all(int(nc) == int(order) + 1 for order, nc in found)
    assert {int(o) for o, _ in found} == set(gpu.BANK_ORDERS)


def test_band_stats_plan_constants():
    src = _src("filterbank.cu")
    assert _int_const(src, r"constexpr int kBankChunk = (\d+);") == gpu.BANK_CHUNK
    assert _int_const(src, r"constexpr int kBankWarps = (\d+);") == gpu.BANK_WARPS
    body = _function(src, "cudaError_t launch_band_stats(")
    assert "int bands_per_cta = a.n_band < kBankWarps ? a.n_band : kBankWarps;" in body
    assert ("while (bands_per_cta > 1 && sig_blocks * ((a.n_band + bands_per_cta - 1) / bands_per_cta) < sm_count()) "
            "--bands_per_cta;") in body


def test_plan_mirrors_cover_their_edges():
    """At the H100's 132 SMs the mirrored plans reach every class the GPU cases are chosen for."""
    for n_fft in gpu.ISTFT_NFFTS:
        labels = [c[0] for c in gpu.istft_plan_cases(n_fft, 132)]
        assert len(labels) == 5
    assert set(gpu.bank_geometries(132)) == set(range(1, gpu.BANK_WARPS + 1))
    assert gpu.istft_plan(3, 8193, 8192 * 128, 256, 132)[1] == 256
