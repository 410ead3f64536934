"""The dispatch sets and launch-plan constants that tests/test_gpu_lengths_instances.py and
tests/test_gpu_stoi_instances.py mirror, parsed out of the CUDA sources: a retuned launcher fails here, on CPU,
instead of quietly moving the GPU cases off their plan edges.  The case generators are checked here too: at the
H100's 132 SMs every labelled case lands on its edge."""
import re

import test_gpu_lengths_instances as glen
import test_gpu_stoi_instances as gstoi
from test_kernel_instances_cpu import _function, _src
from test_post_instances_cpu import _int_const


def test_length_kernels_dispatch_sets():
    src = _src("lengths.cu")
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+launch_stft_lengths_n<(\d+)>",
                       _function(src, "cudaError_t launch_stft_lengths("))
    assert found and all(a == b for a, b in found)
    assert {int(a) for a, _ in found} == set(glen.LEN_NFFTS)
    found = re.findall(r"case\s+(\d+)\s*:\s*return\s+\{\(const void\*\)istft_lengths_kernel<(\d+)>",
                       _function(_src("istft.cu"), "IstftLengthsKernel istft_lengths_kernel_for("))
    assert found and all(a == b for a, b in found)
    assert {int(a) for a, _ in found} == set(glen.LEN_NFFTS)


def test_stft_lengths_plan_constants():
    src = _src("lengths.cu")
    assert _int_const(src, r"constexpr int kLenWarps = (\d+);") == glen.LEN_WARPS
    core = _src("stft_core.cuh")
    ra = _int_const(core, r"static constexpr int RA = N / (\d+);")
    nb = _int_const(core, r"static constexpr int NB = (\d+) / RA;")
    assert {n: nb // (n // ra) for n in glen.LEN_NFFTS} == glen.JOB_NB
    plan = _function(src, "static cudaError_t launch_stft_lengths_n(")
    assert "const int per_cta = kLenWarps * StftJob<N>::NB;" in plan
    assert "const int cols = (a.T + per_cta - 1) / per_cta;" in plan
    assert "for (int p0 = 0; p0 < pairs; p0 += kMaxGridYZ) {" in plan
    assert "b.lengths = a.lengths + s0;" in plan
    assert "stft_lengths_kernel<N><<<dim3(cols, (b.n_sig + 1) / 2), 32 * kLenWarps, 0, st>>>(b);" in plan
    assert _int_const(_src("kernels.h"), r"constexpr int kMaxGridYZ = (\d+);") == glen.GRID_YZ


def test_istft_lengths_plan_constants():
    """launch_istft_lengths' chunk plan is disco_istft's (test_gpu_post_instances.istft_plan) for the longest row."""
    import test_gpu_post_instances as post
    plan = _function(_src("lengths.cu"), "cudaError_t launch_istft_lengths(")
    assert "a.j_end = min(a.j_end, (a.L + n_fft + H - 1) / H);" in plan
    m = re.search(r"while \(pairs \* chunks < sm_count\(\) \* (\d+) && \(T_eff \+ chunks - 1\) / chunks > (\d+) \* k\.items\)"
                  r" chunks \*= 2;", plan)
    assert m, "launch_istft_lengths' chunk doubling changed"
    assert int(m.group(1)) == post.ISTFT_CTAS_PER_SM and int(m.group(2)) == post.ISTFT_MIN_TILES
    assert "a.fpc = ((T_eff + chunks - 1) / chunks + k.items - 1) / k.items * k.items;" in plan
    assert "chunks = (T_eff + a.fpc - 1) / a.fpc;" in plan
    assert "const int* len = lengths + s0;" in plan
    # k.items is IGeom<N>::ITEMS for every n_fft
    assert _int_const(_src("istft.cu"), r"static constexpr int ITEMS = (\d+);") == post.ISTFT_ITEMS
    body = _function(_src("istft.cu"), "IstftLengthsKernel istft_lengths_kernel_for(")
    assert len(re.findall(r"IGeom<(\d+)>::ITEMS", body)) == len(glen.LEN_NFFTS)
    # a CTA past a signal's frames returns; the chunk owning block j_end writes the tail
    kern = _function(_src("istft.cu"), "__global__ void __launch_bounds__(IGeom<N>::THREADS) istft_lengths_kernel(")
    assert "q.j_end = min(p.j_end, 1 + len / H);" in kern
    assert "if ((int)blockIdx.x * p.fpc >= q.j_end) return;" in kern


def test_stoi_plan_constants():
    src = _src("stoi.cu")
    hdr = _src("kernels.h")
    assert _int_const(src, r"constexpr int kSelThreads = (\d+);") == gstoi.SEL_THREADS
    assert _int_const(src, r"constexpr int kBandWarps = (\d+);") == gstoi.BAND_WARPS
    assert _int_const(src, r"constexpr int kScoreThreads = (\d+);") == gstoi.SCORE_THREADS
    assert _int_const(hdr, r"constexpr int kStoiSeg = (\d+);") == gstoi.STOI_SEG
    assert _int_const(hdr, r"constexpr int kStoiBands = (\d+);") == gstoi.STOI_BANDS
    assert _int_const(hdr, r"constexpr int kStoiFrame = (\d+);") == gstoi.STOI_FRAME
    assert "constexpr int kHop = kStoiFrame / 2;" in src
    assert "return L < kStoiFrame ? 0 : (L - kStoiFrame) / kHop + 1;" in src
    launch = _function(src, "cudaError_t launch_stoi(")
    # the workspace layout stoi_run reads the intermediates with
    for line in ("a.n_fr = stoi_n_fr(a.L);",
                 "a.tob = a.energy + (size_t)a.n_clean * a.n_fr;",
                 "a.sel = (int*)(a.tob + ((size_t)a.n_clean + a.n_pair) * a.n_fr * kStoiBands);",
                 "const int groups = (a.n_fr - 1 + kBandWarps - 1) / kBandWarps;",
                 "stoi_select_kernel<<<a.n_clean, kSelThreads, 0, st>>>(a);",
                 "stoi_score_kernel<<<a.n_pair, kScoreThreads, 0, st>>>(a);"):
        assert line in launch, line
    ws = _function(src, "size_t stoi_ws_bytes(")
    assert "return n_fr * ((size_t)n_clean * (sizeof(double) + sizeof(int)) +" in ws
    assert "((size_t)n_clean + n_pair) * kStoiBands * sizeof(double));" in ws
    for C, P, L in ((1, 1, 256), (3, 8, 65792), (11, 21, 30000)):
        n_fr, e_off, tob_off, sel_off, total = gstoi.ws_layout(C, P, L)
        assert total == n_fr * (C * 12 + (C + P) * 15 * 8)
    # the scan's pass and the score loop's stride are the thread counts
    sel = _function(src, "__global__ void __launch_bounds__(kSelThreads) stoi_select_kernel(")
    assert "for (int f0 = 0; f0 < n_fr; f0 += kSelThreads) {" in sel
    score = _function(src, "__global__ void __launch_bounds__(kScoreThreads) stoi_score_kernel(")
    assert "for (int it = tid; it < J * kStoiBands; it += kScoreThreads) {" in score
    bands = _function(src, "__global__ void __launch_bounds__(kBandWarps * 32) stoi_bands_kernel(")
    assert "const int t = (blockIdx.x % groups) * kBandWarps + warp;" in bands
    assert "if (t >= ns - 1) return;" in bands


def test_case_generators_reach_their_edges():
    """At 132 SMs (the H100 SXM) every labelled case of the GPU files lands where its label says."""
    for n_fft in glen.LEN_NFFTS:
        cases = glen.stft_cases(n_fft)
        assert len(cases) == 3
        labels = set(l for _, _, ls in cases for l in ls)
        assert {"H+1", "H+2", "N-1", "N", "N+1", "kH-1", "kH", "kH+1", "L_max", "partner_ends_before_reflect",
                "Tb=2pc-1", "Tb=2pc", "Tb=2pc+1", "lone_last"} == labels
        assert [c[0] for c in glen.istft_plan_cases(n_fft, 132)] == ["one_chunk", "many_chunks", "y_frames_short"]
    lengths = glen.beyond_grid_lengths(2 * glen.GRID_YZ + 3, 128, 600)
    assert len(lengths) == 2 * glen.GRID_YZ + 3
    gstoi.check_select_labels(gstoi.select_cases())
    gstoi.check_band_score_labels(gstoi.BAND_SCORE_NSEL)
    for fs in (8000, 16000, 22050, 44100, 48000):
        gstoi.resample_lengths(fs)
