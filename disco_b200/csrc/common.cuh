// Shared device helpers for the disco_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define DISCO_DEV __device__ __forceinline__

namespace disco {

// ---------------------------------------------------------------- two-lane float arithmetic
// Hopper has no packed FP32 instructions: each helper is one correctly rounded scalar operation per half
// (the _rn intrinsics are never contracted into an FMA), so every result below is fixed to the bit.
DISCO_DEV float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
DISCO_DEV float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
DISCO_DEV float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---------------------------------------------------------------- per-bin solve
// 2^-e for t in [2^e, 2^(e+1)); 1 when t is 0, subnormal, inf or NaN.  The MWF solvers multiply Rss and Rnn by
// it, with t = max(sum |diag Rss| + sum |diag Rnn|, max |Re, Im of any entry|) (the sum for PSD input; the
// maximum covers indefinite input such as an Rss with a zero diagonal), so every bin is solved in the same
// binade whatever the units of the input: the product is exact, every filter they compute is invariant under a
// common scale, and inputs that differ by a power of two give bit-identical filters.  It also puts the absolute 1e-300 of the Cholesky pivot
// floor at a fixed distance below the data, which keeps singular bins (Rnn == 0) finite at any input scale.
DISCO_DEV double solve_scale(double t) {
    if (!(t >= 2.2250738585072014e-308 && t <= 1.7976931348623157e308)) return 1.0;
    const int e = ((__double2hiint(t) >> 20) & 0x7ff) - 1023;
    return __hiloint2double((1023 - e) << 20, 0);
}

// ---------------------------------------------------------------- complex helpers (float2)
DISCO_DEV float2 cadd(float2 a, float2 b) { return fadd2(a, b); }
DISCO_DEV float2 csub(float2 a, float2 b) { return fadd2(a, make_float2(-b.x, -b.y)); }
// Complex products: one fmul2 + one ffma2 each (two FMUL + two FFMA); the half swaps and sign flips
// are free operand modifiers.
// Rounding: re = fma(a.x, b.x, -(a.y b.y)), im = fma(a.x, b.y, a.y b.x).
DISCO_DEV float2 cmul(float2 a, float2 b) {
    const float2 t = fmul2(make_float2(-b.y, b.x), make_float2(a.y, a.y));
    return ffma2(b, make_float2(a.x, a.x), t);
}
// a * conj(b):  re = fma(a.x, b.x, a.y b.y), im = fma(a.y, b.x, -(a.x b.y))
DISCO_DEV float2 cmulc(float2 a, float2 b) {
    const float2 t = fmul2(make_float2(a.y, -a.x), make_float2(b.y, b.y));
    return ffma2(a, make_float2(b.x, b.x), t);
}
// acc + a * b  (two ffma2)
DISCO_DEV float2 cfma(float2 a, float2 b, float2 acc) {
    const float2 t = ffma2(b, make_float2(a.x, a.x), acc);
    return ffma2(make_float2(-b.y, b.x), make_float2(a.y, a.y), t);
}
// acc + conj(a) * b  (two ffma2): the filter-and-sum term  conj(w) x
DISCO_DEV float2 cfma_cj(float2 a, float2 b, float2 acc) {
    const float2 t = ffma2(b, make_float2(a.x, a.x), acc);
    return ffma2(make_float2(b.y, -b.x), make_float2(a.y, a.y), t);
}
DISCO_DEV float2 cscale(float2 a, float s) { return fmul2(a, make_float2(s, s)); }
DISCO_DEV float2 cconj(float2 a) { return make_float2(a.x, -a.y); }
// acc += s * a   (s real)
DISCO_DEV float2 cfma_r(float s, float2 a, float2 acc) { return ffma2(make_float2(s, s), a, acc); }

// Both filters of a single-node array at one (frame, bin): z = w1^H y, zn = y[ref] - z, yf = w2^H y, for the fused
// STFT filter pass.  The same helpers on the same operands in the same order as filter_dual_kernel, so the two agree
// bit for bit (filter_dual.cu keeps its own copy of these lines: calling this reschedules two of its kernels).
template <int C>
DISCO_DEV void dual_filter(const float2 (&w1)[C], const float2 (&w2)[C], const float2 (&y)[C], int ref, float2& z,
                           float2& zn, float2& yf) {
    z = make_float2(0.f, 0.f);
    yf = make_float2(0.f, 0.f);
#pragma unroll
    for (int c = 0; c < C; ++c) {
        z = cfma_cj(w1[c], y[c], z);
        yf = cfma_cj(w2[c], y[c], yf);
    }
    float2 r = y[0];
#pragma unroll
    for (int c = 1; c < C; ++c)
        if (c == ref) r = y[c];
    zn = csub(r, z);
}

// ---------------------------------------------------------------- shared-memory / TMA plumbing
DISCO_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

DISCO_DEV void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
DISCO_DEV void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
DISCO_DEV void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Wait for the phase with the given parity.  try_wait suspends the warp in hardware for up to the
// hinted time instead of spinning, so waiting warps do not steal issue slots from working ones.
DISCO_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity), "r"(20000u)
            : "memory");
    } while (!done);
}
// 1-D bulk tensor-memory-accelerator copy global -> shared, completion on an mbarrier.
// dst, src 16-byte aligned, bytes a multiple of 16.
DISCO_DEV void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
DISCO_DEV void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
DISCO_DEV void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
DISCO_DEV void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

// streaming (evict-first) 8-byte global store: outputs are written once and not re-read by this kernel
DISCO_DEV void st_stream(float2* p, float2 v) { __stcs(p, v); }
DISCO_DEV float ld_stream(const float* p) { return __ldcs(p); }
DISCO_DEV float2 ld_stream(const float2* p) { return __ldcs(p); }

}  // namespace disco
