// Mask-weighted SCMs of WIDE channel stacks (D = C + K - 1 from 5 to 16) that are already in HBM: the
// step-2 statistics of Tango for nodes with many microphones / many neighbours, and the K = 1 middle
// step of large single arrays (with the step-1 filter-and-sum fused in: ZF).
//
// Same contract as scm.cu (reference tango.py:431-440; weights m^2 and (1-m)^2 on one outer product
// per (f, t)), different engine: at D >= 5 the accumulators (2 D(D+1)/2 complex numbers per bin) leave
// no registers for software-pipelined global loads, and the thread-per-bin kernel of scm.cu ran at one
// CTA of 8 warps per SM, exposed to L2 latency.  Here a CTA owns (group, 32-bin block) and streams tiles
// of TS frames through a cp.async ring in shared memory (scm_core.cuh); its warps are
//   NPART pair-partitions x TW time-ways (way w takes the slots ts = w, w + TW, ... of every tile),
// all operands come from shared memory at immediate offsets, and the TW ways are summed through shared
// memory at the end in fixed order (deterministic, no atomics).
#include "kernels.h"
#include "scm_core.cuh"

namespace disco {

template <int D, int NPART, int TW, int TS, int NS>
struct WideCfg {
    static constexpr int NPP = PairGeom<D, NPART>::NPP;
    static constexpr int NW = NPART * TW;
    static constexpr int SL = TS / TW;               // slots per way and tile
    static constexpr int YROWS = D * TS, MROWS = TS;
    static constexpr size_t OFF_M = (size_t)NS * YROWS * 32 * sizeof(float2);
    static constexpr size_t OFF_W = OFF_M + (size_t)NS * MROWS * 32 * sizeof(float);
    static constexpr size_t OFF_P = OFF_W + (size_t)D * 32 * sizeof(float2);
    static constexpr size_t SMEM_PIPE = OFF_P + (size_t)((D + 1) / 2 * 2) * sizeof(void*);
    static constexpr size_t SMEM_RED = TW > 1 ? (size_t)NPART * NPP * 2 * 32 * sizeof(float2) : 0;
    static constexpr size_t SMEM = SMEM_PIPE > SMEM_RED ? SMEM_PIPE : SMEM_RED;
    static_assert(TS % TW == 0 && NW % TS == 0, "loader fast path: every thread keeps one slot");
    static_assert(SL % NPART == 0 || NPART > 2, "fused z output: the slots of a way are dealt to its partitions");
};

// one way's slots of one tile: operands from shared memory, optional fused z = w1^H y output
template <int D, int NPART, int TW, int TS, int NS, bool ZF, int PART>
DISCO_DEV void wide_tile(const ScmArgs& a, const float2* yb, const float* mb, const float2* w1s, bool has_mask,
                         const LaneGeom& lg, int grp, int tfirst, float2 (&ps)[WideCfg<D, NPART, TW, TS, NS>::NPP],
                         float2 (&pn)[WideCfg<D, NPART, TW, TS, NS>::NPP]) {
    using G = WideCfg<D, NPART, TW, TS, NS>;
#pragma unroll
    for (int s = 0; s < G::SL; ++s) {
        float2 x[D];
#pragma unroll
        for (int d = 0; d < D; ++d) x[d] = yb[(d * TS + s * TW) * 32];
        const float m = has_mask ? mb[s * TW * 32] : 1.f;
        wide_point<D, NPART, PART>(x, m, has_mask, ps, pn);
        // K == 1, D == C: z = w1^H y, zn = y[ref] - z (tango.py:369-376); slot s is written by partition s % NPART
        // (every partition holds all D operands), which balances the extra work over the partitions
        if (ZF && (s % NPART == PART)) {
            const int t = tfirst + s * TW * lg.tmul;
            float2 z = cfma(w1s[0], x[0], make_float2(0.f, 0.f)), yr = x[0];
#pragma unroll
            for (int d = 1; d < D; ++d) {
                z = cfma(w1s[d * 32], x[d], z);
                if (d == a.ref) yr = x[d];
            }
            if (lg.ok && t < a.in.T) {
                const size_t o = ((size_t)grp * a.in.T + t) * a.in.F + lg.fcol;
                a.z_out[o] = z;
                if (a.zn_out) a.zn_out[o] = csub(yr, z);
            }
        }
    }
}

template <int D, int NPART, int TW, int TS, int NS, bool ZF, int MINB>
__global__ void __launch_bounds__(32 * NPART * TW, MINB) masked_scm_wide_kernel(ScmArgs a) {
    using G = WideCfg<D, NPART, TW, TS, NS>;
    constexpr int NW = G::NW;
    extern __shared__ __align__(16) unsigned char wide_smem[];
    float2* const ystage = reinterpret_cast<float2*>(wide_smem);
    float* const mstage = reinterpret_cast<float*>(wide_smem + G::OFF_M);
    float2* const w1s = reinterpret_cast<float2*>(wide_smem + G::OFF_W);
    const float2** const plane = reinterpret_cast<const float2**>(wide_smem + G::OFF_P);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int part = warp % NPART, tw = warp / NPART;
    const int grp = blockIdx.y, T = a.in.T, F = a.in.F;
    const LaneGeom lg = lane_geom(blockIdx.x, lane, F);
    const int tspan = TS * lg.tmul;
    const int ntile = (T + tspan - 1) / tspan;
    const bool has_mask = a.mask != nullptr;

    if (threadIdx.x < D) plane[threadIdx.x] = cat_channel(a.in, grp, threadIdx.x);
    if (ZF)
        for (int d = warp; d < D; d += NW) w1s[d * 32 + lane] = cconj(a.W1[((size_t)grp * F + lg.fcol) * D + d]);
    __syncthreads();

    // loader: row r = warp + q * NW of a stage is (channel r / TS, slot r % TS); NW % TS == 0, so a thread
    // keeps the slot warp % TS -> one frame index and one validity per tile
    const int lslot = warp % TS;
    const float* const mbase = !has_mask ? nullptr
                               : a.mask_ft ? a.mask + ((size_t)grp * F + lg.fcol) * T
                                           : a.mask + (size_t)grp * T * F + lg.fcol;
    const int mstride = a.mask_ft ? 1 : F;
    auto issue = [&](int i) {
        if (i < ntile) {
            const int st = i % NS;
            const int t = i * tspan + lg.tl + lslot * lg.tmul;
            const bool v = lg.ok && t < T;
            const size_t toff = (size_t)(v ? t : 0) * F + lg.fcol;
            float2* dst = ystage + (st * G::YROWS + warp) * 32 + lane;
#pragma unroll
            for (int q = 0; q < (G::YROWS + NW - 1) / NW; ++q) {
                const int r = warp + q * NW;
                if (G::YROWS % NW == 0 || r < G::YROWS) cp_async8(dst + q * NW * 32, plane[r / TS] + toff, v);
            }
            if (has_mask && warp < G::MROWS)     // MROWS == TS <= NW: one mask row per warp
                cp_async4(mstage + (st * G::MROWS + warp) * 32 + lane, mbase + (size_t)(v ? t : 0) * mstride, v);
        }
        cp_async_commit();
    };

    float2 ps[G::NPP], pn[G::NPP];
#pragma unroll
    for (int q = 0; q < G::NPP; ++q) ps[q] = pn[q] = make_float2(0.f, 0.f);

#pragma unroll
    for (int i = 0; i < NS - 1; ++i) issue(i);
    for (int i = 0; i < ntile; ++i) {
        cp_async_wait<NS - 2>();                     // tile i has landed (this thread's copies)
        __syncthreads();                             // ... everyone's; stage (i-1) % NS is free
        issue(i + NS - 1);
        const float2* yb = ystage + ((i % NS) * G::YROWS + tw) * 32 + lane;
        const float* mb = mstage + ((i % NS) * G::MROWS + tw) * 32 + lane;
        const int tfirst = i * tspan + lg.tl + tw * lg.tmul;
        switch (part) {   // warp-uniform: keeps the (i, j) of every accumulator compile-time
            case 0: wide_tile<D, NPART, TW, TS, NS, ZF, 0>(a, yb, mb, w1s + lane, has_mask, lg, grp, tfirst, ps, pn); break;
            case 1: if (NPART > 1) wide_tile<D, NPART, TW, TS, NS, ZF, (NPART > 1 ? 1 : 0)>(a, yb, mb, w1s + lane, has_mask, lg, grp, tfirst, ps, pn); break;
            case 2: if (NPART > 2) wide_tile<D, NPART, TW, TS, NS, ZF, (NPART > 2 ? 2 : 0)>(a, yb, mb, w1s + lane, has_mask, lg, grp, tfirst, ps, pn); break;
            default: if (NPART > 3) wide_tile<D, NPART, TW, TS, NS, ZF, (NPART > 3 ? 3 : 0)>(a, yb, mb, w1s + lane, has_mask, lg, grp, tfirst, ps, pn); break;
        }
    }

    // sum the TW time-ways in fixed order through shared memory (aliases the stage ring)
    if constexpr (TW > 1) {
        cp_async_wait<0>();
        float2* red = reinterpret_cast<float2*>(wide_smem) + (size_t)part * G::NPP * 2 * 32 + lane;
        for (int w = 1; w < TW; ++w) {
            __syncthreads();
            if (tw == w) {
#pragma unroll
                for (int q = 0; q < G::NPP; ++q) {
                    red[(q * 2 + 0) * 32] = ps[q];
                    red[(q * 2 + 1) * 32] = pn[q];
                }
            }
            __syncthreads();
            if (tw == 0) {
#pragma unroll
                for (int q = 0; q < G::NPP; ++q) {
                    ps[q] = cadd(ps[q], red[(q * 2 + 0) * 32]);
                    pn[q] = cadd(pn[q], red[(q * 2 + 1) * 32]);
                }
            }
        }
    }
    if (tw == 0) {
        if (lg.nyq) lane_butterfly<G::NPP>(ps, pn);  // CTA-uniform
        if (lg.nyq ? lane == 0 : lg.ok) {
            const size_t m = (size_t)grp * F + lg.fcol;
            store_pairs<D, NPART>(ps, pn, part, 1.0f / (float)T, a.Rss + m * D * D, a.Rnn + m * D * D,
                                  [](int r) { return r; });
        }
    }
}

template <int D, bool ZF>
static cudaError_t launch_wide_dz(const ScmArgs& a, cudaStream_t st) {
    constexpr int NPART = D <= 6 ? 1 : (D <= 8 ? 2 : 4);
    constexpr int TW = 8 / NPART;                    // 8 warps per CTA
    constexpr int TS = TW >= 4 ? 8 : 4;              // NW = 8 is a multiple of TS
    constexpr int NS = 3;
    using G = WideCfg<D, NPART, TW, TS, NS>;
    constexpr int THREADS = 32 * G::NW;
    constexpr int BY_SMEM = (int)((227 * 1024) / (G::SMEM + 1024));
    constexpr int BY_REGS = 65536 / (THREADS * (4 * G::NPP + 3 * D + 26));
    constexpr int MINB = BY_SMEM < BY_REGS ? (BY_SMEM < 1 ? 1 : BY_SMEM) : (BY_REGS < 1 ? 1 : BY_REGS);
    auto kern = masked_scm_wide_kernel<D, NPART, TW, TS, NS, ZF, MINB>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G::SMEM);
    if (e != cudaSuccess) return e;
    dim3 grid((a.in.F + 31) / 32, a.in.n_grp);
    kern<<<grid, THREADS, G::SMEM, st>>>(a);
    return cudaGetLastError();
}

template <int D>
static cudaError_t launch_wide_d(const ScmArgs& a, cudaStream_t st) {
    if (a.W1 != nullptr) {
        if (D > 8) return cudaErrorInvalidValue;
        return launch_wide_dz<(D > 8 ? 5 : D), true>(a, st);
    }
    return launch_wide_dz<D, false>(a, st);
}

cudaError_t launch_masked_scm_wide(const ScmArgs& a, cudaStream_t st) {
    switch (a.in.C + a.in.K - 1) {
        case 5: return launch_wide_d<5>(a, st);
        case 6: return launch_wide_d<6>(a, st);
        case 7: return launch_wide_d<7>(a, st);
        case 8: return launch_wide_d<8>(a, st);
        case 9: return launch_wide_d<9>(a, st);
        case 10: return launch_wide_d<10>(a, st);
        case 11: return launch_wide_d<11>(a, st);
        case 12: return launch_wide_d<12>(a, st);
        case 13: return launch_wide_d<13>(a, st);
        case 14: return launch_wide_d<14>(a, st);
        case 15: return launch_wide_d<15>(a, st);
        case 16: return launch_wide_d<16>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
