// Mask-weighted spatial covariance matrices of D = C + K - 1 <= 4 channel spectra that are already
// in HBM (step 2 of Tango: own microphones + compressed signals of the other nodes).  Wider stacks
// (D = 5..16) use the shared-memory-staged engine of scm_wide.cu.
//
// Replaces the second triple loop of the reference (tango.py:431-440):
//   in_to_phi_s = concat(m * Y_k, m * z_others), in_to_phi_n = concat((1-m) * Y_k, (1-m) * z_others)
//   R_ss[f] = mean_t a a^H,  R_nn[f] = mean_t b b^H          (np.outer convention: R[i][j] = a_i conj(a_j))
// i.e. weights m^2 and (1-m)^2 on ONE outer product y y^H per (f, t), never materialising a, b.
//
// Data are frame-major ([.., T, F], F contiguous), so a warp covers 32 consecutive bins of one
// frame with coalesced 8-byte loads and every thread owns one bin: no shuffles are needed, the
// time reduction is a register accumulation.  A CTA owns (group, 32-bin block) for ALL frames:
//   threads = 32 bins x TW = 8 time-ways
// At D <= 4 the 2 x D(D+1)/2 accumulators AND two software-pipelined frames of operands fit in
// registers; the TW time-ways are reduced through shared memory at the end (fixed order ->
// deterministic), then scaled by 1/T and written with their conjugate mirrors.
#include "kernels.h"
#include "scm_core.cuh"

namespace disco {

template <int D>
struct ScmGeom {
    static constexpr int NPAIR = D * (D + 1) / 2;   // all pairs in one thread
    static constexpr int TW = 8;                    // time-ways (warps)
    static constexpr int THREADS = 32 * TW;
};

// compile-time recursion over the pairs: (i, j) are constants, so y[] and the accumulators stay in registers
template <int D, int Q>
struct PairAcc {
    using G = ScmGeom<D>;
    static DISCO_DEV void run(const float2 (&y)[D], float wa, float wb, float2 (&ps)[G::NPAIR],
                              float2 (&pn)[G::NPAIR]) {
        if constexpr (Q < G::NPAIR) {
            constexpr int i = tri_i<D>(Q), j = tri_j<D>(Q);
            const float2 op = cmulc(y[i], y[j]);
            ps[Q] = cfma_r(wa, op, ps[Q]);
            pn[Q] = cfma_r(wb, op, pn[Q]);
            PairAcc<D, Q + 1>::run(y, wa, wb, ps, pn);
        }
    }
};

// FC > 0: the number of bins is the compile-time constant FC (257 for the 512-point STFT), which turns
// the row-stride multiplications of every address into immediates; FC == 0: runtime F.
template <int D, bool ZF, int FC>
DISCO_DEV void scm_accumulate(const ScmArgs& a, int grp, int f, bool active, int tw,
                              float2 (&ps)[ScmGeom<D>::NPAIR], float2 (&pn)[ScmGeom<D>::NPAIR]) {
    using G = ScmGeom<D>;
    const int T = a.in.T;
    const int F = FC ? FC : a.in.F;
    const float2* ch[D];
#pragma unroll
    for (int d = 0; d < D; ++d) ch[d] = cat_channel(a.in, grp, d) + f;
    const float* mrow = a.mask ? (a.mask_ft ? a.mask + ((size_t)grp * F + f) * T : a.mask + (size_t)grp * T * F + f)
                               : nullptr;
    const int mstride = a.mask_ft ? 1 : F;
    // fused step-1 filter (K == 1 so D == C)
    float2 w1[D];
    if (ZF) {
#pragma unroll
        for (int d = 0; d < D; ++d) w1[d] = cconj(a.W1[((size_t)grp * F + f) * D + d]);
    }
    float2* zrow = ZF ? a.z_out + (size_t)grp * T * F + f : nullptr;
    float2* znrow = (ZF && a.zn_out) ? a.zn_out + (size_t)grp * T * F + f : nullptr;
    const int ref = a.ref;
    auto point = [&](const float2 (&y)[D], float m, int t) {
        const float wa = m * m, wb = mrow ? (1.f - m) * (1.f - m) : 0.f;
        PairAcc<D, 0>::run(y, wa, wb, ps, pn);
        if (ZF && active) {
            float2 z = cfma(w1[0], y[0], make_float2(0.f, 0.f));
#pragma unroll
            for (int d = 1; d < D; ++d) z = cfma(w1[d], y[d], z);
            zrow[t * F] = z;
            if (znrow) {
                float2 r = y[0];
#pragma unroll
                for (int d = 1; d < D; ++d)
                    if (d == ref) r = y[d];
                znrow[t * F] = csub(r, z);
            }
        }
    };
    auto load1 = [&](int t, float2 (&y)[D], float& m) {
        if (active && t < T) {
#pragma unroll
            for (int d = 0; d < D; ++d) y[d] = ch[d][t * F];
            m = mrow ? mrow[t * mstride] : 1.f;
        } else {
#pragma unroll
            for (int d = 0; d < D; ++d) y[d] = make_float2(0.f, 0.f);
            m = 1.f;
        }
    };
    // Software pipeline over time: the loads of the next round are in flight (issued straight into two
    // extra register buffers) while this round's two frames are consumed.
    constexpr int TS = G::TW;
    float2 ya[D], yb[D];
    float ma, mb;
    int t = tw;
    load1(t, ya, ma);
    load1(t + TS, yb, mb);
    for (; t + 3 * TS < T; t += 2 * TS) {   // both frames of this round and of the next exist
        float2 yc[D], yd[D];
        float mc, md;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            yc[d] = ch[d][(t + 2 * TS) * F];
            yd[d] = ch[d][(t + 3 * TS) * F];
        }
        mc = mrow ? mrow[(t + 2 * TS) * mstride] : 1.f;
        md = mrow ? mrow[(t + 3 * TS) * mstride] : 1.f;
        point(ya, ma, t);
        point(yb, mb, t + TS);
#pragma unroll
        for (int d = 0; d < D; ++d) {
            ya[d] = yc[d];
            yb[d] = yd[d];
        }
        ma = mc;
        mb = md;
    }
    for (; t < T; t += 2 * TS) {            // tail rounds (predicated loads)
        float2 yc[D], yd[D];
        float mc, md;
        load1(t + 2 * TS, yc, mc);
        load1(t + 3 * TS, yd, md);
        point(ya, ma, t);
        if (t + TS < T) point(yb, mb, t + TS);
#pragma unroll
        for (int d = 0; d < D; ++d) {
            ya[d] = yc[d];
            yb[d] = yd[d];
        }
        ma = mc;
        mb = md;
    }
}

template <int D, bool ZF, int FC>
__global__ void __launch_bounds__(ScmGeom<D>::THREADS, 2) masked_scm_kernel(ScmArgs a) {
    using G = ScmGeom<D>;
    extern __shared__ float2 red[];  // [NPAIR][2][32]
    const int lane = threadIdx.x & 31;
    const int tw = threadIdx.x >> 5;
    const int grp = blockIdx.y;
    const int f = blockIdx.x * 32 + lane;
    const bool active = f < a.in.F;
    const int fc = active ? f : a.in.F - 1;

    float2 ps[G::NPAIR], pn[G::NPAIR];
#pragma unroll
    for (int q = 0; q < G::NPAIR; ++q) ps[q] = pn[q] = make_float2(0.f, 0.f);

    scm_accumulate<D, ZF, FC>(a, grp, fc, active, tw, ps, pn);

    // reduce the TW time-ways in fixed order: way w adds into way 0 through shared memory
    for (int w = 1; w < G::TW; ++w) {
        if (tw == w) {
#pragma unroll
            for (int q = 0; q < G::NPAIR; ++q) {
                red[(q * 2 + 0) * 32 + lane] = ps[q];
                red[(q * 2 + 1) * 32 + lane] = pn[q];
            }
        }
        __syncthreads();
        if (tw == 0) {
#pragma unroll
            for (int q = 0; q < G::NPAIR; ++q) {
                ps[q] = cadd(ps[q], red[(q * 2 + 0) * 32 + lane]);
                pn[q] = cadd(pn[q], red[(q * 2 + 1) * 32 + lane]);
            }
        }
        __syncthreads();
    }
    if (tw == 0 && active) {
        const float inv_T = 1.0f / (float)a.in.T;
        float2* Rs = a.Rss + ((size_t)grp * a.in.F + f) * D * D;
        float2* Rn = a.Rnn + ((size_t)grp * a.in.F + f) * D * D;
        // scaled pairs with their conjugate mirrors, as store_pairs (scm_core.cuh) writes them; calling store_pairs or
        // taking (i, j) from tri_i / tri_j here makes nvcc reschedule the whole kernel, so the epilogue stays as it is
#pragma unroll
        for (int q = 0; q < G::NPAIR; ++q) {
            int i = 0, n = D, pp = q;
            while (pp >= n) {
                pp -= n;
                --n;
                ++i;
            }
            const int j = i + pp;
            float2 s = cscale(ps[q], inv_T), nn = cscale(pn[q], inv_T);
            if (i == j) s.y = 0.f, nn.y = 0.f;
            Rs[i * D + j] = s;
            Rn[i * D + j] = nn;
            if (i != j) {
                Rs[j * D + i] = cconj(s);
                Rn[j * D + i] = cconj(nn);
            }
        }
    }
}

template <int D, bool ZF, int FC>
static cudaError_t launch_dzf(const ScmArgs& a, cudaStream_t st) {
    using G = ScmGeom<D>;
    const size_t smem = (size_t)G::NPAIR * 2 * 32 * sizeof(float2);
    auto kern = masked_scm_kernel<D, ZF, FC>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
    }
    dim3 grid((a.in.F + 31) / 32, a.in.n_grp);
    kern<<<grid, G::THREADS, smem, st>>>(a);
    return cudaGetLastError();
}

template <int D, bool ZF>
static cudaError_t launch_dz(const ScmArgs& a, cudaStream_t st) {
    // the 512-point STFT (F = 257) of small nodes is the hot configuration: compile-time row stride
    if (a.in.F == 257) return launch_dzf<D, ZF, 257>(a, st);
    return launch_dzf<D, ZF, 0>(a, st);
}

template <int D>
static cudaError_t launch_d(const ScmArgs& a, cudaStream_t st) {
    if (a.W1 != nullptr) return launch_dz<D, true>(a, st);
    return launch_dz<D, false>(a, st);
}

cudaError_t launch_masked_scm(const ScmArgs& a, cudaStream_t st) {
    const int D = a.in.C + a.in.K - 1;
    if (D >= 5) return launch_masked_scm_wide(a, st);
    switch (D) {
        case 1: return launch_d<1>(a, st);
        case 2: return launch_d<2>(a, st);
        case 3: return launch_d<3>(a, st);
        case 4: return launch_d<4>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
