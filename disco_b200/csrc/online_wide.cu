// Recursive (online) SCMs of WIDE channel stacks, D = C + K - 1 from 9 to 16 (online.cu covers 1..8).
//
// Same values as online.cu's two-level scan, evaluated in the same operation order:
//   A_j = the sequential float32 sum over the frames of block j in frame order, each term WidePairAcc's arithmetic
//         with weight gw[t1 - 1 - t] * w_t                                   (scm_blocks_kernel)
//   R_j = fmaf(lam_j, R_(j-1), A_j), lam_j = lambda^P (lambda^(frames) for a short last block)   (scm_combine_kernel)
// so every (group, block, bin) entry is bit-identical to that definition whatever the launch geometry or batch.
//
// Different engine: at D >= 9 one thread per (bin, block) with all D(D+1)/2 pairs of both matrices in registers
// spills.  Here a CTA owns (group, 32-bin block) and streams the group's frames through the cp.async ring of
// scm_core.cuh; its 4 warps are the NPART = 4 pair partitions of masked_scm_wide and one time-way, so each warp
// walks every frame in order and closes block j at its last frame:
//   R_j = lam_j R_(j-1) + A_j on its pairs, stored with store_pairs (both triangles), A reset to 0.
// The carry R_(j-1) is re-read from the thread's own store of the previous block (an L2 hit), so it costs no
// registers and the kernel writes every R_j once (no separate combine pass over the block matrices).
// R0 (block -1) is read on the upper triangle only, and of its diagonal only the real part.
//
// The Nyquist block of F = 32n + 1 keeps lane 0 on bin F - 1 and leaves the other 31 lanes idle (their copies are
// zero-filled, nothing is read or stored): a lane butterfly or lanes mapped to blocks would change the order of the
// sums, and an idle-lane CTA takes no longer than a full one.
//
// LEN = true (a.frames set): the group's utterance has its own Tn <= T frames.  The ring streams frames [0, Tn) only,
// the last block closes at Tn - 1 with lam_n[frames - 1], and the blocks past it are stored as exact zeros: the same
// frames, tiles and operations as a call on that utterance alone, so the same bits.
#include "kernels.h"
#include "scm_core.cuh"

namespace disco {

template <int D, int TS, int NS>
struct OnlineWideCfg {
    static constexpr int NPART = 4;                  // warps: pair partitions, one time-way
    static constexpr int NPP = PairGeom<D, NPART>::NPP;
    static constexpr int YROWS = D * TS;             // stage row d * TS + s: channel d, frame slot s
    static constexpr size_t OFF_M = (size_t)NS * YROWS * 32 * sizeof(float2);
    static constexpr size_t OFF_P = OFF_M + (size_t)NS * TS * 32 * sizeof(float);
    static constexpr size_t SMEM = OFF_P + (size_t)D * sizeof(void*);
    static_assert(TS == NPART, "loader: warp w copies slot w of every channel");
};

// block j closes: R_j = lam_j R_(j-1) + A_j on this partition's pairs (R_(-1) = R0 or 0), stored with mirrors
template <int D, int PART, bool LEN>
DISCO_DEV void online_close(const OnlineParams<LEN>& a, int grp, int f, int j, int Tn,
                            float2 (&ps)[PairGeom<D, 4>::NPP], float2 (&pn)[PairGeom<D, 4>::NPP]) {
    using G = PairGeom<D, 4>;
    const int F = a.in.F;
    float lam;
    if constexpr (LEN) {   // the utterance's last block may be short: lambda^(its frames)
        const int n = min(Tn - j * a.P, a.P);
        lam = a.lam_n[n - 1];
    } else {
        lam = (j == a.J - 1 && a.in.T - j * a.P != a.P) ? a.lam_last : a.lam_block;
    }
    const float2 *cs = nullptr, *cn = nullptr;
    if (j > 0) {   // this thread's own store of block j - 1
        const size_t prev = ((size_t)(grp * a.J + j - 1) * F + f) * D * D;
        cs = a.Rss + prev;
        cn = a.Rnn + prev;
    } else if (a.R0ss) {
        const size_t r0 = ((size_t)grp * F + f) * D * D;
        cs = a.R0ss + r0;
        cn = a.R0nn + r0;
    }
#pragma unroll
    for (int q = 0; q < G::NPP; ++q) {
        const int pidx = q * 4 + PART;
        if (pidx < G::NPAIR) {
            const int r = tri_i<D>(pidx), c = tri_j<D>(pidx);
            float2 rs = make_float2(0.f, 0.f), rn = rs;
            if (cs) {
                rs = cs[r * D + c];
                rn = cn[r * D + c];
                if (r == c) rs.y = rn.y = 0.f;
            }
            ps[q] = make_float2(fmaf(lam, rs.x, ps[q].x), fmaf(lam, rs.y, ps[q].y));
            pn[q] = make_float2(fmaf(lam, rn.x, pn[q].x), fmaf(lam, rn.y, pn[q].y));
        }
    }
    const size_t mat = ((size_t)(grp * a.J + j) * F + f) * D * D;
    store_pairs<D, 4>(ps, pn, PART, 1.0f, a.Rss + mat, a.Rnn + mat, [](int r) { return r; });
}

// one warp's pass over the ns frames [t, t + ns) of a stage; closes every block whose last frame is among them
template <int D, int TS, int PART, bool LEN>
DISCO_DEV void online_tile(const OnlineParams<LEN>& a, const float2* yb, const float* mb, bool has_mask, int grp, int f,
                           bool ok, int t, int ns, int Tn, int& j, int& t1, float2 (&ps)[PairGeom<D, 4>::NPP],
                           float2 (&pn)[PairGeom<D, 4>::NPP]) {
    using G = PairGeom<D, 4>;
#pragma unroll 1
    for (int s = 0; s < ns; ++s, ++t) {
        float2 x[D], xs[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            x[d] = yb[(d * TS + s) * 32];
            xs[d] = make_float2(x[d].y, -x[d].x);
        }
        const float m = has_mask ? mb[s * 32] : 1.f;
        const float g = a.gw[t1 - 1 - t];                   // (1 - lambda) lambda^(frames until the block's end)
        const float ws = a.power == 2 ? m * m : m;
        const float wn = !has_mask ? 0.f : (a.power == 2 ? (1.f - m) * (1.f - m) : 1.f - m);
        WidePairAcc<D, 4, PART>::run(x, xs, g * ws, g * wn, ps, pn);
        if (t == t1 - 1) {
            if (ok) online_close<D, PART, LEN>(a, grp, f, j, Tn, ps, pn);
#pragma unroll
            for (int q = 0; q < G::NPP; ++q) ps[q] = pn[q] = make_float2(0.f, 0.f);
            ++j;
            t1 = min(LEN ? Tn : a.in.T, t1 + a.P);
        }
    }
}

template <int D, int TS, int NS, int MINB, bool LEN>
__global__ void __launch_bounds__(32 * 4, MINB) scm_recursive_wide_kernel(OnlineParams<LEN> a) {
    using G = OnlineWideCfg<D, TS, NS>;
    extern __shared__ __align__(16) unsigned char online_smem[];
    float2* const ystage = reinterpret_cast<float2*>(online_smem);
    float* const mstage = reinterpret_cast<float*>(online_smem + G::OFF_M);
    const float2** const plane = reinterpret_cast<const float2**>(online_smem + G::OFF_P);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = blockIdx.y, T = a.in.T, F = a.in.F;
    const int f = blockIdx.x * 32 + lane;
    const bool ok = f < F;                           // lanes past F (31 of the Nyquist block) stay idle
    const int fcol = ok ? f : F - 1;
    int Tn = T;                                      // frames of this group's utterance (T: the row stride)
    if constexpr (LEN) Tn = a.frames[grp / a.in.n_sel];
    const int ntile = (Tn + TS - 1) / TS;
    const bool has_mask = a.mask != nullptr;

    if (threadIdx.x < D) plane[threadIdx.x] = cat_channel(a.in, grp, threadIdx.x);
    __syncthreads();

    const float* const mbase = has_mask ? a.mask + (size_t)grp * T * F + fcol : nullptr;
    auto issue = [&](int i) {
        if (i < ntile) {
            const int st = i % NS;
            const int t = i * TS + warp;             // warp w copies frame slot w of every channel
            const bool v = ok && t < Tn;
            const size_t toff = (size_t)(v ? t : 0) * F + fcol;
            float2* dst = ystage + (st * G::YROWS + warp) * 32 + lane;
#pragma unroll
            for (int d = 0; d < D; ++d) cp_async8(dst + d * TS * 32, plane[d] + toff, v);
            if (has_mask) cp_async4(mstage + (st * TS + warp) * 32 + lane, mbase + (size_t)(v ? t : 0) * F, v);
        }
        cp_async_commit();
    };

    float2 ps[G::NPP], pn[G::NPP];
#pragma unroll
    for (int q = 0; q < G::NPP; ++q) ps[q] = pn[q] = make_float2(0.f, 0.f);
    int j = 0, t1 = min(Tn, a.P);                    // current block and its end

#pragma unroll
    for (int i = 0; i < NS - 1; ++i) issue(i);
    for (int i = 0; i < ntile; ++i) {
        cp_async_wait<NS - 2>();                     // tile i has landed (this thread's copies)
        __syncthreads();                             // ... everyone's; stage (i-1) % NS is free
        issue(i + NS - 1);
        const float2* yb = ystage + (i % NS) * G::YROWS * 32 + lane;
        const float* mb = mstage + (i % NS) * TS * 32 + lane;
        const int t0 = i * TS, ns = min(TS, Tn - t0);
        switch (warp) {   // warp-uniform: keeps the (i, j) of every accumulator compile-time
            case 0: online_tile<D, TS, 0, LEN>(a, yb, mb, has_mask, grp, f, ok, t0, ns, Tn, j, t1, ps, pn); break;
            case 1: online_tile<D, TS, 1, LEN>(a, yb, mb, has_mask, grp, f, ok, t0, ns, Tn, j, t1, ps, pn); break;
            case 2: online_tile<D, TS, 2, LEN>(a, yb, mb, has_mask, grp, f, ok, t0, ns, Tn, j, t1, ps, pn); break;
            default: online_tile<D, TS, 3, LEN>(a, yb, mb, has_mask, grp, f, ok, t0, ns, Tn, j, t1, ps, pn); break;
        }
    }
    if constexpr (LEN) {   // blocks past the utterance's end: exact zeros (this CTA's bins are contiguous per block)
        const int n = min(32, F - (int)blockIdx.x * 32) * D * D;
        for (int jj = (Tn + a.P - 1) / a.P; jj < a.J; ++jj) {
            const size_t mat = ((size_t)(grp * a.J + jj) * F + blockIdx.x * 32) * D * D;
            for (int e = threadIdx.x; e < n; e += blockDim.x) a.Rss[mat + e] = a.Rnn[mat + e] = make_float2(0.f, 0.f);
        }
    }
}

template <int D>
static cudaError_t launch_recursive_wide_d(const OnlineLengthsArgs& a, cudaStream_t st) {
    constexpr int TS = 4, NS = 4;
    constexpr int MINB = 1;
    using G = OnlineWideCfg<D, TS, NS>;
    dim3 grid((a.in.F + 31) / 32, a.in.n_grp);
    if (a.frames) {
        auto kern = scm_recursive_wide_kernel<D, TS, NS, MINB, true>;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G::SMEM);
        if (e != cudaSuccess) return e;
        kern<<<grid, 32 * 4, G::SMEM, st>>>(a);
    } else {
        auto kern = scm_recursive_wide_kernel<D, TS, NS, MINB, false>;
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G::SMEM);
        if (e != cudaSuccess) return e;
        kern<<<grid, 32 * 4, G::SMEM, st>>>(static_cast<const OnlineArgs&>(a));
    }
    return cudaGetLastError();
}

cudaError_t launch_scm_recursive_wide(const OnlineLengthsArgs& a, cudaStream_t st) {
    switch (a.in.C + a.in.K - 1) {
        case 9: return launch_recursive_wide_d<9>(a, st);
        case 10: return launch_recursive_wide_d<10>(a, st);
        case 11: return launch_recursive_wide_d<11>(a, st);
        case 12: return launch_recursive_wide_d<12>(a, st);
        case 13: return launch_recursive_wide_d<13>(a, st);
        case 14: return launch_recursive_wide_d<14>(a, st);
        case 15: return launch_recursive_wide_d<15>(a, st);
        case 16: return launch_recursive_wide_d<16>(a, st);
        default: return cudaErrorNotSupported;
    }
}

}  // namespace disco
