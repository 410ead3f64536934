// Recursive (online) statistics and block-wise filtering: the causal variant of the Tango kernels
// (SURVEY.md §8 f-4).  The reference's only streaming primitive is the one-frame update
//   spatial_correlation_matrix(Rxx, x, lambda_cor, M):  R <- lambda R + (1 - lambda) [M] x x^H
// (se_utils/internal_formulas.py:84-103), meant to be called once per frame and bin from Python.
//
// A first-order recursion is a scan; it is evaluated here in two levels so that the time axis is parallel:
//   scm_blocks   every block j of P frames independently:  A_j = sum_i (1 - lambda) lambda^(n_j-1-i) w_i x_i x_i^H
//                (thread = (bin, block), all D(D+1)/2 pairs in registers, w = m^2 / (1-m)^2 or m / (1-m))
//   scm_combine  the short serial part, elementwise over (group, bin, matrix entry):  R_j = lambda^(n_j) R_(j-1) + A_j
// The result is the smoothed pair (R_ss, R_nn) after the last frame of every block: [group][J][F][D][D], which
// the batched solver (solve.cu / solve_small.cu) turns into one filter per block, and
//   filter_sum_blocks   applies filter j(t) = t / P - lag to frame t  (lag = 1: strictly causal, the filter of
//                the last COMPLETED block; frames before the first filter pass the reference channel through).
// With a.frames set (template LEN = true) utterance b = grp / n_sel has its own T_b <= T frames and J_b blocks: block
// j ends at min((j + 1) P, T_b), a short last block decays by lam_n[frames - 1] (the same float as a run of that
// utterance alone), nothing past T_b is read, and blocks >= J_b / frames >= T_b are written as exact zeros.  Every
// (group, block, bin) entry then equals the utterance run alone bit for bit.  LEN = false is the uniform kernel.
#include "kernels.h"
#include "scm_core.cuh"

namespace disco {

constexpr int kOnlineBY = 4;   // blocks of frames per CTA (threadIdx.y)

template <int D, bool LEN>
__global__ void __launch_bounds__(32 * kOnlineBY) scm_blocks_kernel(OnlineParams<LEN> a) {
    using G = PairGeom<D, 1>;
    const int T = a.in.T, F = a.in.F;
    const int f = blockIdx.x * 32 + threadIdx.x;
    const int j = blockIdx.y * kOnlineBY + threadIdx.y;
    const int grp = blockIdx.z;
    if (f >= F || j >= a.J) return;
    int Tn = T;                                             // frames of this group's utterance
    if constexpr (LEN) Tn = a.frames[grp / a.in.n_sel];
    const int t0 = j * a.P, t1 = min(Tn, t0 + a.P);         // frames [t0, t1): none past the end (A_j = 0 stored)
    const float2* ch[D];
#pragma unroll
    for (int d = 0; d < D; ++d) ch[d] = cat_channel(a.in, grp, d) + f;
    const float* mrow = a.mask ? a.mask + (size_t)grp * T * F + f : nullptr;

    float2 ps[G::NPP], pn[G::NPP];
#pragma unroll
    for (int q = 0; q < G::NPP; ++q) ps[q] = pn[q] = make_float2(0.f, 0.f);
    for (int t = t0; t < t1; ++t) {
        float2 x[D], xs[D];
#pragma unroll
        for (int d = 0; d < D; ++d) {
            x[d] = ch[d][(size_t)t * F];
            xs[d] = make_float2(x[d].y, -x[d].x);
        }
        const float m = mrow ? mrow[(size_t)t * F] : 1.f;
        const float g = a.gw[t1 - 1 - t];                   // (1 - lambda) lambda^(frames until the block's end)
        const float ws = a.power == 2 ? m * m : m;
        const float wn = !mrow ? 0.f : (a.power == 2 ? (1.f - m) * (1.f - m) : 1.f - m);
        WidePairAcc<D, 1, 0>::run(x, xs, g * ws, g * wn, ps, pn);
    }
    const size_t mat = ((size_t)(grp * a.J + j) * F + f) * D * D;
    store_pairs<D, 1>(ps, pn, 0, 1.0f, a.Rss + mat, a.Rnn + mat, [](int r) { return r; });
}

// R_j = lam_j R_(j-1) + A_j in place, one thread per (group, bin, entry); R_(-1) = R0 (or 0)
template <bool LEN>
__global__ void scm_combine_kernel(OnlineParams<LEN> a, int DD) {
    const size_t per_grp = (size_t)a.in.F * DD;
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= per_grp) return;
    const int grp = blockIdx.y;
    const int last = a.in.T - (a.J - 1) * a.P;              // frames in the last block
    float2* mats[2] = {a.Rss, a.Rnn};
    const float2* init[2] = {a.R0ss, a.R0nn};
#pragma unroll
    for (int w = 0; w < 2; ++w) {
        float2 r = init[w] ? init[w][(size_t)grp * per_grp + e] : make_float2(0.f, 0.f);
        float2* p = mats[w] + (size_t)grp * a.J * per_grp + e;
        if constexpr (LEN) {   // this utterance's J_b blocks (the later ones keep the zeros of scm_blocks)
            const int Tn = a.frames[grp / a.in.n_sel], Jn = (Tn + a.P - 1) / a.P;
            const float lam_end = a.lam_n[Tn - (Jn - 1) * a.P - 1];
            for (int j = 0; j < Jn; ++j) {
                const float lam = j == Jn - 1 ? lam_end : a.lam_block;
                const float2 v = p[(size_t)j * per_grp];
                r = make_float2(fmaf(lam, r.x, v.x), fmaf(lam, r.y, v.y));
                p[(size_t)j * per_grp] = r;
            }
            continue;
        }
        for (int j = 0; j < a.J; ++j) {
            const float lam = (j == a.J - 1 && last != a.P) ? a.lam_last : a.lam_block;
            const float2 v = p[(size_t)j * per_grp];
            r = make_float2(fmaf(lam, r.x, v.x), fmaf(lam, r.y, v.y));
            p[(size_t)j * per_grp] = r;
        }
    }
}

template <int D, bool LEN>
__global__ void __launch_bounds__(32 * kOnlineBY) filter_sum_blocks_kernel(OnlineFilterArgs a) {
    const int T = a.in.T, F = a.in.F;
    const int f = blockIdx.x * 32 + threadIdx.x;
    const int j = blockIdx.y * kOnlineBY + threadIdx.y;
    const int grp = blockIdx.z;
    if (f >= F || j >= a.J) return;
    const int t0 = j * a.P;
    int t1 = min(T, t0 + a.P);
    if constexpr (LEN) {   // frames past the utterance's end are 0, and neither x nor W is read for them
        const int Tn = a.frames[grp / a.in.n_sel];
        for (int t = max(t0, Tn); t < t1; ++t) {
            const size_t o = ((size_t)grp * T + t) * F + f;
            a.out[o] = make_float2(0.f, 0.f);
            if (a.resid) a.resid[o] = make_float2(0.f, 0.f);
        }
        if (t0 >= Tn) return;                               // block j >= J_b: its filter jw < j is never needed
        t1 = min(t1, Tn);
    }
    const int jw = j - a.lag;                               // filter in force during block j
    float2 w[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        if (jw >= 0) {
            const float2 v = a.W[((size_t)(grp * a.J + jw) * F + f) * D + d];
            w[d] = a.conj_w ? cconj(v) : v;
        } else {
            w[d] = make_float2(d == a.ref ? 1.f : 0.f, 0.f);    // no filter yet: pass the reference channel
        }
    }
    const float2* ch[D];
#pragma unroll
    for (int d = 0; d < D; ++d) ch[d] = cat_channel(a.in, grp, d) + f;
    for (int t = t0; t < t1; ++t) {
        float2 z = make_float2(0.f, 0.f), yr = make_float2(0.f, 0.f);
#pragma unroll
        for (int d = 0; d < D; ++d) {
            const float2 x = ch[d][(size_t)t * F];
            z = cfma(w[d], x, z);
            if (d == a.ref) yr = x;
        }
        const size_t o = ((size_t)grp * T + t) * F + f;
        a.out[o] = z;
        if (a.resid) a.resid[o] = csub(yr, z);
    }
}

template <int D>
static cudaError_t launch_blocks_d(const OnlineLengthsArgs& a, cudaStream_t st) {
    dim3 grid((a.in.F + 31) / 32, (a.J + kOnlineBY - 1) / kOnlineBY, a.in.n_grp), block(32, kOnlineBY);
    const OnlineArgs& u = a;   // the uniform kernels' parameters
    if (a.frames) scm_blocks_kernel<D, true><<<grid, block, 0, st>>>(a);
    else scm_blocks_kernel<D, false><<<grid, block, 0, st>>>(u);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t per_grp = (size_t)a.in.F * D * D;
    dim3 grid2((unsigned)((per_grp + 255) / 256), a.in.n_grp);
    if (a.frames) scm_combine_kernel<true><<<grid2, 256, 0, st>>>(a, D * D);
    else scm_combine_kernel<false><<<grid2, 256, 0, st>>>(u, D * D);
    return cudaGetLastError();
}

template <int D>
static cudaError_t launch_filter_d(const OnlineFilterArgs& a, cudaStream_t st) {
    dim3 grid((a.in.F + 31) / 32, (a.J + kOnlineBY - 1) / kOnlineBY, a.in.n_grp), block(32, kOnlineBY);
    if (a.frames) filter_sum_blocks_kernel<D, true><<<grid, block, 0, st>>>(a);
    else filter_sum_blocks_kernel<D, false><<<grid, block, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_scm_recursive(const OnlineLengthsArgs& a, cudaStream_t st) {
    switch (a.in.C + a.in.K - 1) {
        case 1: return launch_blocks_d<1>(a, st);
        case 2: return launch_blocks_d<2>(a, st);
        case 3: return launch_blocks_d<3>(a, st);
        case 4: return launch_blocks_d<4>(a, st);
        case 5: return launch_blocks_d<5>(a, st);
        case 6: return launch_blocks_d<6>(a, st);
        case 7: return launch_blocks_d<7>(a, st);
        case 8: return launch_blocks_d<8>(a, st);
        default: return launch_scm_recursive_wide(a, st);   // D = 9..16: online_wide.cu
    }
}

cudaError_t launch_filter_sum_blocks(const OnlineFilterArgs& a, cudaStream_t st) {
    switch (a.in.C + a.in.K - 1) {
        case 1: return launch_filter_d<1>(a, st);
        case 2: return launch_filter_d<2>(a, st);
        case 3: return launch_filter_d<3>(a, st);
        case 4: return launch_filter_d<4>(a, st);
        case 5: return launch_filter_d<5>(a, st);
        case 6: return launch_filter_d<6>(a, st);
        case 7: return launch_filter_d<7>(a, st);
        case 8: return launch_filter_d<8>(a, st);
        default: return launch_filter_sum_blocks_wide(a, st);
    }
}

// D = 9..16: the same block filter (its registers hold the D taps and one frame's D operands, no pairs)
cudaError_t launch_filter_sum_blocks_wide(const OnlineFilterArgs& a, cudaStream_t st) {
    switch (a.in.C + a.in.K - 1) {
        case 9: return launch_filter_d<9>(a, st);
        case 10: return launch_filter_d<10>(a, st);
        case 11: return launch_filter_d<11>(a, st);
        case 12: return launch_filter_d<12>(a, st);
        case 13: return launch_filter_d<13>(a, st);
        case 14: return launch_filter_d<14>(a, st);
        case 15: return launch_filter_d<15>(a, st);
        case 16: return launch_filter_d<16>(a, st);
        default: return cudaErrorNotSupported;
    }
}

}  // namespace disco
