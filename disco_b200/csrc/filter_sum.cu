// Complex filter-and-sum: out[g][t][f] = sum_d conj(w[g][f][d]) * x_d[g][t][f]  (w^H x), optionally
// the residual x_ref - out.  Replaces the per-(f, t) np.inner calls of the reference
// (tango.py:369-376 for step 1, :445-450 for step 2) for a whole batch in one launch.
//
// The D input channels are the "concatenated" view of CatArgs (own microphones, then the
// compressed signals of the other nodes), so step 2 never materialises the concatenation.
// Frame-major data: a warp covers 32 consecutive bins of one frame (coalesced 8-byte loads and
// stores); each thread keeps its bin's D filter taps in registers for all frames.
// out_ft = 1 writes the reference's (F, T) layout through a 32x32 shared-memory transpose.
#include "common.cuh"
#include "kernels.h"

namespace disco {

template <int D>
__global__ void __launch_bounds__(256) filter_sum_kernel(FilterArgs a, int frames_per_slab) {
    __shared__ float2 tile_o[32][33];
    __shared__ float2 tile_r[32][33];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int grp = blockIdx.y;
    const int f0 = blockIdx.x * 32;
    const int f = f0 + lane;
    const int T = a.in.T, F = a.in.F;
    const bool active = f < F;
    const int fc = active ? f : F - 1;
    const int t_begin = blockIdx.z * frames_per_slab;
    const int t_end = min(T, t_begin + frames_per_slab);

    float2 w[D];
    const float2* ch[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float2 v = a.W[((size_t)grp * F + fc) * D + d];
        w[d] = a.conj_w ? cconj(v) : v;
        ch[d] = cat_channel(a.in, grp, d) + fc;
    }
    const float2* refch = cat_channel(a.in, grp, a.ref) + fc;

    // Software pipeline (small D): the 4 frames this warp owns in the NEXT 32-frame tile are loaded
    // before the current ones are consumed, keeping 4 D loads per thread in flight.
    constexpr bool PF = (D <= 5);
    float2 nx[PF ? 4 : 1][D];
    float2 nr[PF ? 4 : 1];
    auto fetch = [&](int t0) {
        if (PF) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int t = t0 + wrp * 4 + i;
                const bool ok = t < t_end;
#pragma unroll
                for (int d = 0; d < D; ++d) nx[i][d] = ok ? ch[d][(size_t)t * F] : make_float2(0.f, 0.f);
                nr[i] = (ok && a.resid) ? refch[(size_t)t * F] : make_float2(0.f, 0.f);
            }
        }
    };
    fetch(t_begin);
    for (int t0 = t_begin; t0 < t_end; t0 += 32) {
        float2 cx[4][D], cr[4];
        if (PF) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
#pragma unroll
                for (int d = 0; d < D; ++d) cx[i][d] = nx[i][d];
                cr[i] = nr[i];
            }
            fetch(t0 + 32);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int tl = wrp * 4 + i, t = t0 + tl;
            float2 acc = make_float2(0.f, 0.f), r = make_float2(0.f, 0.f);
            if (t < t_end) {
                if (!PF) {
#pragma unroll
                    for (int d = 0; d < D; ++d) cx[i][d] = ch[d][(size_t)t * F];
                    cr[i] = a.resid ? refch[(size_t)t * F] : make_float2(0.f, 0.f);
                }
#pragma unroll
                for (int d = 0; d < D; ++d) acc = cfma(w[d], cx[i][d], acc);
                if (a.resid) r = csub(cr[i], acc);
                if (!a.out_ft && active) {
                    a.out[((size_t)grp * T + t) * F + f] = acc;
                    if (a.resid) a.resid[((size_t)grp * T + t) * F + f] = r;
                }
            }
            if (a.out_ft) {
                tile_o[tl][lane] = acc;
                tile_r[tl][lane] = r;
            }
        }
        if (a.out_ft) {
            __syncthreads();
            const int t = t0 + lane;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int fl = wrp * 4 + i, ff = f0 + fl;
                if (ff < F && t < t_end) {
                    a.out[((size_t)grp * F + ff) * T + t] = tile_o[lane][fl];
                    if (a.resid) a.resid[((size_t)grp * F + ff) * T + t] = tile_r[lane][fl];
                }
            }
            __syncthreads();
        }
    }
}

// Frame-major output (the pipeline's internal layout): pure streaming.  Thread (bin, way) handles frames
// way, way + 8, ...; two register buffers of UF frames each are used alternately so UF * D loads per
// thread are always in flight; FC > 0 makes the row stride a compile-time constant (F = 257).
template <int D, int FC>
__global__ void __launch_bounds__(256, (D <= 4 ? 2 : 1)) filter_sum_tf_kernel(FilterArgs a, int frames_per_slab) {
    constexpr int UF = (D <= 4) ? 2 : 1;
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int grp = blockIdx.y;
    const int T = a.in.T, F = FC ? FC : a.in.F;
    const int f = blockIdx.x * 32 + lane;
    if (f >= F) return;
    const int t_begin = blockIdx.z * frames_per_slab;
    const int t_end = min(T, t_begin + frames_per_slab);
    float2 w[D];
    const float2* ch[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        const float2 v = a.W[((size_t)grp * F + f) * D + d];
        w[d] = a.conj_w ? cconj(v) : v;
        ch[d] = cat_channel(a.in, grp, d) + f;
    }
    const float2* refch = cat_channel(a.in, grp, a.ref) + f;
    float2* out = a.out + (size_t)grp * T * F + f;
    float2* res = a.resid ? a.resid + (size_t)grp * T * F + f : nullptr;
    constexpr int TS = 8;                         // warps per block = time ways
    auto load = [&](int t, float2 (&x)[UF][D], float2 (&r)[UF]) {
#pragma unroll
        for (int u = 0; u < UF; ++u) {
            const int tt = t + u * TS;
            const bool ok = tt < t_end;
#pragma unroll
            for (int d = 0; d < D; ++d) x[u][d] = ok ? ch[d][tt * F] : make_float2(0.f, 0.f);
            r[u] = (ok && res) ? refch[tt * F] : make_float2(0.f, 0.f);
        }
    };
    auto emit = [&](int t, const float2 (&x)[UF][D], const float2 (&r)[UF]) {
#pragma unroll
        for (int u = 0; u < UF; ++u) {
            const int tt = t + u * TS;
            if (tt < t_end) {
                float2 acc = cfma(w[0], x[u][0], make_float2(0.f, 0.f));
#pragma unroll
                for (int d = 1; d < D; ++d) acc = cfma(w[d], x[u][d], acc);
                out[tt * F] = acc;
                if (res) res[tt * F] = csub(r[u], acc);
            }
        }
    };
    float2 xa[UF][D], xb[UF][D], ra[UF], rb[UF];
    int t = t_begin + wrp;
    load(t, xa, ra);
    for (; t < t_end; t += 2 * UF * TS) {
        load(t + UF * TS, xb, rb);
        emit(t, xa, ra);
        load(t + 2 * UF * TS, xa, ra);
        emit(t + UF * TS, xb, rb);
    }
}

template <int D>
static cudaError_t launch_d(const FilterArgs& a, cudaStream_t st) {
    const int fblocks = (a.in.F + 31) / 32;
    // enough CTAs to fill the machine (4 per SM): split time into slabs when groups are few
    const int fps = filter_slab_frames(a.in.T, fblocks * a.in.n_grp, sm_count() * 4);
    const int slabs = (a.in.T + fps - 1) / fps;
    dim3 grid(fblocks, a.in.n_grp, slabs);
    if (!a.out_ft) {
        if (D <= 4 && a.in.F == 257)
            filter_sum_tf_kernel<D, (D <= 4 ? 257 : 0)><<<grid, 256, 0, st>>>(a, fps);
        else
            filter_sum_tf_kernel<D, 0><<<grid, 256, 0, st>>>(a, fps);
    } else {
        filter_sum_kernel<D><<<grid, 256, 0, st>>>(a, fps);
    }
    return cudaGetLastError();
}

cudaError_t launch_filter_sum(const FilterArgs& a, cudaStream_t st) {
    const int D = a.in.C + a.in.K - 1;
    {   // all nodes of a multi-node array, frame-major output: one pass over Y and Z (filter_sum_multi.cu)
        const cudaError_t e = launch_filter_sum_multi(a, st);
        if (e != cudaErrorNotSupported) return e;
    }
    switch (D) {
        case 1: return launch_d<1>(a, st);
        case 2: return launch_d<2>(a, st);
        case 3: return launch_d<3>(a, st);
        case 4: return launch_d<4>(a, st);
        case 5: return launch_d<5>(a, st);
        case 6: return launch_d<6>(a, st);
        case 7: return launch_d<7>(a, st);
        case 8: return launch_d<8>(a, st);
        case 9: return launch_d<9>(a, st);
        case 10: return launch_d<10>(a, st);
        case 11: return launch_d<11>(a, st);
        case 12: return launch_d<12>(a, st);
        case 13: return launch_d<13>(a, st);
        case 14: return launch_d<14>(a, st);
        case 15: return launch_d<15>(a, st);
        case 16: return launch_d<16>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
