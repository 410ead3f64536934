// Single-node arrays (K = 1) with both masks known up front: BOTH filter-and-sum steps of Tango in
// one pass over Y.
//   z  = w1^H y,  zn = y[ref] - z        step 1, reference tango.py:369-376
//   yf = w2^H y                           step 2, reference tango.py:445-450 (no exchanged signals)
// With the two-mask fused STFT+SCM kernel (stft_scm.cu, NM = 2) this makes the whole K = 1 path
// read Y exactly once.  Frame-major data: a warp covers 32 consecutive bins of one frame (coalesced
// 8-byte loads and stores); each thread keeps its bin's 2 C filter taps in registers for all frames.
// out_ft = 1 writes the reference's (F, T) layout through 32 x 32 shared-memory transposes.
#include "common.cuh"
#include "kernels.h"

namespace disco {

// Two resident CTAs per SM (a third is 35 % slower on an H100), 4 frames per thread and register buffer, streaming
// stores for the three outputs: no other setting beat these by more than the run-to-run spread (DESIGN.md 4.1).
template <int C, bool OUT_FT>
__global__ void __launch_bounds__(256, 2) filter_dual_kernel(DualFilterArgs a, int frames_per_slab) {
    constexpr int TS = 8;                         // warps per block = time ways
    constexpr int UF = 4;                         // frames per thread and buffer
    __shared__ float2 tile[OUT_FT ? 3 : 1][OUT_FT ? 32 : 1][33];
    const int lane = threadIdx.x & 31, wrp = threadIdx.x >> 5;
    const int grp = blockIdx.y;
    const int T = a.T, F = a.F;
    const int f0 = blockIdx.x * 32;
    const int f = f0 + lane;
    const bool active = f < F;
    const int fc = active ? f : F - 1;
    if (!OUT_FT && !active) return;
    const int t_begin = blockIdx.z * frames_per_slab;
    const int t_end = min(T, t_begin + frames_per_slab);
    float2 w1[C], w2[C];
#pragma unroll
    for (int c = 0; c < C; ++c) {
        w1[c] = a.W1[((size_t)grp * F + fc) * C + c];
        w2[c] = a.W2[((size_t)grp * F + fc) * C + c];
    }
    const float2* y = a.Y + (size_t)grp * C * T * F + fc;
    const size_t cs = (size_t)T * F;
    const size_t go = (size_t)grp * T * F;

    // frame index of slot u of this thread in the block of frames starting at t
    auto frame = [&](int t, int u) { return OUT_FT ? t + wrp * UF + u : t + wrp + u * TS; };
    auto load = [&](int t, float2 (&x)[UF][C]) {
#pragma unroll
        for (int u = 0; u < UF; ++u) {
            const int tt = frame(t, u);
            const bool ok = tt < t_end;
#pragma unroll
            for (int c = 0; c < C; ++c) x[u][c] = ok ? ld_stream(y + c * cs + (size_t)tt * F) : make_float2(0.f, 0.f);
        }
    };
    auto emit = [&](int t, const float2 (&x)[UF][C]) {
#pragma unroll
        for (int u = 0; u < UF; ++u) {
            const int tt = frame(t, u);
            float2 z = make_float2(0.f, 0.f), yf = make_float2(0.f, 0.f);
#pragma unroll
            for (int c = 0; c < C; ++c) {
                z = cfma_cj(w1[c], x[u][c], z);
                yf = cfma_cj(w2[c], x[u][c], yf);
            }
            float2 r = x[u][0];
#pragma unroll
            for (int c = 1; c < C; ++c)
                if (c == a.ref) r = x[u][c];
            const float2 zn = csub(r, z);
            if (!OUT_FT) {
                if (tt < t_end) {
                    st_stream(a.z + go + (size_t)tt * F + f, z);
                    if (a.zn) st_stream(a.zn + go + (size_t)tt * F + f, zn);
                    st_stream(a.yf + go + (size_t)tt * F + f, yf);
                }
            } else {
                const int tl = wrp * UF + u;
                tile[0][tl][lane] = z;
                tile[1][tl][lane] = zn;
                tile[2][tl][lane] = yf;
            }
        }
        if (OUT_FT) {   // transposed write-out: lane <-> frame, (warp, i) <-> bin
            __syncthreads();
            const int tt = t + lane;
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int fl = wrp * 4 + i, ff = f0 + fl;
                if (ff < F && tt < t_end) {
                    const size_t o = ((size_t)grp * F + ff) * T + tt;
                    a.z[o] = tile[0][lane][fl];
                    if (a.zn) a.zn[o] = tile[1][lane][fl];
                    a.yf[o] = tile[2][lane][fl];
                }
            }
            __syncthreads();
        }
    };
    constexpr int STEP = UF * TS;                  // frames per block of the software pipeline (16 or 32)
    float2 xa[UF][C], xb[UF][C];
    int t = t_begin;
    load(t, xa);
    for (; t < t_end; t += 2 * STEP) {
        load(t + STEP, xb);
        emit(t, xa);
        if (t + STEP >= t_end) break;              // CTA-uniform
        load(t + 2 * STEP, xa);
        emit(t + STEP, xb);
    }
}

template <int C>
static cudaError_t launch_c(const DualFilterArgs& a, int sm, cudaStream_t st) {
    const int fblocks = (a.F + 31) / 32;
    // enough CTAs to fill the machine: split time into slabs when groups are few.  32 CTAs per SM: the CTAs are
    // equal-sized, so more waves make a shorter tail
    const int fps = filter_slab_frames(a.T, fblocks * a.n_grp, sm * 32);
    const int slabs = (a.T + fps - 1) / fps;
    if (a.n_grp > 65535 || slabs > 65535) return cudaErrorInvalidConfiguration;
    dim3 grid(fblocks, a.n_grp, slabs);
    if (a.out_ft)
        filter_dual_kernel<C, true><<<grid, 256, 0, st>>>(a, fps);
    else
        filter_dual_kernel<C, false><<<grid, 256, 0, st>>>(a, fps);
    return cudaGetLastError();
}

cudaError_t launch_filter_dual(const DualFilterArgs& a, int sm_count, cudaStream_t st) {
    switch (a.C) {
        case 1: return launch_c<1>(a, sm_count, st);
        case 2: return launch_c<2>(a, sm_count, st);
        case 3: return launch_c<3>(a, sm_count, st);
        case 4: return launch_c<4>(a, sm_count, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
