// Streaming STFT and iSTFT of the online Tango session (disco_b200/stream.py): the transforms of disco_stft and
// disco_istft evaluated on a signal that arrives chunk by chunk, with the same arithmetic in the same order, so that
// a stream's spectra and time samples equal those of the whole-signal calls value for value.
//
//   stream_stft    frames [t0, t0 + n_fr) of every signal, read in place from a carried history of the last N
//                  samples (samples [L0 - N, L0)) and the pushed chunk (samples [L0, length)).  librosa's reflect
//                  padding (center=True) applies at the start of the stream and, on the final call, at its end.
//                  Grid: signal pairs x groups of frames; a warp runs one job of NB = 32 / RA transforms, as an FFT
//                  warp of stft_scm.cu does (kernel body: stft_scm.cu run_job + the SCM warps' un-mixing + the
//                  loader's Nyquist bin).  The first CTA column also writes the history after the chunk
//                  (a separate buffer: the other CTAs still read the old one).
//   stream_istft   the hop blocks of the new frames, with the windowed second half of the previous frame carried in
//                  a [n_sig][H] buffer between calls; the final call adds the tail block and the zero fill up to the
//                  length.  Kernel body: istft.cu, one CTA per signal pair.
//
// Both pair signals 2p and 2p + 1 of the flattened signal list into one complex transform as disco_stft and
// disco_istft do (an odd last signal runs alone, with a zero imaginary part): the rounding of a two-for-one
// transform depends on its partner, so the pairing is part of the result.  The FFT sequence is restated here
// rather than shared with stft_scm.cu and istft.cu, whose machine code stays as it is.
#include "common.cuh"
#include "fft_reg.cuh"
#include "kernels.h"

namespace disco {

template <int N>
struct StreamStftGeom {
    static constexpr int RA = N / 32, NB = 32 / RA, H = N / 2, F = N / 2 + 1;
    static constexpr int ROWP = 1056 / NB;   // spectrum row pitch of a job's 32 x 33 scratch (stft_scm.cu)
    static constexpr int WARPS = 4;          // jobs per CTA
};

template <int N>
__global__ void __launch_bounds__(32 * StreamStftGeom<N>::WARPS) stream_stft_kernel(StreamStftArgs p) {
    using G = StreamStftGeom<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROWP = G::ROWP;
    __shared__ float2 scratch[G::WARPS][1056];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sa = 2 * blockIdx.y, sb = 2 * blockIdx.y + 1;
    const bool has_b = sb < p.n_sig;
    const int L = p.length, L0 = p.length - p.n_new;
    // sample s (absolute index, [L0 - N, L)) of signal sig as it stands in memory
    auto raw = [&](int sig, int s) -> float {
        return s >= L0 ? p.chunk[(size_t)sig * p.n_new + (s - L0)] : p.hist[(size_t)sig * N + (s - (L0 - N))];
    };
    // sample s of the padded signal: librosa center=True, pad_mode='reflect' (stft_scm.cu, edge-tile fill)
    auto sample = [&](int sig, int s) -> float {
        if (s < 0) s = -s;
        if (p.final_call && s >= L) s = 2 * (L - 1) - s;
        if (s < 0 || s >= L || s < L0 - N) return 0.f;   // not reached for frames the host declares complete
        return raw(sig, s);
    };

    if (p.hist_out && blockIdx.x == 0) {   // history after the chunk: samples [L - N, L)
        for (int i = threadIdx.x; i < N; i += blockDim.x) {
            const int s = L - N + i;
            p.hist_out[(size_t)sa * N + i] = s >= 0 ? raw(sa, s) : 0.f;
            if (has_b) p.hist_out[(size_t)sb * N + i] = s >= 0 ? raw(sb, s) : 0.f;
        }
    }
    const int tj = (blockIdx.x * G::WARPS + warp) * NB;   // first frame (relative to t0) of this warp's job
    if (tj >= p.n_fr) return;                              // warp-uniform; no CTA barrier follows
    float2* job = scratch[warp];
#pragma unroll
    for (int q = 0; q < NB; ++q) {
        const int tl = tj + q;
        const int s0 = (p.t0 + tl) * H - H;                // frame t reads samples [t H - H, t H + H)
        float2 v[RA];
        if (tl < p.n_fr && has_b) {
#pragma unroll
            for (int j = 0; j < RA; ++j) {
                const float wj = p.window[lane + 32 * j];
                v[j] = fmul2(make_float2(sample(sa, s0 + lane + 32 * j), sample(sb, s0 + lane + 32 * j)),
                             make_float2(wj, wj));
            }
        } else if (tl < p.n_fr) {
#pragma unroll
            for (int j = 0; j < RA; ++j) {
                const float wj = p.window[lane + 32 * j];
                v[j] = make_float2(sample(sa, s0 + lane + 32 * j) * wj, 0.f);
            }
        } else {
#pragma unroll
            for (int j = 0; j < RA; ++j) v[j] = make_float2(0.f, 0.f);
        }
        dft_reg<RA, false>(v);
#pragma unroll
        for (int k1 = 1; k1 < RA; ++k1) v[k1] = cmul(v[k1], p.twiddle[k1 * 32 + lane]);
#pragma unroll
        for (int k1 = 0; k1 < RA; ++k1) job[(q * RA + k1) * 33 + lane] = v[k1];   // scratch [32 rows][33]
    }
    __syncwarp();
    float2 u[32];
#pragma unroll
    for (int l = 0; l < 32; ++l) u[l] = job[lane * 33 + l];
    __syncwarp();
    dft_reg<32, false>(u);
    {
        float2* row = job + (lane / RA) * ROWP + (lane % RA);
#pragma unroll
        for (int k2 = 0; k2 < 32; ++k2) row[RA * k2] = u[k2];
    }
    __syncwarp();
    // un-mix the two-for-one spectra (the window carries the 1/2):
    //   A = Z[f] + conj(Z[N-f]),  B = -i (Z[f] - conj(Z[N-f]));  at the Nyquist bin A = 2 Re Z, B = 2 Im Z (real)
#pragma unroll
    for (int q = 0; q < NB; ++q) {
        const int tl = tj + q;
        if (tl >= p.n_fr) break;
        const float2* row = job + q * ROWP;
        const size_t oa = ((size_t)sa * p.n_fr + tl) * F, ob = ((size_t)sb * p.n_fr + tl) * F;
        const size_t ba = ((size_t)sa * p.blk_frames + p.blk_slot + tl) * F;
        const size_t bb = ((size_t)sb * p.blk_frames + p.blk_slot + tl) * F;
        for (int f = lane; f < F; f += 32) {
            float2 ya, yb;
            if (f < N / 2) {
                const float2 zf = row[f], zn = row[(N - f) & (N - 1)];
                ya = fadd2(zf, make_float2(zn.x, -zn.y));
                yb = fadd2(make_float2(zf.y, -zf.x), make_float2(zn.y, zn.x));
            } else {
                const float2 z = row[N / 2];
                ya = make_float2(z.x + z.x, 0.f);
                yb = make_float2(z.y + z.y, 0.f);
            }
            p.Y[oa + f] = ya;
            if (p.Y_blk) p.Y_blk[ba + f] = ya;
            if (has_b) {
                p.Y[ob + f] = yb;
                if (p.Y_blk) p.Y_blk[bb + f] = yb;
            }
        }
    }
}

template <int N>
struct StreamIstftGeom {   // = IGeom of istft.cu
    static constexpr int RA = N / 32, NB = 32 / RA, H = N / 2, F = N / 2 + 1;
    static constexpr int ROW = N + (RA == 8 ? 8 : 0);
    static constexpr int FFT_WARPS = N / 64;
    static constexpr int THREADS = N / 2 + 32;
    static constexpr int ITEMS = 16;
};

template <int N>
__global__ void __launch_bounds__(StreamIstftGeom<N>::THREADS) stream_istft_kernel(StreamIstftArgs p) {
    using G = StreamIstftGeom<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROW = G::ROW, TT = G::ITEMS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2* rows = reinterpret_cast<float2*>(smem_raw);    // [TT][ROW]
    float2* carry = rows + TT * ROW;                       // [H] second half of the previous frame (windowed)
    float2* tw = carry + H;                                // [RA][32]
    float* win = reinterpret_cast<float*>(tw + N);         // [N]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int sa = 2 * blockIdx.x, sb = 2 * blockIdx.x + 1;
    const bool has_b = sb < p.n_sig;
    const int n_fr = p.n_fr, L = p.length;
    // spectra and outputs are addressed from the parameter block at each use: held in registers across the
    // 1024-point transform, the four row pointers would spill
    auto Ya = [&](size_t off) { return p.Y[(size_t)sa * n_fr * F + off]; };
    auto Yb = [&](size_t off) { return p.Y[(size_t)sb * n_fr * F + off]; };
    auto xa = [&](int s) -> float& { return p.x[(size_t)sa * p.ld + (s - p.x_first)]; };
    auto xb = [&](int s) -> float& { return p.x[(size_t)sb * p.ld + (s - p.x_first)]; };

    for (int i = tid; i < N; i += blockDim.x) {
        tw[i] = p.twiddle[i];
        win[i] = p.window[i];
    }
    if (tid < H) carry[tid] = make_float2(p.carry[(size_t)sa * H + tid], has_b ? p.carry[(size_t)sb * H + tid] : 0.f);
    __syncthreads();
    const float inv_n = 1.0f / (float)N;
    const float tiny = 1.17549435e-38f;

    for (int c0 = 0; c0 < n_fr; c0 += TT) {
        const int nfr = min(TT, n_fr - c0);
        // ---- 1. gather the two half spectra into one full complex spectrum per frame
        if (tid < F) {
            const int f = tid;
            for (int tl = 0; tl < nfr; ++tl) {
                const size_t off = (size_t)(c0 + tl) * F + f;
                float2 A = Ya(off);
                float2 B = has_b ? Yb(off) : make_float2(0.f, 0.f);
                float2* row = rows + tl * ROW;
                if (f == 0 || f == N / 2) {
                    row[f] = make_float2(A.x, B.x);  // irfft ignores the imaginary part of DC / Nyquist
                } else {
                    row[f] = make_float2(A.x - B.y, A.y + B.x);
                    row[N - f] = make_float2(A.x + B.y, B.x - A.y);
                }
            }
        }
        __syncthreads();
        // ---- 2. inverse FFT, in place in the rows
        if (warp < G::FFT_WARPS) {
            float2* job = rows + (size_t)warp * NB * ROW;
            float2 v[NB][RA];
#pragma unroll
            for (int q = 0; q < NB; ++q)
#pragma unroll
                for (int j = 0; j < RA; ++j) v[q][j] = job[q * ROW + lane + 32 * j];
            __syncwarp();
#pragma unroll
            for (int q = 0; q < NB; ++q) {
                dft_reg<RA, true>(v[q]);
#pragma unroll
                for (int k1 = 0; k1 < RA; ++k1) {
                    float2 val = (k1 == 0) ? v[q][0] : cmul(v[q][k1], cconj(tw[k1 * 32 + lane]));
                    const int m = q * RA + k1;
                    job[m * 32 + ((lane + m) & 31)] = val;
                }
            }
            __syncwarp();
            const int m = lane, qq = m / RA, k1 = m % RA;
            float2 u[32];
#pragma unroll
            for (int l = 0; l < 32; ++l) u[l] = job[m * 32 + ((l + m) & 31)];
            __syncwarp();
            dft_reg<32, true>(u);
            float2* row = job + qq * ROW + k1;
#pragma unroll
            for (int k2 = 0; k2 < 32; ++k2) row[RA * k2] = u[k2];
        }
        __syncthreads();
        // ---- 3. overlap-add: thread n <-> sample offset n inside a hop block
        if (tid < H) {
            const int n = tid;
            const float w0 = win[n], w1 = win[n + H];
            float2 prev = carry[n];
            for (int tl = 0; tl < nfr; ++tl) {
                const int j = p.t0 + c0 + tl;        // frame j, hop block j
                const float2 cur = rows[tl * ROW + n];
                const float2 nxt = rows[tl * ROW + n + H];
                float2 val = cadd(cscale(cur, w0 * inv_n), prev);
                const float wss = w0 * w0 + (j >= 1 ? w1 * w1 : 0.f);
                if (wss > tiny) val = cscale(val, 1.0f / wss);
                const int s = (j - 1) * H + n;
                if (s >= 0 && s < L) {
                    xa(s) = val.x;
                    if (has_b) xb(s) = val.y;
                }
                prev = cscale(nxt, w1 * inv_n);
            }
            carry[n] = prev;
        }
        __syncthreads();
    }
    if (tid < H) {
        p.carry[(size_t)sa * H + tid] = carry[tid].x;
        if (has_b) p.carry[(size_t)sb * H + tid] = carry[tid].y;
    }
    // ---- final call: block T has only the second half of the last frame; then zero-fill up to L
    if (p.final_call) {
        const int T = p.t0 + n_fr;
        if (tid < H) {
            const int n = tid;
            const float w1 = win[n + H];
            float2 val = carry[n];
            const float wss = w1 * w1;
            if (wss > tiny) val = cscale(val, 1.0f / wss);
            const int s = (T - 1) * H + n;
            if (s >= 0 && s < L) {
                xa(s) = val.x;
                if (has_b) xb(s) = val.y;
            }
        }
        for (int s = T * H + tid; s < L; s += blockDim.x) {
            xa(s) = 0.f;
            if (has_b) xb(s) = 0.f;
        }
    }
}

template <int N>
static cudaError_t launch_stft_n(const StreamStftArgs& a, cudaStream_t st) {
    using G = StreamStftGeom<N>;
    const int per_cta = G::WARPS * G::NB;
    const int cols = a.n_fr > 0 ? (a.n_fr + per_cta - 1) / per_cta : 1;
    dim3 grid(cols, (a.n_sig + 1) / 2);
    stream_stft_kernel<N><<<grid, 32 * G::WARPS, 0, st>>>(a);
    return cudaGetLastError();
}

template <int N>
static cudaError_t launch_istft_n(const StreamIstftArgs& a, cudaStream_t st) {
    using G = StreamIstftGeom<N>;
    const size_t smem = (size_t)G::ITEMS * G::ROW * sizeof(float2) + G::H * sizeof(float2) + N * sizeof(float2) +
                        N * sizeof(float);
    auto kern = stream_istft_kernel<N>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<(a.n_sig + 1) / 2, G::THREADS, smem, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_stream_stft(const StreamStftArgs& a, int n_fft, cudaStream_t st) {
    if (a.n_fr <= 0 && !a.hist_out) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_stft_n<256>(a, st);
        case 512: return launch_stft_n<512>(a, st);
        case 1024: return launch_stft_n<1024>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_stream_istft(const StreamIstftArgs& a, int n_fft, cudaStream_t st) {
    if (a.n_fr <= 0 && !a.final_call) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_istft_n<256>(a, st);
        case 512: return launch_istft_n<512>(a, st);
        case 1024: return launch_istft_n<1024>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
