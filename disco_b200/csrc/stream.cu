// Streaming STFT of the online Tango session (disco_b200/stream.py): disco_stft evaluated on a signal that arrives
// chunk by chunk, so that a stream's spectra equal those of the whole-signal call value for value.  The stream's iSTFT
// is the whole-signal kernel of istft.cu, run on the new frames with a carried half frame (disco_stream_istft).
//
//   stream_stft    frames [t0, t0 + n_fr) of every signal, read in place from a carried history of the last N
//                  samples (samples [L0 - N, L0)) and the pushed chunk (samples [L0, length)).  librosa's reflect
//                  padding (center=True) applies at the start of the stream and, on the final call, at its end.
//                  Grid: signal pairs x groups of frames; a warp runs one job of NB = 32 / RA transforms, the FFT
//                  job, un-mixing and Nyquist bin of stft_scm.cu (stft_core.cuh).  The first CTA column also
//                  writes the history after the chunk (a separate buffer: the other CTAs still read the old one).
//
// It pairs signals 2p and 2p + 1 of the flattened signal list into one complex transform as disco_stft does (an odd
// last signal runs alone, with a zero imaginary part): the rounding of a two-for-one transform depends on its
// partner, so the pairing is part of the result.
#include "common.cuh"
#include "kernels.h"
#include "stft_core.cuh"

namespace disco {

constexpr int kStreamWarps = 4;   // jobs per CTA

template <int N>
__global__ void __launch_bounds__(32 * kStreamWarps) stream_stft_kernel(StreamStftArgs p) {
    using G = StftJob<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROWP = G::ROWP;
    __shared__ float2 scratch[kStreamWarps][1056];
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
        if (s >= L && !p.final_call) return 0.f;   // the end is mirrored only once the stream has ended
        s = reflect_index(s, L);
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
    const int tj = (blockIdx.x * kStreamWarps + warp) * NB;   // first frame (relative to t0) of this warp's job
    if (tj >= p.n_fr) return;                              // warp-uniform; no CTA barrier follows
    float2* job = scratch[warp];
    constexpr bool TWREG = RA <= 16;   // inter-pass twiddles in registers, as in stft_scm.cu
    float2 twr[TWREG ? RA : 1];
    if (TWREG) {
#pragma unroll
        for (int k1 = 1; k1 < RA; ++k1) twr[k1] = p.twiddle[k1 * 32 + lane];
    }
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
        stft_pass1<RA, TWREG>(v, job, q, lane, twr, p.twiddle);
    }
    stft_pass2<RA>(job, lane);
    __syncwarp();
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
                stft_unmix(row[f], row[(N - f) & (N - 1)], ya, yb);
            } else {
                ya = make_float2(stft_nyquist(row[N / 2], false), 0.f);
                yb = make_float2(stft_nyquist(row[N / 2], true), 0.f);
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
static cudaError_t launch_stft_n(const StreamStftArgs& a, cudaStream_t st) {
    const int per_cta = kStreamWarps * StftJob<N>::NB;
    const int cols = a.n_fr > 0 ? (a.n_fr + per_cta - 1) / per_cta : 1;
    dim3 grid(cols, (a.n_sig + 1) / 2);
    stream_stft_kernel<N><<<grid, 32 * kStreamWarps, 0, st>>>(a);
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

}  // namespace disco
