// Streaming STFT of the online Tango session (disco_b200/stream.py): disco_stft evaluated on a signal that arrives
// chunk by chunk, so that a stream's spectra equal those of the whole-signal call value for value.  The stream's iSTFT
// is the whole-signal kernel body of istft.cu, run on the new frames with a carried half frame (stream_istft_kernel).
//
//   stream_stft_kernel  frames [t0, t0 + n_fr) of every signal of a slot, read in place from a carried history of
//                  the last N samples (samples [L0 - N, L0)) and the pushed chunk (samples [L0, length)).  librosa's
//                  reflect padding (center=True) applies at the start of the stream and, on the final call, at its
//                  end.  Grid: groups of frames x signal pairs of a slot x slots; a warp runs one job of NB = 32 / RA
//                  transforms, the FFT job, un-mixing and Nyquist bin of stft_scm.cu (stft_core.cuh).  The first CTA
//                  column also writes the history after the chunk (to the other buffer: the other CTAs still read
//                  the old one).
//
// A slot's record comes from the device array `slots` (a pool, disco_stream_stft_slots) or, for a single lockstep
// stream (disco_stream_stft), is passed by value in the kernel parameters: the lockstep stream of n_sig signals is one
// slot of n_sig signals.  It pairs signals 2p and 2p + 1 of a slot into one complex transform as disco_stft does (an
// odd last signal runs alone, with a zero imaginary part): the rounding of a two-for-one transform depends on its
// partner, so the pairing is part of the result.
#include "common.cuh"
#include "kernels.h"
#include "stft_core.cuh"

namespace disco {

constexpr int kStreamWarps = 4;   // jobs per CTA

// Slot blockIdx.z: its signals are rows [z n_sig, (z + 1) n_sig) of every buffer, the chunk rows are n_max floats
// apart and the frame rows of Y f_max frames apart.  History buffer hist_sel is read; with hist_write the samples
// [length - N, length) go to the other one.
template <int N>
__global__ void __launch_bounds__(32 * kStreamWarps) stream_stft_kernel(StreamStftArgs p) {
    using G = StftJob<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROWP = G::ROWP;
    __shared__ float2 scratch[kStreamWarps][1056];
    StftSlot r = p.one;
    if (p.slots) r = p.slots[blockIdx.z];
    const int L = r.length, n_new = r.n_new, t0 = r.t0, n_fr = r.n_fr, blk_slot = r.blk_slot;
    const int final_call = r.final_call, sel = r.hist_sel, write = r.hist_write;
    if (n_fr <= 0 && !write) return;   // CTA-uniform: nothing of this slot changes in this call
    const size_t row0 = (size_t)blockIdx.z * p.n_sig;
    float* const h0 = p.hist[0];
    float* const h1 = p.hist[1];
    const float* hist = (sel ? h1 : h0) + row0 * N;
    float* hist_out = write ? (sel ? h0 : h1) + row0 * N : nullptr;
    const float* chunk = p.chunk + row0 * p.n_max;
    float2* Y = p.Y + row0 * p.f_max * F;
    float2* Y_blk = p.Y_blk ? p.Y_blk + row0 * p.blk_frames * F : nullptr;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sa = 2 * blockIdx.y, sb = 2 * blockIdx.y + 1;
    const bool has_b = sb < p.n_sig;
    const int L0 = L - n_new;
    // sample s (absolute index, [L0 - N, L)) of signal sig as it stands in memory
    auto raw = [&](int sig, int s) -> float {
        return s >= L0 ? chunk[(size_t)sig * p.n_max + (s - L0)] : hist[(size_t)sig * N + (s - (L0 - N))];
    };
    // sample s of the padded signal: librosa center=True, pad_mode='reflect' (stft_scm.cu, edge-tile fill)
    auto sample = [&](int sig, int s) -> float {
        if (s >= L && !final_call) return 0.f;   // the end is mirrored only once the stream has ended
        s = reflect_index(s, L);
        if (s < 0 || s >= L || s < L0 - N) return 0.f;   // not reached for frames the host declares complete
        return raw(sig, s);
    };

    if (hist_out && blockIdx.x == 0) {   // history after the chunk: samples [L - N, L)
        for (int i = threadIdx.x; i < N; i += blockDim.x) {
            const int s = L - N + i;
            hist_out[(size_t)sa * N + i] = s >= 0 ? raw(sa, s) : 0.f;
            if (has_b) hist_out[(size_t)sb * N + i] = s >= 0 ? raw(sb, s) : 0.f;
        }
    }
    const int tj = (blockIdx.x * kStreamWarps + warp) * NB;   // first frame (relative to t0) of this warp's job
    if (tj >= n_fr) return;                              // warp-uniform; no CTA barrier follows
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
        const int s0 = (t0 + tl) * H - H;                // frame t reads samples [t H - H, t H + H)
        float2 v[RA];
#pragma unroll
        for (int j = 0; j < RA; ++j) {
            const float wj = p.window[lane + 32 * j];
            if (tl >= n_fr) v[j] = make_float2(0.f, 0.f);
            else if (has_b) v[j] = fmul2(make_float2(sample(sa, s0 + lane + 32 * j), sample(sb, s0 + lane + 32 * j)),
                                         make_float2(wj, wj));
            else v[j] = make_float2(sample(sa, s0 + lane + 32 * j) * wj, 0.f);
        }
        stft_pass1<RA, TWREG>(v, job, q, lane, twr, p.twiddle);
    }
    stft_pass2<RA>(job, lane);
    __syncwarp();
#pragma unroll
    for (int q = 0; q < NB; ++q) {
        const int tl = tj + q;
        if (tl >= n_fr) break;
        const float2* row = job + q * ROWP;
        const size_t oa = ((size_t)sa * p.f_max + tl) * F, ob = ((size_t)sb * p.f_max + tl) * F;
        const size_t ba = ((size_t)sa * p.blk_frames + blk_slot + tl) * F;
        const size_t bb = ((size_t)sb * p.blk_frames + blk_slot + tl) * F;
        for (int f = lane; f < F; f += 32) {
            float2 ya, yb;
            if (f < N / 2) {
                stft_unmix(row[f], row[(N - f) & (N - 1)], ya, yb);
            } else {
                ya = make_float2(stft_nyquist(row[N / 2], false), 0.f);
                yb = make_float2(stft_nyquist(row[N / 2], true), 0.f);
            }
            Y[oa + f] = ya;
            if (Y_blk) Y_blk[ba + f] = ya;
            if (has_b) {
                Y[ob + f] = yb;
                if (Y_blk) Y_blk[bb + f] = yb;
            }
        }
    }
}

// a.f_max: the most frames of any slot (the grid covers it)
template <int N>
static cudaError_t launch_stft_slots_n(const StreamStftArgs& a, cudaStream_t st) {
    const int per_cta = kStreamWarps * StftJob<N>::NB;
    const int cols = a.f_max > 0 ? (a.f_max + per_cta - 1) / per_cta : 1;
    dim3 grid(cols, (a.n_sig + 1) / 2, a.n_slot);
    stream_stft_kernel<N><<<grid, 32 * kStreamWarps, 0, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_stream_stft_slots(const StreamStftArgs& a, int n_fft, cudaStream_t st) {
    if (a.n_slot <= 0 || (!a.slots && a.one.n_fr <= 0 && !a.one.hist_write)) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_stft_slots_n<256>(a, st);
        case 512: return launch_stft_slots_n<512>(a, st);
        case 1024: return launch_stft_slots_n<1024>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
