// STFT and iSTFT of a batch of signals of different lengths held in rows of a common length L (disco_stft_lengths,
// disco_istft_lengths): what disco_stft / disco_istft give for each signal trimmed to its own length, in the shapes of
// the whole batch, with zeros past each signal's end.
//
//   stft_lengths   frame t < T_s = 1 + lengths[s] / hop of signal s is librosa's centred frame with reflect padding at
//                  that signal's start and end; frames T_s .. T - 1 are written as zero.  The FFT job, un-mixing,
//                  Nyquist bin and reflect fill of stft_core.cuh (shared with stft_scm.cu and stream.cu); one warp per
//                  job of NB = 32 / RA transforms, four jobs per CTA, grid signal pairs x frame groups.  Signals 2p and
//                  2p + 1 of the flattened list share one complex transform as in disco_stft (an odd last signal runs
//                  alone), so a frame equals disco_stft's of the trimmed signal bit for bit when its partner is the
//                  same trimmed signal; a partner that has already ended contributes zeros.
//   istft_lengths  istft.cu's istft_body, run per pair by istft_lengths_kernel (istft.cu) with each signal's own
//                  frame count and length; the chunk plan is disco_istft's for the longest signal.
#include "common.cuh"
#include "kernels.h"
#include "stft_core.cuh"

namespace disco {

constexpr int kLenWarps = 4;   // jobs per CTA

template <int N>
__global__ void __launch_bounds__(32 * kLenWarps) stft_lengths_kernel(StftLengthsArgs p) {
    using G = StftJob<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROWP = G::ROWP;
    __shared__ float2 scratch[kLenWarps][1056];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sa = 2 * blockIdx.y, sb = 2 * blockIdx.y + 1;
    const bool has_b = sb < p.n_sig;
    const int La = p.lengths[sa], Lb = has_b ? p.lengths[sb] : 0;
    const int Ta = 1 + La / H, Tb = has_b ? 1 + Lb / H : 0;
    const float* xa = p.x + (size_t)sa * p.L;
    const float* xb = p.x + (size_t)sb * p.L;
    // sample s of the padded signal x of length len: librosa center=True, pad_mode='reflect' (len > H, so every
    // reflected index of a frame t < 1 + len / H lies in [0, len))
    auto sample = [](const float* x, int len, int s) -> float { return x[reflect_index(s, len)]; };

    const int tj = (blockIdx.x * kLenWarps + warp) * NB;   // first frame of this warp's job
    if (tj >= p.T) return;                                 // warp-uniform; no CTA barrier follows
    float2* job = scratch[warp];
    constexpr bool TWREG = RA <= 16;   // inter-pass twiddles in registers, as in stft_scm.cu
    float2 twr[TWREG ? RA : 1];
    if (TWREG) {
#pragma unroll
        for (int k1 = 1; k1 < RA; ++k1) twr[k1] = p.twiddle[k1 * 32 + lane];
    }
#pragma unroll
    for (int q = 0; q < NB; ++q) {
        const int t = tj + q;
        const int s0 = t * H - H;                          // frame t reads samples [t H - H, t H + H)
        const bool va = t < Ta, vb = t < Tb;
        float2 v[RA];
        if (has_b && (va || vb)) {
#pragma unroll
            for (int j = 0; j < RA; ++j) {
                const float wj = p.window[lane + 32 * j];
                const int s = s0 + lane + 32 * j;
                v[j] = fmul2(make_float2(va ? sample(xa, La, s) : 0.f, vb ? sample(xb, Lb, s) : 0.f),
                             make_float2(wj, wj));
            }
        } else if (va) {
#pragma unroll
            for (int j = 0; j < RA; ++j) {
                const float wj = p.window[lane + 32 * j];
                v[j] = make_float2(sample(xa, La, s0 + lane + 32 * j) * wj, 0.f);
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
        const int t = tj + q;
        if (t >= p.T) break;
        const bool va = t < Ta, vb = t < Tb;
        const float2* row = job + q * ROWP;
        float2* ya = p.Y + ((size_t)sa * p.T + t) * F;
        float2* yb = p.Y + ((size_t)sb * p.T + t) * F;
        for (int f = lane; f < F; f += 32) {
            float2 za, zb;
            if (f < N / 2) {
                stft_unmix(row[f], row[(N - f) & (N - 1)], za, zb);
            } else {
                za = make_float2(stft_nyquist(row[N / 2], false), 0.f);
                zb = make_float2(stft_nyquist(row[N / 2], true), 0.f);
            }
            ya[f] = va ? za : make_float2(0.f, 0.f);
            if (has_b) yb[f] = vb ? zb : make_float2(0.f, 0.f);
        }
    }
}

template <int N>
static cudaError_t launch_stft_lengths_n(const StftLengthsArgs& a, cudaStream_t st) {
    const int per_cta = kLenWarps * StftJob<N>::NB;
    const int cols = (a.T + per_cta - 1) / per_cta;
    const int pairs = (a.n_sig + 1) / 2;
    // pairs sit in grid.y: launches of at most kMaxGridYZ pairs, each starting at an even signal
    for (int p0 = 0; p0 < pairs; p0 += kMaxGridYZ) {
        StftLengthsArgs b = a;
        const int s0 = 2 * p0;
        b.x = a.x + (size_t)s0 * a.L;
        b.lengths = a.lengths + s0;
        b.Y = a.Y + (size_t)s0 * a.T * (N / 2 + 1);
        b.n_sig = min(a.n_sig - s0, 2 * kMaxGridYZ);
        stft_lengths_kernel<N><<<dim3(cols, (b.n_sig + 1) / 2), 32 * kLenWarps, 0, st>>>(b);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

cudaError_t launch_stft_lengths(const StftLengthsArgs& a, int n_fft, cudaStream_t st) {
    if (a.n_sig <= 0) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_stft_lengths_n<256>(a, st);
        case 512: return launch_stft_lengths_n<512>(a, st);
        case 1024: return launch_stft_lengths_n<1024>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_istft_lengths(const IstftArgs& a0, const int* lengths, int n_fft, cudaStream_t st) {
    if (a0.n_sig <= 0) return cudaSuccess;
    const IstftLengthsKernel k = istft_lengths_kernel_for(n_fft);
    if (!k.fn) return cudaErrorInvalidValue;
    const int H = n_fft / 2, F = H + 1;
    IstftArgs a = a0;
    // the chunk plan of disco_istft for the longest signal (a.L): chunks past a shorter signal's frames return at once
    a.j_end = min(a.j_end, (a.L + n_fft + H - 1) / H);
    const int T_eff = a.j_end - a.j_begin;
    if (T_eff < 1) return cudaErrorInvalidValue;
    const int pairs = (a.n_sig + 1) / 2;
    int chunks = 1;
    while (pairs * chunks < sm_count() * 2 && (T_eff + chunks - 1) / chunks > 4 * k.items) chunks *= 2;
    a.fpc = ((T_eff + chunks - 1) / chunks + k.items - 1) / k.items * k.items;
    chunks = (T_eff + a.fpc - 1) / a.fpc;
    cudaError_t e = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    if (e != cudaSuccess) return e;
    for (int p0 = 0; p0 < pairs; p0 += kMaxGridYZ) {
        IstftArgs b = a;
        const int s0 = 2 * p0;
        b.Y = a.Y + (size_t)s0 * a.y_frames * F;
        b.x = a.x + (size_t)s0 * a.ld;
        b.n_sig = min(a.n_sig - s0, 2 * kMaxGridYZ);
        const int* len = lengths + s0;
        void* args[] = {&b, &len};
        e = cudaLaunchKernel(k.fn, dim3(chunks, (b.n_sig + 1) / 2), dim3(k.threads), args, k.smem, st);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

}  // namespace disco
