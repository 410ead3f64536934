// The forward STFT's arithmetic, shared by the fused STFT + SCM kernel (stft_scm.cu) and the streaming STFT
// (stream.cu), so that both give the same spectra value for value.
//
// Two real signals are transformed by one complex FFT of z = (a + i b) w / 2 (the window carries the 1/2).  A warp
// runs a JOB of NB = 32 / RA such transforms (RA = N / 32): per transform an RA-point in-register DFT per lane
// (pass 1), a padded transposition through a 32 x 33 shared scratch, then one 32-point in-register DFT per lane over
// all NB transforms (pass 2), which leaves the NB spectra in the scratch as rows of pitch ROWP.  The two real spectra
// are un-mixed per bin from Z[f] and Z[N - f].
#pragma once
#include "common.cuh"
#include "fft_reg.cuh"

namespace disco {

template <int N>
struct StftJob {
    static constexpr int RA = N / 32;       // radix of the per-lane first pass
    static constexpr int NB = 32 / RA;      // transforms per warp job
    static constexpr int H = N / 2;         // hop (50 % overlap)
    static constexpr int F = N / 2 + 1;     // bins
    static constexpr int ROWP = 1056 / NB;  // spectrum row pitch (complex): a job = 32 x 33 scratch
};

// Pass 1 of transform q of a job: v[j] holds the windowed pair at sample lane + 32 j.  The inter-pass twiddles
// W_N^(lane k1), k1 = 1 .. RA-1, come from twr[k1] (TWREG: held in registers across the job's transforms) or from the
// [RA][32] table tw.
template <int RA, bool TWREG>
DISCO_DEV void stft_pass1(float2 (&v)[RA], float2* job, int q, int lane, const float2 (&twr)[TWREG ? RA : 1],
                          const float2* tw) {
    dft_reg<RA, false>(v);
#pragma unroll
    for (int k1 = 1; k1 < RA; ++k1) v[k1] = cmul(v[k1], TWREG ? twr[k1] : tw[k1 * 32 + lane]);
#pragma unroll
    for (int k1 = 0; k1 < RA; ++k1) job[(q * RA + k1) * 33 + lane] = v[k1];   // scratch [32 rows][33]
}

// Pass 2 of a job, after pass 1 of all its NB transforms: spectrum q of the job at job + q * ROWP.
template <int RA>
DISCO_DEV void stft_pass2(float2* job, int lane) {
    constexpr int ROWP = StftJob<32 * RA>::ROWP;
    __syncwarp();
    float2 u[32];
#pragma unroll
    for (int l = 0; l < 32; ++l) u[l] = job[lane * 33 + l];
    __syncwarp();
    dft_reg<32, false>(u);
    float2* row = job + (lane / RA) * ROWP + (lane % RA);
#pragma unroll
    for (int k2 = 0; k2 < 32; ++k2) row[RA * k2] = u[k2];
}

// Un-mix the two-for-one spectra at bin f < N/2 from zf = Z[f], zn = Z[(N - f) mod N]:
//   A = Z[f] + conj(Z[N-f]),  B = -i (Z[f] - conj(Z[N-f]))
DISCO_DEV void stft_unmix(float2 zf, float2 zn, float2& a, float2& b) {
    a = fadd2(zf, make_float2(zn.x, -zn.y));
    b = fadd2(make_float2(zf.y, -zf.x), make_float2(zn.y, zn.x));
}
// At the Nyquist bin both spectra are real: A = 2 Re Z (second = 0), B = 2 Im Z (second = 1).
DISCO_DEV float stft_nyquist(float2 z, bool second) { return second ? z.y + z.y : z.x + z.x; }

// Sample index s of the padded signal of length L: librosa center=True, pad_mode='reflect' (an index still outside
// [0, L) afterwards, possible only for L <= N/2, reads as zero at the caller).  The end is mirrored as (L - 1) -
// (s - (L - 1)), not 2 (L - 1) - s, which would overflow int for L > 2^30 + 1.
DISCO_DEV int reflect_index(int s, int L) {
    if (s < 0) s = -s;
    if (s >= L) s = (L - 1) - (s - (L - 1));
    return s;
}

}  // namespace disco
