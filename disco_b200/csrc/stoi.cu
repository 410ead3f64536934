// Classic STOI (pystoi 0.3, pystoi.stoi.stoi(x, y, fs_sig); the intelligibility scores of the reference's tango.main,
// disco_theque/speech_enhancement/tango.py:569-578) in float64 on the FP64 pipe, and the polyphase resampler that
// brings a signal to STOI's 10 kHz.
//
//   resample_poly_kernel  one thread per output sample: scipy.signal.resample_poly(x, up, down, window=taps), i.e.
//                         y[j] = sum_n x[n] up h[(j + pre_remove) down - pre_pad - n up] with scipy's zero pre-pad
//                         that centres the output and its length ceil(n_in up / down).
//   stoi_select_kernel    one CTA per clean: the energies 20 log10(‖w x_f‖ + eps) of the frames starting every 128
//                         samples, their maximum, the 40 dB mask and an in-order scan to the kept-frame list.
//   stoi_bands_kernel     one warp per (spectrogram, STFT frame).  Sample n of the overlap-added signal of the kept
//                         frames is the sum of at most two kept frames, so STFT frame t gathers kept frames t - 1 .. t + 1
//                         through the kept-frame list and nothing compacted is materialised.  A 512-point radix-2 FFT in
//                         shared memory (float64 twiddles), then the 15 band values sqrt(sum |X_k|^2).  A spectrogram is
//                         a clean under its own selection, or a pair's degraded signal under the pair's clean's selection.
//   stoi_score_kernel     one CTA per pair: every (30-frame segment, band) item's clipped, normalised correlation, summed
//                         per thread in item order and then over a fixed tree.
//
// No atomics: every value depends on its own signals only, never on the position in the batch.
#include <math.h>

#include "kernels.h"

namespace disco {

namespace {

constexpr double kEps = 2.220446049250313e-16;      // np.finfo(float).eps
constexpr double kClip = 6.623413251903491;         // 1 + 10^(-BETA / 20), BETA = -15 dB, as Python rounds it
constexpr double kDynRange = 40.0;
constexpr int kHop = kStoiFrame / 2;
constexpr int kNfft = 512;
// band i sums the bins kStoiEdges[i] <= k < kStoiEdges[i + 1] (pystoi's thirdoct at 10 kHz, 512 points, from 150 Hz)
__constant__ int kStoiEdges[kStoiBands + 1] = {7, 9, 11, 14, 17, 22, 27, 34, 43, 55, 69, 87, 109, 138, 174, 219};

// np.hanning(258)[1:-1][n] = 0.5 + 0.5 cos(pi (2 n - 255) / 257)
__device__ __forceinline__ double stoi_hann(int n) { return 0.5 + 0.5 * cospi((double)(2 * n - 255) / 257.0); }

__host__ __device__ __forceinline__ int stoi_frames(int L) { return L < kStoiFrame ? 0 : (L - kStoiFrame) / kHop + 1; }

__device__ __forceinline__ long long floor_div(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

__global__ void __launch_bounds__(256) resample_poly_kernel(ResampleArgs a, int blocks_per_sig) {
    const int sig = blockIdx.x / blocks_per_sig;
    const long long j = (long long)(blockIdx.x % blocks_per_sig) * blockDim.x + threadIdx.x;
    if (j >= a.n_out) return;
    // a signal of its own length n_in_s <= n_in: output samples from ceil(n_in_s up / down) on are 0
    const long long n_in_s = a.lengths ? a.lengths[sig] : a.n_in;
    if (a.lengths && j >= (n_in_s * a.up + a.down - 1) / a.down) {
        a.y[(size_t)sig * a.n_out + j] = 0.0;
        return;
    }
    const int half = (a.n_taps - 1) / 2;
    const int pre_pad = a.down - half % a.down;
    const int pre_remove = (half + pre_pad) / a.down;
    const long long t = (j + pre_remove) * a.down - pre_pad;    // tap index of x[0]; x[n] meets tap t - n up
    const long long n_lo = max(floor_div(t - a.n_taps + a.up, a.up), 0LL);
    const long long n_hi = min(floor_div(t, a.up), n_in_s - 1);
    const float* x = a.x + (size_t)sig * a.n_in;
    double acc = 0.0;
    for (long long n = n_lo; n <= n_hi; ++n) acc = fma((double)__ldg(x + n), __ldg(a.taps + (t - n * a.up)) * a.up, acc);
    a.y[(size_t)sig * a.n_out + j] = acc;
}

constexpr int kSelThreads = 256;
constexpr int kSelWarps = kSelThreads / 32;

__global__ void __launch_bounds__(kSelThreads) stoi_select_kernel(StoiArgs a) {
    __shared__ double win[kStoiFrame];
    __shared__ double wmax[kSelWarps];
    __shared__ int cnt[kSelWarps];
    const int c = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int n = tid; n < kStoiFrame; n += kSelThreads) win[n] = stoi_hann(n);
    __syncthreads();
    const double* x = a.cleans + (size_t)c * a.L;
    double* e = a.energy + (size_t)c * a.n_fr;
    int* sel = a.sel + (size_t)c * a.n_fr;
    // frames of this clean: pystoi's framing of the clean trimmed to its own length stops at its last full frame
    const int n_fr = a.lengths ? stoi_frames(a.lengths[c]) : a.n_fr;
    double mx = -INFINITY;
    for (int f = warp; f < n_fr; f += kSelWarps) {
        const double* fr = x + (size_t)f * kHop;
        double s = 0.0;
        for (int r = lane; r < kStoiFrame; r += 32) {
            const double v = win[r] * fr[r];
            s = fma(v, v, s);
        }
        // butterfly: every lane ends with the same sum
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const double en = 20.0 * log10(sqrt(s) + kEps);
        if (lane == 0) e[f] = en;
        mx = fmax(mx, en);
    }
    if (lane == 0) wmax[warp] = mx;
    __syncthreads();
    double emax = wmax[0];
    for (int w = 1; w < kSelWarps; ++w) emax = fmax(emax, wmax[w]);
    const double thr = emax - kDynRange;
    int base = 0;
    for (int f0 = 0; f0 < n_fr; f0 += kSelThreads) {
        const int f = f0 + tid;
        const bool keep = f < n_fr && thr - e[f] < 0.0;
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) cnt[warp] = __popc(b);
        __syncthreads();
        int off = base, tot = 0;
        for (int w = 0; w < kSelWarps; ++w) {
            off += w < warp ? cnt[w] : 0;
            tot += cnt[w];
        }
        if (keep) sel[off + __popc(b & ((1u << lane) - 1u))] = f;
        base += tot;
        __syncthreads();
    }
    if (tid == 0) a.n_sel[c] = base;
}

constexpr int kBandWarps = 4;

__device__ __forceinline__ bool bad_pair(const StoiArgs& a, int c, int g) {
    return c < 0 || c >= a.n_clean || g < 0 || g >= a.n_deg;
}

// grid (n_clean + n_pair) * groups: CTA b runs STFT frames (b % groups) * 4 .. + 3 of spectrogram b / groups
__global__ void __launch_bounds__(kBandWarps * 32) stoi_bands_kernel(StoiArgs a, int groups) {
    __shared__ double win[kStoiFrame];
    __shared__ double2 tw[kNfft / 2];          // exp(-2 pi i k / 512)
    __shared__ double2 buf[kBandWarps][kNfft];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int n = tid; n < kStoiFrame; n += kBandWarps * 32) {
        win[n] = stoi_hann(n);
        double s, co;
        sincospi(-(double)n / (kNfft / 2), &s, &co);
        tw[n] = make_double2(co, s);
    }
    __syncthreads();
    const int spec = blockIdx.x / groups;
    const int t = (blockIdx.x % groups) * kBandWarps + warp;
    int c;
    const double* x;
    if (spec < a.n_clean) {
        c = spec;
        x = a.cleans + (size_t)c * a.L;
    } else {
        const int p = spec - a.n_clean, g = a.pairs[2 * p + 1];
        c = a.pairs[2 * p];
        if (bad_pair(a, c, g)) return;
        x = a.degraded + (size_t)g * a.L;
    }
    const int ns = a.n_sel[c];
    if (t >= ns - 1) return;                   // the STFT takes n_sel - 1 frames of the overlap-added signal
    const int* sel = a.sel + (size_t)c * a.n_fr;
    double2* z = buf[warp];
    // sample n < 256 of STFT frame t lies in hop block j = t + n / 128 of the overlap-added signal: the first half of
    // kept frame j (j < n_sel always holds here) plus the second half of kept frame j - 1
    for (int n = lane; n < kNfft; n += 32) {
        double v = 0.0;
        if (n < kStoiFrame) {
            const int j = t + n / kHop, r = n % kHop;
            double s = win[r] * x[(size_t)sel[j] * kHop + r];
            if (j >= 1) s += win[kHop + r] * x[(size_t)sel[j - 1] * kHop + kHop + r];
            v = win[n] * s;
        }
        z[__brev(n) >> 23] = make_double2(v, 0.0);
    }
    __syncwarp();
    for (int st = 0; st < 9; ++st) {           // radix-2 decimation in time, 2^9 = 512 points
        const int half = 1 << st;
        for (int b = lane; b < kNfft / 2; b += 32) {
            const int pos = b & (half - 1);
            const int i = ((b >> st) << (st + 1)) + pos, k = i + half;
            const double2 w = tw[pos << (8 - st)], u = z[i], v = z[k];
            const double2 wv = make_double2(w.x * v.x - w.y * v.y, w.x * v.y + w.y * v.x);
            z[i] = make_double2(u.x + wv.x, u.y + wv.y);
            z[k] = make_double2(u.x - wv.x, u.y - wv.y);
        }
        __syncwarp();
    }
    if (lane < kStoiBands) {
        double s = 0.0;
        for (int k = kStoiEdges[lane]; k < kStoiEdges[lane + 1]; ++k) s += z[k].x * z[k].x + z[k].y * z[k].y;
        a.tob[((size_t)spec * a.n_fr + t) * kStoiBands + lane] = sqrt(s);
    }
}

constexpr int kScoreThreads = 256;

__global__ void __launch_bounds__(kScoreThreads) stoi_score_kernel(StoiArgs a) {
    __shared__ double red[kScoreThreads];
    const int p = blockIdx.x, tid = threadIdx.x;
    const int c = a.pairs[2 * p], g = a.pairs[2 * p + 1];
    if (bad_pair(a, c, g)) {
        if (tid == 0) {
            a.d[p] = __longlong_as_double(0x7ff8000000000000LL);
            a.n_frames[p] = -1;
        }
        return;
    }
    const int nf = a.n_sel[c] - 1;
    if (nf < kStoiSeg) {                       // pystoi returns 1e-5 (and warns) below 30 frames
        if (tid == 0) {
            a.d[p] = 1e-5;
            a.n_frames[p] = nf;
        }
        return;
    }
    const int J = nf - kStoiSeg + 1;
    const double* X = a.tob + (size_t)c * a.n_fr * kStoiBands;
    const double* Y = a.tob + (size_t)(a.n_clean + p) * a.n_fr * kStoiBands;
    double acc = 0.0;
    for (int it = tid; it < J * kStoiBands; it += kScoreThreads) {
        const int m = it / kStoiBands, b = it % kStoiBands;
        double xv[kStoiSeg], yv[kStoiSeg];
        double sxx = 0.0, syy = 0.0;
#pragma unroll
        for (int q = 0; q < kStoiSeg; ++q) {
            xv[q] = X[(size_t)(m + q) * kStoiBands + b];
            yv[q] = Y[(size_t)(m + q) * kStoiBands + b];
            sxx = fma(xv[q], xv[q], sxx);
            syy = fma(yv[q], yv[q], syy);
        }
        const double alpha = sqrt(sxx) / (sqrt(syy) + kEps);
        double sx = 0.0, sy = 0.0;
#pragma unroll
        for (int q = 0; q < kStoiSeg; ++q) {
            yv[q] = fmin(yv[q] * alpha, xv[q] * kClip);
            sx += xv[q];
            sy += yv[q];
        }
        const double mx = sx / kStoiSeg, my = sy / kStoiSeg;
        sxx = 0.0;
        syy = 0.0;
#pragma unroll
        for (int q = 0; q < kStoiSeg; ++q) {
            xv[q] -= mx;
            yv[q] -= my;
            sxx = fma(xv[q], xv[q], sxx);
            syy = fma(yv[q], yv[q], syy);
        }
        const double nx = sqrt(sxx) + kEps, ny = sqrt(syy) + kEps;
        double dot = 0.0;
#pragma unroll
        for (int q = 0; q < kStoiSeg; ++q) dot = fma(yv[q] / ny, xv[q] / nx, dot);
        acc += dot;
    }
    red[tid] = acc;
    __syncthreads();
    for (int h = kScoreThreads / 2; h > 0; h >>= 1) {
        if (tid < h) red[tid] += red[tid + h];
        __syncthreads();
    }
    if (tid == 0) {
        a.d[p] = red[0] / ((double)J * kStoiBands);
        a.n_frames[p] = nf;
    }
}

}  // namespace

cudaError_t launch_resample_poly(const ResampleArgs& a, cudaStream_t st) {
    const int per = (a.n_out + 255) / 256;
    resample_poly_kernel<<<a.n_sig * per, 256, 0, st>>>(a, per);
    return cudaGetLastError();
}

int stoi_n_fr(int L) { return stoi_frames(L); }

size_t stoi_ws_bytes(int n_clean, int n_pair, int L) {
    const size_t n_fr = (size_t)stoi_n_fr(L);
    return n_fr * ((size_t)n_clean * (sizeof(double) + sizeof(int)) +
                   ((size_t)n_clean + n_pair) * kStoiBands * sizeof(double));
}

cudaError_t launch_stoi(StoiArgs a, cudaStream_t st) {
    // workspace (set by the caller in `energy`): energy [n_clean][n_fr], tob [n_clean + n_pair][n_fr][15] (doubles),
    // then sel [n_clean][n_fr] (ints)
    a.n_fr = stoi_n_fr(a.L);
    a.tob = a.energy + (size_t)a.n_clean * a.n_fr;
    a.sel = (int*)(a.tob + ((size_t)a.n_clean + a.n_pair) * a.n_fr * kStoiBands);
    stoi_select_kernel<<<a.n_clean, kSelThreads, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (a.n_fr > 1) {
        const int groups = (a.n_fr - 1 + kBandWarps - 1) / kBandWarps;
        stoi_bands_kernel<<<(a.n_clean + a.n_pair) * groups, kBandWarps * 32, 0, st>>>(a, groups);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    stoi_score_kernel<<<a.n_pair, kScoreThreads, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace disco
