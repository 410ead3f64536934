// BSS-eval source scores (mir_eval.separation.bss_eval_sources, the SDR / SIR / SAR of the reference's tango.main,
// disco_theque/speech_enhancement/tango.py:552-567) in float64.
//
// For references r_1 .. r_n and an estimate e of L samples, mir_eval projects e onto the span of the reference copies
// delayed by 0 .. flen-1 samples.  Everything the scores need is ‖e‖² and the squared norms ‖y_S‖² of the forward
// substitutions L_S y_S = D_S, G_S = L_S L_S^T, where G = A^T A is the Gram matrix of the delayed copies and D = A^T e
// (‖P_S e‖² = D_S^T G_S^-1 D_S = ‖y_S‖²).  Two kernels plus a small reduction produce them:
//
//   bss_corr_kernel    Q[set][i][s][k] = sum_t x_s(t) r_i(t - k), k < flen, for every reference r_i of a set and every
//                      signal x_s of it (its references, then its estimate rows), per time segment of kBssSeg samples.
//                      G's Toeplitz blocks are G[(i,a),(j,b)] = Q[i][j][a-b] (a >= b) or Q[j][i][b-a]; D = Q[j][e][b].
//                      A thread owns 8 consecutive lags of up to 4 signals: per sample it reads one new reference value
//                      (a register window slides along the lags) and issues 32 DFMAs.  Float32 inputs make every
//                      product exact in float64; each output is one sequential sum over the segment's samples.
//   bss_reduce_kernel  sums the segments in order.
//   bss_factor_kernel  one CTA per (set, job): job 0 assembles the full G (nsrc flen square) with the D rows of every
//                      estimate appended below it, job q >= 1 the diagonal block G_qq with the D_q rows; a left-looking
//                      blocked Cholesky of the stacked matrix turns the appended rows into y = L^-1 D (the Cholesky row
//                      of an appended row IS the forward substitution), and the squared norms of y are written per
//                      reference block.  The single-reference factor of reference 0 is the leading block of job 0.
//
// Pivot policy: a pivot d <= delta * max diag G (kBssDelta) marks its column as dependent: the column is zeroed and
// its y component is 0, which is the exact projection onto the span of the other columns (a singular G, e.g. when
// L + flen - 1 < nsrc flen).  No atomics anywhere: every result depends on its set's data, L and flen only, never on
// the set's position in the batch or on the batch size.
#include <math.h>

#include "kernels.h"

namespace disco {

namespace {

constexpr int kCorrThreads = kBssMaxFlen / 8;  // one thread per 8 lags
constexpr int kChunk = 256;                      // samples per shared-memory chunk
constexpr int kSig = 4;                          // signals per CTA
__host__ __device__ constexpr int skew(int v) { return v + (v >> 3); }   // conflict-free lanes 8 doubles apart
constexpr int kWin = skew(kBssMaxFlen + kChunk - 1) + 1;

// signal s of a set: its references first, then its estimate rows
__device__ __forceinline__ const float* bss_signal(const BssArgs& a, int set, int s) {
    return s < a.nsrc ? a.refs + ((size_t)set * a.nsrc + s) * a.L : a.ests + ((size_t)set * a.n_est + (s - a.nsrc)) * a.L;
}

template <int A>
__device__ __forceinline__ void corr_run(const BssArgs& a, const float* r, int set, int s0, double* out, double* W,
                                         double (*X)[kChunk], int seg) {
    const int fl8 = (a.flen + 7) & ~7;
    const int k0 = threadIdx.x * 8;
    const bool live = k0 < a.flen;
    const int t_lo = seg * kBssSeg, t_hi = min(a.L, t_lo + kBssSeg);
    double acc[A][8];
#pragma unroll
    for (int q = 0; q < A; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[q][j] = 0.0;

    for (int tc = t_lo; tc < t_hi; tc += kChunk) {
        __syncthreads();                                   // the previous chunk is consumed
        // W[v] = r(tc - fl8 + v), v < fl8 + kChunk (zero outside [0, L)); X[q][dt] = x_q(tc + dt) (zero past the segment)
        for (int v = threadIdx.x; v < fl8 + kChunk; v += blockDim.x) {
            const int u = tc - fl8 + v;
            W[skew(v)] = (u >= 0 && u < a.L) ? (double)__ldg(r + u) : 0.0;
        }
        for (int e = threadIdx.x; e < A * kChunk; e += blockDim.x) {
            const int q = e / kChunk, t = tc + e % kChunk;
            X[q][e % kChunk] = t < t_hi ? (double)__ldg(bss_signal(a, set, s0 + q) + t) : 0.0;
        }
        __syncthreads();
        if (!live) continue;
        const int nblk = (min(kChunk, t_hi - tc) + 7) / 8;
        // rw[i] = W[vb + db + i]: sample tc + db + dt at lag k0 + j reads W[fl8 + db + dt - k0 - j] = rw[8 + dt - j]
        const int vb = fl8 - k0 - 8;
        double rw[16];
#pragma unroll
        for (int i = 0; i < 8; ++i) rw[i] = W[skew(vb + i)];
        for (int b = 0; b < nblk; ++b) {
            const int db = b * 8;
#pragma unroll
            for (int i = 0; i < 8; ++i) rw[8 + i] = W[skew(vb + db + 8 + i)];
#pragma unroll
            for (int dt = 0; dt < 8; ++dt) {
#pragma unroll
                for (int q = 0; q < A; ++q) {
                    const double xv = X[q][db + dt];
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[q][j] = fma(xv, rw[8 + dt - j], acc[q][j]);
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) rw[i] = rw[8 + i];
        }
    }
    if (!live) return;
    const size_t sstride = (size_t)a.n_seg * a.flen;
#pragma unroll
    for (int q = 0; q < A; ++q)
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (k0 + j < a.flen) out[q * sstride + k0 + j] = acc[q][j];
}

// grid (n_set * nsrc, ceil(M / 4), n_seg): the CTA of (set, reference i) correlates signals s0 .. s0 + 3 with r_i
__global__ void __launch_bounds__(kCorrThreads) bss_corr_kernel(BssArgs a) {
    __shared__ double W[kWin];
    __shared__ double X[kSig][kChunk];
    const int M = a.nsrc + a.n_est;
    const int set = blockIdx.x / a.nsrc, i = blockIdx.x % a.nsrc;
    const int s0 = blockIdx.y * kSig, seg = blockIdx.z;
    const int nsig = min(kSig, M - s0);
    const float* r = a.refs + ((size_t)set * a.nsrc + i) * a.L;
    double* out = a.part + (((size_t)set * a.nsrc + i) * M + s0) * a.n_seg * a.flen + (size_t)seg * a.flen;
    switch (nsig) {
        case 1: corr_run<1>(a, r, set, s0, out, W, X, seg); break;
        case 2: corr_run<2>(a, r, set, s0, out, W, X, seg); break;
        case 3: corr_run<3>(a, r, set, s0, out, W, X, seg); break;
        default: corr_run<4>(a, r, set, s0, out, W, X, seg); break;
    }
}

// corr[row][k] = sum over the segments, in segment order, of part[row][seg][k]
__global__ void bss_reduce_kernel(BssArgs a, size_t n) {
    for (size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x; idx < n; idx += (size_t)gridDim.x * blockDim.x) {
        const size_t row = idx / a.flen, k = idx % a.flen;
        const double* p = a.part + row * a.n_seg * a.flen + k;
        double s = 0.0;
        for (int g = 0; g < a.n_seg; ++g) s += p[(size_t)g * a.flen];
        a.corr[idx] = s;
    }
}

constexpr int kFacThreads = 256;
constexpr int kNB = 64;        // Cholesky block
constexpr int kKK = 16;        // inner dimension staged per step of the block-column update
constexpr int kLd = kNB + 1;   // padded smem row

// C[rr][cc] = A[r0 + rr][kb + cc] - sum_{m < kb} A[r0 + rr][m] A[kb + cc][m]   (rr < 64, cc < nbk; zero elsewhere)
// The sum runs over m in increasing order, kKK at a time, one fma chain per output.
__device__ void block_update(const double* A, int ld, int rows, int r0, int kb, int nbk, double* C, double* As,
                             double* Bs) {
    const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
    double acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
    for (int m0 = 0; m0 < kb; m0 += kKK) {
        __syncthreads();
        for (int e = tid; e < kNB * kKK; e += kFacThreads) {
            const int rr = e / kKK, kk = e % kKK;
            As[kk * kLd + rr] = r0 + rr < rows ? A[(size_t)(r0 + rr) * ld + m0 + kk] : 0.0;
            Bs[kk * kLd + rr] = rr < nbk ? A[(size_t)(kb + rr) * ld + m0 + kk] : 0.0;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < kKK; ++kk) {
            double av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[kk * kLd + ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[kk * kLd + tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fma(av[i], bv[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int rr = ty + 16 * i, cc = tx + 16 * j;
            C[rr * kLd + cc] = (r0 + rr < rows && cc < nbk) ? A[(size_t)(r0 + rr) * ld + kb + cc] - acc[i][j] : 0.0;
        }
    __syncthreads();
}

// grid (n_set * nsrc): job 0 = the full reference set, job q >= 1 = reference q alone
__global__ void __launch_bounds__(kFacThreads) bss_factor_kernel(BssArgs a) {
    extern __shared__ double sm[];
    double* Dg = sm;                      // [kNB][kLd] diagonal block, factored in place
    double* Ct = Dg + kNB * kLd;          // [kNB][kLd] block of rows below it
    double* As = Ct + kNB * kLd;          // [kKK][kLd]
    double* Bs = As + kKK * kLd;          // [kKK][kLd]
    double* dinv = Bs + kKK * kLd;        // [kNB] 1 / pivot, 0 for a dependent column
    double* red = dinv + kNB;             // [kFacThreads]

    const int tid = threadIdx.x;
    const int nsrc = a.nsrc, flen = a.flen, n_est = a.n_est, M = nsrc + n_est;
    const int set = blockIdx.x / nsrc, q = blockIdx.x % nsrc;
    const double* Q = a.corr + (size_t)set * nsrc * M * flen;   // Q[i][s][k] = Q[(i * M + s) * flen + k]
    const int NF = nsrc * flen;
    const int N = q == 0 ? NF : flen;
    const int rows = N + n_est;
    double* A = a.mat + (size_t)set * a.mat_per_set +
                (q == 0 ? 0 : (size_t)(NF + n_est) * NF + (size_t)(q - 1) * (flen + n_est) * flen);
    const int nw = 1 + 2 * nsrc;
    double* norms = a.norms + (size_t)set * n_est * nw;

    // assemble [G; D^T] row-major, ld = N
    for (size_t idx = tid; idx < (size_t)rows * N; idx += kFacThreads) {
        const int r = (int)(idx / N), c = (int)(idx % N);
        const int j = q == 0 ? c / flen : q, b = q == 0 ? c % flen : c;
        double v;
        if (r < N) {
            const int i = q == 0 ? r / flen : q, aa = q == 0 ? r % flen : r;
            v = aa >= b ? Q[((size_t)i * M + j) * flen + aa - b] : Q[((size_t)j * M + i) * flen + b - aa];
        } else {
            v = Q[((size_t)j * M + nsrc + (r - N)) * flen + b];
        }
        A[idx] = v;
    }
    double maxdiag = 0.0;
    for (int i = (q == 0 ? 0 : q); i < (q == 0 ? nsrc : q + 1); ++i) maxdiag = fmax(maxdiag, Q[((size_t)i * M + i) * flen]);
    const double thr = kBssDelta * maxdiag;

    if (q == 0) {   // ‖e‖² of every estimate row: strided sequential sums, then a fixed tree
        for (int e = 0; e < n_est; ++e) {
            const float* x = a.ests + ((size_t)set * n_est + e) * a.L;
            double s = 0.0;
            for (int t = tid; t < a.L; t += kFacThreads) {
                const double v = (double)x[t];
                s = fma(v, v, s);
            }
            red[tid] = s;
            __syncthreads();
            for (int h = kFacThreads / 2; h > 0; h >>= 1) {
                if (tid < h) red[tid] += red[tid + h];
                __syncthreads();
            }
            if (tid == 0) norms[(size_t)e * nw] = red[0];
            __syncthreads();
        }
    }
    __syncthreads();

    for (int kb = 0; kb < N; kb += kNB) {
        const int nbk = min(kNB, N - kb);
        block_update(A, N, rows, kb, kb, nbk, Dg, As, Bs);
        // unblocked Cholesky of the diagonal block with the dependent-column rule
        for (int j = 0; j < nbk; ++j) {
            const double d = Dg[j * kLd + j];
            const bool dep = !(d > thr);
            const double piv = dep ? 0.0 : sqrt(d);
            const double inv = dep ? 0.0 : 1.0 / piv;
            __syncthreads();                                  // every thread has read d
            for (int i = j + 1 + tid; i < nbk; i += kFacThreads) Dg[i * kLd + j] *= inv;
            if (tid == 0) {
                Dg[j * kLd + j] = piv;
                dinv[j] = inv;
            }
            __syncthreads();
            const int w = nbk - j - 1;
            for (int e = tid; e < w * w; e += kFacThreads) {
                const int i = j + 1 + e / w, c = j + 1 + e % w;
                if (c <= i) Dg[i * kLd + c] -= Dg[i * kLd + j] * Dg[c * kLd + j];
            }
            __syncthreads();
        }
        for (int e = tid; e < nbk * nbk; e += kFacThreads) {
            const int i = e / nbk, c = e % nbk;
            A[(size_t)(kb + i) * N + kb + c] = c <= i ? Dg[i * kLd + c] : 0.0;
        }
        // rows below: X L_kk^T = C, solved row by row, 4 lanes per row (lane qq owns the columns = qq mod 4)
        for (int r0 = kb + nbk; r0 < rows; r0 += kNB) {
            block_update(A, N, rows, r0, kb, nbk, Ct, As, Bs);
            const int rr = tid / 4, qq = tid % 4;
            for (int j = 0; j < nbk; ++j) {
                double p = 0.0;
                for (int m = qq; m < j; m += 4) p = fma(Ct[rr * kLd + m], Dg[j * kLd + m], p);
                p += __shfl_xor_sync(0xffffffffu, p, 1);
                p += __shfl_xor_sync(0xffffffffu, p, 2);
                if ((j & 3) == qq) Ct[rr * kLd + j] = (Ct[rr * kLd + j] - p) * dinv[j];
            }
            __syncthreads();
            for (int e = tid; e < kNB * nbk; e += kFacThreads) {
                const int i = e / nbk, c = e % nbk;
                if (r0 + i < rows) A[(size_t)(r0 + i) * N + kb + c] = Ct[i * kLd + c];
            }
            __syncthreads();
        }
        __syncthreads();
    }

    // squared norms of y per reference block, each a sequential sum over its flen entries
    const int nblk = q == 0 ? nsrc : 1;
    for (int p = tid; p < n_est * nblk; p += kFacThreads) {
        const int e = p / nblk, b = p % nblk;
        const double* y = A + (size_t)(N + e) * N + (size_t)b * flen;
        double s = 0.0;
        for (int c = 0; c < flen; ++c) s = fma(y[c], y[c], s);
        double* o = norms + (size_t)e * nw;
        if (q == 0) {
            o[1 + b] = s;
            if (b == 0) o[1 + nsrc] = s;
        } else {
            o[1 + nsrc + q] = s;
        }
    }
}

constexpr size_t kFacSmem = (size_t)(2 * kNB * kLd + 2 * kKK * kLd + kNB + kFacThreads) * sizeof(double);

}  // namespace

size_t bss_mat_per_set(int nsrc, int n_est, int flen) {
    const size_t NF = (size_t)nsrc * flen;
    return (NF + n_est) * NF + (size_t)(nsrc - 1) * (flen + n_est) * flen;
}

int bss_n_seg(int L) { return (L + kBssSeg - 1) / kBssSeg; }

size_t bss_ws_doubles(int n_set, int nsrc, int n_est, int L, int flen) {
    const size_t M = (size_t)nsrc + n_est;
    return (size_t)n_set * (nsrc * M * flen * ((size_t)bss_n_seg(L) + 1) + bss_mat_per_set(nsrc, n_est, flen));
}

cudaError_t launch_bss_eval(BssArgs a, cudaStream_t st) {
    const int M = a.nsrc + a.n_est;
    a.n_seg = bss_n_seg(a.L);
    a.mat_per_set = bss_mat_per_set(a.nsrc, a.n_est, a.flen);
    const size_t n_corr = (size_t)a.n_set * a.nsrc * M * a.flen;
    // workspace: part [n_corr][n_seg], corr [n_corr], matrices [n_set][mat_per_set]
    double* ws = a.part;
    a.corr = ws + n_corr * a.n_seg;
    a.mat = a.corr + n_corr;
    bss_corr_kernel<<<dim3(a.n_set * a.nsrc, (M + kSig - 1) / kSig, a.n_seg), kCorrThreads, 0, st>>>(a);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const size_t reduce_blocks = (n_corr + 255) / 256, max_blocks = (size_t)sm_count() * 16;
    bss_reduce_kernel<<<(int)(reduce_blocks < max_blocks ? reduce_blocks : max_blocks), 256, 0, st>>>(a, n_corr);
    e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(bss_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFacSmem);
    if (e != cudaSuccess) return e;
    bss_factor_kernel<<<a.n_set * a.nsrc, kFacThreads, kFacSmem, st>>>(a);
    return cudaGetLastError();
}

}  // namespace disco
