// Inverse STFT with overlap-add and window-sum-square normalisation, batched: disco_istft over whole signals and
// disco_stream_istft / disco_stream_istft_slots over the new frames of a stream run one kernel body (istft_body), so a
// stream's time samples equal those of the whole-signal call value for value.
//
// Replaces lb.core.istft(S, hop_length=N/2, win_length=N, center=True, length=L)
// (reference tango.py:528-539, math_utils.py:143-152; librosa <= 0.9 semantics, SURVEY App. A.2):
//   per frame irfft -> * periodic Hann -> overlap-add -> divide by overlap-added window^2 where
//   it exceeds tiny(float32) -> drop N/2 leading samples -> crop / zero-pad to L.
//
// One CTA owns a PAIR of signals and a chunk of hop blocks.  The two real inverse transforms are done
// by one complex inverse FFT: Z[k] = A[k] + i B[k] (k <= N/2), Z[N-k] = conj(A[k]) + i conj(B[k]),
// so Re z = a, Im z = b.  The FFT itself is the same two-pass in-register scheme as the forward
// kernel (stft_scm.cu) with conjugated twiddles.  With 50 % overlap every output hop block j
// (samples [(j-1) hop, j hop)) is  w[n] frame_j[n] + w[n+hop] frame_{j-1}[n+hop]; the second half of
// the last frame of a tile is carried in shared memory to the next tile.  Over a whole signal a chunk
// recomputes the one frame before its first block, so there are no atomics and the result is deterministic;
// a stream carries that half frame between calls in a global buffer instead.
#include "common.cuh"
#include "fft_reg.cuh"
#include "kernels.h"

namespace disco {

template <int N>
struct IGeom {
    static constexpr int RA = N / 32, NB = 32 / RA, H = N / 2, F = N / 2 + 1;
    static constexpr int ROW = N + (RA == 8 ? 8 : 0);
    static constexpr int FFT_WARPS = N / 64;
    static constexpr int THREADS = N / 2 + 32;
    static constexpr int ITEMS = 16;
    static constexpr size_t SMEM = (size_t)ITEMS * ROW * sizeof(float2) + H * sizeof(float2) + N * sizeof(float2) +
                                   N * sizeof(float);
};

// The body of both kernels below.  STREAM is a template parameter, not a test of p.carry, so that the whole-signal
// kernel keeps its own machine code: with the stream's carry and offsets as runtime cases it ran 4 % slower.
template <int N, bool STREAM>
DISCO_DEV void istft_body(const IstftArgs& p) {
    using G = IGeom<N>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROW = G::ROW, TT = G::ITEMS;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2* rows = reinterpret_cast<float2*>(smem_raw);    // [TT][ROW]
    float2* carry = rows + TT * ROW;                       // [H] second half of the previous frame (windowed)
    float2* tw = carry + H;                                // [RA][32]
    float* win = reinterpret_cast<float*>(tw + N);         // [N]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pair = blockIdx.y, chunk = blockIdx.x;
    const int sa = 2 * pair, sb = 2 * pair + 1;
    const bool has_b = sb < p.n_sig;
    const int L = p.L;
    const int y_t0 = STREAM ? p.y_t0 : 0, x_first = STREAM ? p.x_first : 0;
    // (the stream's b rows are offsets from the a rows: as pointers of their own they spill at 1024 points)
    const float2* Ya = p.Y + (size_t)sa * p.y_frames * F;                 // frame j at row j - y_t0
    const float2* Yb = STREAM ? Ya + (has_b ? (size_t)p.y_frames * F : 0) : p.Y + (size_t)(has_b ? sb : sa) * p.y_frames * F;
    float* xa = p.x + (size_t)sa * p.ld;                                  // sample s at s - x_first
    float* xb = STREAM ? xa + (has_b ? (size_t)p.ld : 0) : p.x + (size_t)(has_b ? sb : sa) * p.ld;

    const int j_begin = (STREAM ? p.j_begin : 0) + chunk * p.fpc;   // first hop block of this chunk
    const int j_end = min(p.j_end, j_begin + p.fpc);              // blocks [j_begin, j_end) (+ j_end with the tail)
    const bool tail = (!STREAM || p.tail) && j_end == p.j_end;
    const int fs = STREAM ? j_begin : max(j_begin - 1, 0);       // first frame to transform

    for (int i = tid; i < N; i += blockDim.x) {
        tw[i] = p.twiddle[i];
        win[i] = p.window[i];
    }
    if (tid < H)
        carry[tid] = STREAM ? make_float2(p.carry[(size_t)sa * H + tid], has_b ? p.carry[(size_t)sb * H + tid] : 0.f)
                             : make_float2(0.f, 0.f);
    __syncthreads();
    const float inv_n = 1.0f / (float)N;
    const float tiny = 1.17549435e-38f;

    for (int t0 = fs; t0 < j_end; t0 += TT) {
        const int nfr = min(TT, j_end - t0);
        // ---- 1. gather the two half spectra into one full complex spectrum per frame
        if (tid < F) {
            const int f = tid;
            for (int tl = 0; tl < nfr; ++tl) {
                const size_t off = (size_t)(t0 + tl - y_t0) * F + f;
                float2 A = Ya[off];
                float2 B = has_b ? Yb[off] : make_float2(0.f, 0.f);
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
                const int j = t0 + tl;               // frame j, hop block j
                const float2 cur = rows[tl * ROW + n];
                const float2 nxt = rows[tl * ROW + n + H];
                if (j >= j_begin) {
                    float2 val = cadd(cscale(cur, w0 * inv_n), prev);
                    const float wss = w0 * w0 + (j >= 1 ? w1 * w1 : 0.f);
                    if (wss > tiny) val = cscale(val, 1.0f / wss);
                    const int s = (j - 1) * H + n;
                    if (s >= 0 && s < L) {
                        xa[s - x_first] = val.x;
                        if (has_b) xb[s - x_first] = val.y;
                    }
                }
                prev = cscale(nxt, w1 * inv_n);
            }
            carry[n] = prev;
        }
        __syncthreads();
    }
    if (STREAM && tid < H) {
        p.carry[(size_t)sa * H + tid] = carry[tid].x;
        if (has_b) p.carry[(size_t)sb * H + tid] = carry[tid].y;
    }
    // ---- tail: block j_end has only the second half of the last frame; then zero-fill up to L
    if (tail) {
        if (tid < H) {
            const int n = tid;
            const float w1 = win[n + H];
            float2 val = carry[n];
            const float wss = w1 * w1;
            if (wss > tiny) val = cscale(val, 1.0f / wss);
            const int s = (j_end - 1) * H + n;
            if (s >= 0 && s < L) {
                xa[s - x_first] = val.x;
                if (has_b) xb[s - x_first] = val.y;
            }
        }
        for (int s = j_end * H + tid; s < L; s += blockDim.x) {
            xa[s - x_first] = 0.f;
            if (has_b) xb[s - x_first] = 0.f;
        }
    }
}

template <int N>
__global__ void __launch_bounds__(IGeom<N>::THREADS) istft_kernel(IstftArgs p) {
    istft_body<N, false>(p);
}

// Whole signals of their own lengths (disco_istft_lengths, launched from lengths.cu): signal s is the iSTFT of its
// frames [0, min(j_end, 1 + lengths[s] / H)) cut to lengths[s] samples, exactly as disco_istft runs it on those frames
// and that length, and is zero from lengths[s] to L (the row length).  A pair of equal lengths runs as a pair, as
// disco_istft pairs it; the two signals of a pair of different lengths run one after the other, each alone.
template <int N>
__global__ void __launch_bounds__(IGeom<N>::THREADS) istft_lengths_kernel(IstftArgs p, const int* lengths) {
    constexpr int H = IGeom<N>::H, F = IGeom<N>::F;
    const int sa = 2 * blockIdx.y, sb = sa + 1;
    const bool has_b = sb < p.n_sig;
    const int La = lengths[sa], Lb = has_b ? lengths[sb] : La;
    // s0: the signal the body sees as the pair's first; alone: no partner
    auto run = [&](int s0, bool alone, int len) {
        IstftArgs q = p;
        q.L = len;
        q.j_end = min(p.j_end, 1 + len / H);
        if ((int)blockIdx.x * p.fpc >= q.j_end) return;   // CTA-uniform: this chunk lies past the signal's frames
        if (alone) {
            q.Y = p.Y + (ptrdiff_t)(s0 - sa) * p.y_frames * F;
            q.x = p.x + (ptrdiff_t)(s0 - sa) * p.ld;
            q.n_sig = sa + 1;
        }
        istft_body<N, false>(q);
    };
    if (La == Lb) {
        run(sa, false, La);
    } else {
        run(sa, true, La);
        __syncthreads();   // the second run reloads the shared tables and the carry
        run(sb, true, Lb);
    }
    if (blockIdx.x == 0) {
        for (int s = La + threadIdx.x; s < p.L; s += blockDim.x) p.x[(size_t)sa * p.ld + s] = 0.f;
        if (has_b)
            for (int s = Lb + threadIdx.x; s < p.L; s += blockDim.x) p.x[(size_t)sb * p.ld + s] = 0.f;
    }
}

// A stream: grid (1, signal pairs of a slot, slots).  Slot blockIdx.z runs the stream body on its own rows with its
// record {t0, n_fr, length, final, x_first}: from `slots` (a pool) or, with slots = null, `one` (a lockstep stream).
template <int N>
__global__ void __launch_bounds__(IGeom<N>::THREADS) stream_istft_kernel(IstftArgs p, const IstftSlot* slots,
                                                                         IstftSlot one) {
    constexpr int H = IGeom<N>::H, F = IGeom<N>::F;
    IstftSlot r = one;
    if (slots) r = slots[blockIdx.z];
    if (r.n_fr <= 0 && !r.final_call) return;   // CTA-uniform: no frames, not the end of the stream
    IstftArgs q = p;
    const size_t row0 = (size_t)blockIdx.z * p.n_sig;
    q.Y = p.Y + row0 * p.y_frames * F;
    q.x = p.x ? p.x + row0 * p.ld : nullptr;
    q.carry = p.carry + row0 * H;
    q.L = r.length;
    q.y_t0 = r.t0;
    q.j_begin = r.t0;
    q.j_end = r.t0 + r.n_fr;
    q.fpc = r.n_fr;
    q.tail = r.final_call;
    q.x_first = r.x_first;
    istft_body<N, true>(q);
}

template <int N>
static cudaError_t launch_slots_n(const IstftArgs& a, const IstftSlot* slots, const IstftSlot& one, int n_slot,
                                   cudaStream_t st) {
    using G = IGeom<N>;
    cudaError_t e = cudaFuncSetAttribute(stream_istft_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)G::SMEM);
    if (e != cudaSuccess) return e;
    stream_istft_kernel<N><<<dim3(1, (a.n_sig + 1) / 2, n_slot), G::THREADS, G::SMEM, st>>>(a, slots, one);
    return cudaGetLastError();
}

// n_slot slots; a lockstep stream is one slot whose record is `one`
cudaError_t launch_stream_istft_slots(const IstftArgs& a, const IstftSlot* slots, const IstftSlot& one, int n_slot,
                                      int n_fft, cudaStream_t st) {
    if (a.n_sig <= 0 || n_slot <= 0 || (!slots && one.n_fr <= 0 && !one.final_call)) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_slots_n<256>(a, slots, one, n_slot, st);
        case 512: return launch_slots_n<512>(a, slots, one, n_slot, st);
        case 1024: return launch_slots_n<1024>(a, slots, one, n_slot, st);
        default: return cudaErrorInvalidValue;
    }
}

IstftLengthsKernel istft_lengths_kernel_for(int n_fft) {
    switch (n_fft) {
        case 256: return {(const void*)istft_lengths_kernel<256>, IGeom<256>::THREADS, IGeom<256>::SMEM, IGeom<256>::ITEMS};
        case 512: return {(const void*)istft_lengths_kernel<512>, IGeom<512>::THREADS, IGeom<512>::SMEM, IGeom<512>::ITEMS};
        case 1024: return {(const void*)istft_lengths_kernel<1024>, IGeom<1024>::THREADS, IGeom<1024>::SMEM,
                           IGeom<1024>::ITEMS};
        default: return {nullptr, 0, 0, 0};
    }
}

template <int N>
static cudaError_t launch_n(IstftArgs a, cudaStream_t st) {
    using G = IGeom<N>;
    const int H = G::H;
    const int pairs = (a.n_sig + 1) / 2;
    // the blocks past the last sample are not computed; chunks of fpc blocks
    a.j_end = min(a.j_end, (a.L + N + H - 1) / H);
    const int T_eff = a.j_end - a.j_begin;
    if (T_eff < 1) return cudaErrorInvalidValue;
    int chunks = 1;
    while (pairs * chunks < sm_count() * 2 && (T_eff + chunks - 1) / chunks > 4 * G::ITEMS) chunks *= 2;
    a.fpc = ((T_eff + chunks - 1) / chunks + G::ITEMS - 1) / G::ITEMS * G::ITEMS;
    chunks = (T_eff + a.fpc - 1) / a.fpc;
    cudaError_t e = cudaFuncSetAttribute(istft_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G::SMEM);
    if (e != cudaSuccess) return e;
    // pairs sit in grid.y: consecutive launches of at most kMaxGridYZ pairs, each starting at an even signal (a pair
    // keeps its partner) with Y and x advanced to it (whole-signal rows are contiguous per signal)
    const int n_sig = a.n_sig, F = N / 2 + 1;
    for (int p0 = 0; p0 < pairs; p0 += kMaxGridYZ) {
        IstftArgs b = a;
        const int s0 = 2 * p0;
        b.Y = a.Y + (size_t)s0 * a.y_frames * F;
        b.x = a.x + (size_t)s0 * a.ld;
        b.n_sig = min(n_sig - s0, 2 * kMaxGridYZ);
        istft_kernel<N><<<dim3(chunks, (b.n_sig + 1) / 2), G::THREADS, G::SMEM, st>>>(b);
        e = cudaGetLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// Whole signals (a.carry = null, a.tail = 1)
cudaError_t launch_istft(const IstftArgs& a, int n_fft, cudaStream_t st) {
    if (a.n_sig <= 0) return cudaSuccess;
    switch (n_fft) {
        case 256: return launch_n<256>(a, st);
        case 512: return launch_n<512>(a, st);
        case 1024: return launch_n<1024>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
