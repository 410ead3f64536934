// Fused STFT + mask-weighted spatial-covariance (SCM) accumulation, and the plain STFT.
//
// Replaces, for a whole batch in one launch:
//   lb.core.stft(x, n_fft, hop, center=True)            reference tango.py:335-337
//   s_hat = m * Y, n_hat = (1 - m) * Y                   reference tango.py:347-348, :413-414
//   np.outer(.., conj(..)) per (f, t) + np.mean over t   reference tango.py:357-364, :433-440
// for up to 8 microphones per array node and for ONE or TWO masks at once (NM = 2: the step-1 mask
// AND the step-2 mask of a single-node array, whose step-2 input is the same Y -- tango.py:431-440
// with K = 1 -- so Y never has to be read back for the second set of statistics).
//
// Persistent, warp-specialised kernel: one CTA per SM walks a contiguous range of TILES
// (tile = TT consecutive frames of one group; group = one array node of one utterance, C mics).
// Three warp roles form a two-stage producer/consumer pipeline through shared memory, linked by
// mbarriers (no __syncthreads in the steady state):
//
//   warp 0        LOADER   stages the (TT+1)*hop samples of every channel with one 1-D bulk TMA
//                          copy per channel (edge tiles: the FFT warps fill in librosa's reflect
//                          padding), one tile ahead.  It also owns the Nyquist bin: lanes <-> channel
//                          PAIRS (the Nyquist spectrum is real, an SCM entry a plain product).
//   FFT warps     two real channels are transformed by ONE complex FFT.  A job is 32/RA transforms
//                          (RA = N/32): an RA-point in-register DFT per lane, a padded transposition
//                          through shared memory, then one 32-point in-register DFT per lane
//                          (stft_core.cuh, shared with stream.cu).  Spectra of the pairs stay in smem.
//   SCM warps     thread f owns frequency bin f.  It un-mixes the two-for-one spectra, writes Y
//                          (frame-major rows, coalesced), and accumulates the Hermitian upper
//                          triangles of  sum_t m^2 y y^H  and  sum_t (1-m)^2 y y^H  (per mask) in
//                          registers: one outer product (fmul2 + ffma2) feeds all of them.
//                          Mask values are prefetched a chunk of frames ahead.
// For 5..8 microphones the 128 accumulators of a bin need ~184 registers, so the roles are laid out
// on warpgroup boundaries and the register file is redistributed with setmaxnreg (loader 32, SCM 184,
// FFT what is left: 112) -- the same mechanism the TMA/wgmma kernels of this architecture use.
// Two masks at 512 points (3 or 4 microphones): the loader and 7 FFT warps share the first two
// warpgroups at 104 registers, the 8 SCM warps get 152, and the 8 FFT jobs of a tile are dealt over
// the 7 FFT warps across the CTA's tile stream (StftCfg::DEAL).
//
// A CTA's tile range may cross group boundaries; accumulators are flushed per (group, CTA)
// segment into a small workspace and reduced in fixed order by scm_finalize_kernel or directly by
// the solver (deterministic, no atomics).
#include "common.cuh"
#include "kernels.h"
#include "stft_core.cuh"

namespace disco {

// What the consumer warps write per (frame, bin): the spectrum Y; nothing (NM > 0: the statistics are the only
// output); or, with NM = 0, the single-node dual filter  z = w1^H y, zn = y[ref] - z, yf = w2^H y  of filter_dual.cu,
// so that the filter pass transforms the time signals again instead of reading a stored Y back; OUT_FILTER writes the
// three outputs frame-major ([T][F]), OUT_FILTER_FT in the reference's (F, T) layout.
enum : int { OUT_Y = 0, OUT_NONE = 1, OUT_FILTER = 2, OUT_FILTER_FT = 3 };

template <int N, int C, int NM = 1, int OUT = OUT_Y>
struct StftCfg : StftJob<N> {                      // RA, NB, H, F, ROWP: the FFT job (stft_core.cuh)
    static constexpr bool WIDE = C > 4;            // 128 accumulators per bin
    static constexpr int NSTG = 2;                 // pipeline stages (samples and spectra)
    static constexpr int JOBS = 8;                 // jobs per tile
    static constexpr int ITEMS = JOBS * StftJob<N>::NB;   // (frame, channel-pair) transforms per tile
    static constexpr int P = (C + 1) / 2;          // channel pairs per frame
    static constexpr int TT = ITEMS / P;           // frames per tile
    // Roles on warpgroup boundaries + setmaxnreg: the SCM warps of wide arrays (128 accumulators) and of
    // two-mask runs (64) need more registers than an even split of the register file gives them.
    static constexpr bool REALLOC = (N == 512) || (WIDE && N == 256);
    // with one mask eight FFT warps are faster than four (H100 A/B: 218-220 us against 223-226, 64 x 4 mics x 10 s;
    // DESIGN.md 4.1).  Two masks at 512 points, 3-4 microphones (DEAL): the SCM warps need 152 registers, which
    // leaves room for 7 FFT warps at 104 only if the three padding warps of the loader's warpgroup become FFT warps;
    // the 8 jobs of a tile are dealt over them across the tile stream (job j of the CTA -> warp j mod 7), so no warp
    // runs two jobs of a tile while another idles.  With 4 FFT warps running two jobs each, the role clocks showed
    // the FFT warps busy 94 % of the time and the SCM warps waiting on spec_full 40 % (DESIGN.md 4.1).
    // (3-4 microphones only: a tile of 1-2 microphones is 16 frames, so the single-node 2-microphone cfg 1 runs one tile
    // per CTA, where dealing cannot shorten the FFT path and its step was 4 % slower.  The two-mask kernels of 1-2
    // microphones keep 4 FFT warps running two jobs each per tile next to SCM warps at 152 registers.)
    static constexpr bool DEAL = N == 512 && NM == 2 && C >= 3 && !WIDE;
    static constexpr int FFT_WARPS = DEAL ? 7 : (N == 512 && (WIDE || NM == 2)) ? 4 : 8;
    static constexpr int JPW = JOBS / FFT_WARPS;   // jobs per FFT warp and tile (without DEAL)
    static constexpr int FFT_ARRIVALS = DEAL ? JOBS : FFT_WARPS;   // samp_empty / spec_full arrivals per tile
    static constexpr int SCM_WARPS = N / 64;       // bins 0 .. N/2-1, one per thread
    static constexpr int LEAD_WARPS = (REALLOC && !DEAL) ? 4 : 1;   // warp 0 = loader; 1..3 idle (warpgroup padding)
    static constexpr int WARPS = LEAD_WARPS + FFT_WARPS + SCM_WARPS;
    static constexpr int THREADS = 32 * WARPS;
    static constexpr int SPEC = ITEMS * StftJob<N>::ROWP;   // complex per spectrum stage
    static constexpr int SAMP = C * (TT + 1) * StftJob<N>::H;   // floats per sample stage
    // registers per thread at launch: each of the 4 SM sub-partitions holds 16384 registers and ceil(WARPS/4) warps
    static constexpr int REG_LAUNCH = 16384 / ((WARPS + 3) / 4) / 32 / 8 * 8;
    // REALLOC only: setmaxnreg budgets per thread of the roles.  The sm_90a build of every 256- and 512-point
    // variant is free of local-memory spills with these (ptxas -v); the loader needs 32 for the two Nyquist pair
    // slots of 7-8 microphones, and the FFT warps 104-112 for a 512-point transform.  The loader warpgroup and the
    // SCM warps (5..8 microphones / up to 4 next to 4 FFT warps / up to 4 next to 8 FFT warps) get fixed budgets;
    // the FFT warps get what is left of the CTA's allocation (a multiple of 8), capped at 256.
    // The filter consumer (OUT_FILTER) holds 2 C filter taps and one frame's C spectra instead of accumulators, and its
    // loader also applies the Nyquist-bin filters (2 C taps of its own), so the loader gets more and the consumer far
    // fewer registers; the FFT warps take what is left as always.
    // DEAL: the loader shares its warpgroup with three FFT warps, so both leading warpgroups get the FFT budget
    // (2 x 128 x 104 + 256 x 152 = 65 536, all of the launch allocation of 16 warps x 128).
    static constexpr bool FILT = OUT == OUT_FILTER || OUT == OUT_FILTER_FT;
    static constexpr int REG_SCM = FILT ? 80 : WIDE ? 184 : ((N == 512 && NM == 2) ? 152 : 120);
    static constexpr int REG_FFT_CAP = 256;
    static constexpr int REG_ALLOC = (REG_LAUNCH > 255 ? 255 : REG_LAUNCH) * THREADS;
    static constexpr int REG_LEAD_OWN = FILT ? 56 : 32;   // the loader warpgroup's budget without DEAL
    static constexpr int REG_FFT_LEFT =
        DEAL ? (REG_ALLOC - 32 * SCM_WARPS * REG_SCM) / (32 * (LEAD_WARPS + FFT_WARPS)) / 8 * 8
             : (REG_ALLOC - 128 * REG_LEAD_OWN - 32 * SCM_WARPS * REG_SCM) / (32 * FFT_WARPS) / 8 * 8;
    static constexpr int REG_FFT = REG_FFT_LEFT < REG_FFT_CAP ? REG_FFT_LEFT : REG_FFT_CAP;
    static constexpr int REG_LEAD = DEAL ? REG_FFT : REG_LEAD_OWN;
    static constexpr int REG_SUM = DEAL ? 32 * (LEAD_WARPS + FFT_WARPS) * REG_FFT + 32 * SCM_WARPS * REG_SCM
                                        : 128 * REG_LEAD + 32 * FFT_WARPS * REG_FFT + 32 * SCM_WARPS * REG_SCM;
    // OUT_FILTER_FT: per consumer warp one output of 8 frames x its 32 bins, staged for the transposed store (pitch 34:
    // conflict-free both as rows of 32 bins and as the columns that 8 lanes (frames) x 4 bins read)
    static constexpr int FT_PITCH = 34;
    static constexpr int FT_STAGE = OUT == OUT_FILTER_FT ? SCM_WARPS * 8 * FT_PITCH : 0;   // complex
    static_assert(!REALLOC || (REG_LEAD >= 24 && REG_FFT >= 24), "setmaxnreg budgets start at 24");
    static_assert(!REALLOC || REG_SUM <= (REG_LAUNCH > 255 ? 255 : REG_LAUNCH) * THREADS,
                  "register budgets exceed the CTA's allocation");
    static_assert(!DEAL || (REALLOC && LEAD_WARPS + FFT_WARPS == 8 && WARPS == 16 && REG_LAUNCH == 128 &&
                            REG_FFT == 104 && REG_SUM == 65536),
                  "DEAL: loader + 7 FFT warps fill two warpgroups at 104 registers next to 8 SCM warps at 152");
    static_assert(DEAL || WIDE || NM != 2 || N != 512 || (FFT_WARPS == 4 && REG_SCM == 152 && REG_FFT == 176),
                  "two masks, 1-2 microphones at 512 points: 4 FFT warps at 176 registers next to SCM warps at 152");
    static_assert(!DEAL || JOBS >= FFT_WARPS, "DEAL: every FFT warp must run a job of every tile (the fill barrier)");
};

int stft_tile_frames(int n_fft, int C) { return (8 * (32 / (n_fft / 32))) / ((C + 1) / 2); }

template <int N, int C, int OUT = OUT_Y>
__host__ __device__ inline size_t smem_bytes() {
    using G = StftCfg<N, C, 1, OUT>;
    return G::NSTG * ((size_t)G::SPEC * sizeof(float2) + (size_t)G::SAMP * sizeof(float)) + (size_t)N * sizeof(float2) + 256 +
           64 * sizeof(float) + (size_t)G::FT_STAGE * sizeof(float2);
}

__device__ __forceinline__ long long range_lo(long long total, int b, int nb) { return total * b / nb; }

// Warpgroup register reallocation: grow (inc) or shrink (dec) relative to the launch allocation; the PTX
// rules make the wrong direction undefined behaviour (an illegal-instruction fault).
template <int R, int LAUNCH>
DISCO_DEV void set_maxnreg() {
    if constexpr (R > LAUNCH) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(R));
    } else if constexpr (R < LAUNCH) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(R));
    }
}

// Accumulators of one bin: per mask, C diagonal pairs (s-weighted, n-weighted) and C(C-1)/2
// complex off-diagonal sums for each of the two weights.
template <int C, int NM>
struct ScmAcc {
    static constexpr int NOFF = C * (C - 1) / 2;
    static constexpr int NO = NOFF > 0 ? NOFF : 1;
    float2 d[NM > 0 ? NM : 1][C];     // (sum m^2 |y_i|^2, sum (1-m)^2 |y_i|^2)
    float2 os[NM > 0 ? NM : 1][NO];   // sum m^2 y_i conj(y_j), i < j row-major
    float2 on[NM > 0 ? NM : 1][NO];   // sum (1-m)^2 y_i conj(y_j)
    DISCO_DEV void reset() {
#pragma unroll
        for (int q = 0; q < NM; ++q) {
#pragma unroll
            for (int i = 0; i < C; ++i) d[q][i] = make_float2(0.f, 0.f);
#pragma unroll
            for (int i = 0; i < NOFF; ++i) os[q][i] = on[q][i] = make_float2(0.f, 0.f);
        }
    }
    // one (frame, bin) point: masks m[q]
    DISCO_DEV void step(const float2 (&y)[C], const float (&m)[NM > 0 ? NM : 1]) {
        float2 ab[NM > 0 ? NM : 1];
#pragma unroll
        for (int q = 0; q < NM; ++q) {
            const float om = 1.f - m[q];
            ab[q] = make_float2(m[q] * m[q], om * om);
        }
        int o = 0;
#pragma unroll
        for (int i = 0; i < C; ++i) {
            const float dd = fmaf(y[i].x, y[i].x, y[i].y * y[i].y);
#pragma unroll
            for (int q = 0; q < NM; ++q) d[q][i] = ffma2(make_float2(dd, dd), ab[q], d[q][i]);
#pragma unroll
            for (int j = i + 1; j < C; ++j) {
                const float2 op = cmulc(y[i], y[j]);
#pragma unroll
                for (int q = 0; q < NM; ++q) {
                    os[q][o] = cfma_r(ab[q].x, op, os[q][o]);
                    on[q][o] = cfma_r(ab[q].y, op, on[q][o]);
                }
                ++o;
            }
        }
    }
    // rows of the workspace for bin f: per mask [s: C diag, NOFF x (re, im)][n: the same]
    DISCO_DEV void flush(float* out, int F) const {
        int a = 0;
#pragma unroll
        for (int q = 0; q < NM; ++q) {
#pragma unroll
            for (int i = 0; i < C; ++i) out[(size_t)(a++) * F] = d[q][i].x;
#pragma unroll
            for (int i = 0; i < NOFF; ++i) {
                out[(size_t)(a++) * F] = os[q][i].x;
                out[(size_t)(a++) * F] = os[q][i].y;
            }
#pragma unroll
            for (int i = 0; i < C; ++i) out[(size_t)(a++) * F] = d[q][i].y;
#pragma unroll
            for (int i = 0; i < NOFF; ++i) {
                out[(size_t)(a++) * F] = on[q][i].x;
                out[(size_t)(a++) * F] = on[q][i].y;
            }
        }
    }
};

// Per-role cycle accounting, compiled in only with -DDISCO_ROLE_CLOCKS (scripts/role_clocks.py builds that variant
// into a library of its own).  Lane 0 of every working warp records clock64 cycles spent in each kind of mbarrier
// wait, its total cycles from the role's start to its end, and the tiles (and, for the FFT warps, jobs) it processed
// into g_role_clocks[cta][warp][RC_SLOTS] of the last launch; disco_role_clocks copies the buffer out.  Without the
// switch RoleClocks is empty and wait() is mbar_wait.
enum : int { RC_SAMP_FULL = 0, RC_SAMP_EMPTY = 1, RC_SPEC_FULL = 2, RC_SPEC_EMPTY = 3 };
enum : int { RC_ROLE_LOADER = 1, RC_ROLE_FFT = 2, RC_ROLE_SCM = 3 };
#ifdef DISCO_ROLE_CLOCKS
// slots: role, tiles, jobs, total cycles, then the wait cycles of samp_full, samp_empty, spec_full, spec_empty
constexpr int RC_MAX_CTAS = 1024, RC_SLOTS = 8;
__device__ unsigned long long g_role_clocks[RC_MAX_CTAS * 32 * RC_SLOTS];
DISCO_DEV long long rc_clock() {
    long long t;
    asm volatile("mov.u64 %0, %%clock64;" : "=l"(t)::"memory");
    return t;
}
struct RoleClocks {
    long long t0, w[4] = {0, 0, 0, 0};
    int tiles = 0, jobs = 0;
    DISCO_DEV RoleClocks() : t0(rc_clock()) {}
    DISCO_DEV void wait(int k, uint64_t* bar, uint32_t parity) {
        const long long a = rc_clock();
        mbar_wait(bar, parity);
        w[k] += rc_clock() - a;
    }
    DISCO_DEV void tile() { ++tiles; }
    DISCO_DEV void job() { ++jobs; }
    DISCO_DEV void done(int role) {
        const long long t1 = rc_clock();
        if ((threadIdx.x & 31) != 0 || blockIdx.x >= RC_MAX_CTAS) return;
        unsigned long long* o = g_role_clocks + ((size_t)blockIdx.x * 32 + (threadIdx.x >> 5)) * RC_SLOTS;
        o[0] = role;
        o[1] = tiles;
        o[2] = jobs;
        o[3] = t1 - t0;
        for (int k = 0; k < 4; ++k) o[4 + k] = w[k];
    }
};
#else
struct RoleClocks {
    DISCO_DEV void wait(int, uint64_t* bar, uint32_t parity) { mbar_wait(bar, parity); }
    DISCO_DEV void tile() {}
    DISCO_DEV void job() {}
    DISCO_DEV void done(int) {}
};
#endif

template <int OUT>
struct StftParam {
    using type = StftArgs;
};
template <>
struct StftParam<OUT_FILTER> {
    using type = StftFilterArgs;
};
template <>
struct StftParam<OUT_FILTER_FT> {
    using type = StftFilterArgs;
};

template <int N, int C, int NM, int OUT>
__global__ void __launch_bounds__(StftCfg<N, C, NM, OUT>::THREADS, 1) stft_scm_kernel(typename StftParam<OUT>::type p) {
    using G = StftCfg<N, C, NM, OUT>;
    constexpr int RA = G::RA, NB = G::NB, H = G::H, F = G::F, ROWP = G::ROWP, P = G::P, TT = G::TT;
    constexpr int SAMP = G::SAMP;
    constexpr int NACC = NM * 2 * C * C;
    constexpr int NMX = NM > 0 ? NM : 1;
    constexpr bool SCM = NM > 0;
    constexpr bool STORE_Y = OUT == OUT_Y, FILT = G::FILT, FT = OUT == OUT_FILTER_FT;
    static_assert(!FILT || NM == 0, "the filter consumer accumulates no statistics");
    constexpr int MCAP = (G::REALLOC && G::REG_SCM >= 152 && !G::WIDE) ? 16 : 8;     // mask values in flight per thread
    constexpr int MC = (TT * NM <= MCAP) ? TT : ((MCAP / NMX) < TT ? (MCAP / NMX) : TT);   // frames per mask chunk
    constexpr int NCH = (TT + MC - 1) / MC;

    extern __shared__ __align__(128) unsigned char smem_raw[];
    constexpr int NSTG = G::NSTG;
    float2* spec = reinterpret_cast<float2*>(smem_raw);                  // [NSTG][ITEMS][ROWP]
    float* samp = reinterpret_cast<float*>(spec + NSTG * G::SPEC);       // [NSTG][C][(TT+1)*H]
    float2* tw = reinterpret_cast<float2*>(samp + NSTG * SAMP);          // [RA][32]
    uint64_t* bars = reinterpret_cast<uint64_t*>(tw + N);
    uint64_t* samp_full = bars;               // [NSTG]  loader -> FFT   (1 arrival + TMA bytes)
    uint64_t* samp_empty = bars + NSTG;       // [NSTG]  FFT -> loader   (FFT_ARRIVALS: per warp, or per job with DEAL)
    uint64_t* spec_full = bars + 2 * NSTG;    // [NSTG]  FFT -> SCM      (FFT_ARRIVALS)
    uint64_t* spec_empty = bars + 3 * NSTG;   // [NSTG]  SCM -> FFT      (SCM_WARPS + 1 arrivals)
    float* nyq = reinterpret_cast<float*>(bars + 32);   // [TT * C <= 64] Nyquist-bin values of the current tile
    float2* ft_stage = reinterpret_cast<float2*>(nyq + 64);   // OUT_FILTER_FT: [SCM_WARPS][8][FT_PITCH]
    static_assert(4 * NSTG <= 32, "barrier area");
    static_assert(TT * C <= 64 && TT <= 32, "Nyquist staging");

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int L = p.L, T = p.T;
    const int tiles_per_grp = (T + TT - 1) / TT;
    const long long total = (long long)p.n_grp * tiles_per_grp;
    const long long lo = range_lo(total, blockIdx.x, gridDim.x), hi = range_lo(total, blockIdx.x + 1, gridDim.x);
    const int n_it = (int)(hi - lo);
    if (n_it <= 0) return;

    for (int i = tid; i < N; i += blockDim.x) tw[i] = p.twiddle[i];
    if (tid == 0) {
        for (int s = 0; s < NSTG; ++s) {
            mbar_init(&samp_full[s], 1);
            mbar_init(&samp_empty[s], G::FFT_ARRIVALS);
            mbar_init(&spec_full[s], G::FFT_ARRIVALS);
            mbar_init(&spec_empty[s], G::SCM_WARPS + 1);
        }
        fence_mbar_init();
    }
    __syncthreads();

    auto tile_of = [&](int it, int& grp, int& t0) {
        const long long i = lo + it;
        grp = (int)(i / tiles_per_grp);
        t0 = (int)(i % tiles_per_grp) * TT;
    };
    // The loader and the consumer warps walk their tiles with a cursor, (group, tile within the group), that starts
    // at the range's first tile (grp_lo, tg_lo) and advances tile by tile, so that no tile costs them a 64-bit
    // division (but the 1024-point SCM consumers, below).  The FFT warps still divide once per tile, in enter_tile.
    auto next_tile = [&](int& grp, int& tg) {
        if (++tg == tiles_per_grp) {
            tg = 0;
            ++grp;
        }
    };
    auto seg_slot = [&](int grp) { return blockIdx.x - seg_slots(grp, tiles_per_grp, total, gridDim.x).first; };
    auto mask_at = [&](int q, int grp, int t, int f) {
        const float* m = q == 0 ? p.mask : p.mask2;
        return p.mask_ft ? m[((size_t)grp * F + f) * T + t] : m[((size_t)grp * T + t) * F + f];
    };

    // role layout: lead warp(s), then the FFT warps, then the SCM warps
    constexpr int FFT_WARP0 = G::LEAD_WARPS;
    constexpr int SCM_WARP0 = G::LEAD_WARPS + G::FFT_WARPS;
    const bool is_fft = warp >= FFT_WARP0 && warp < FFT_WARP0 + G::FFT_WARPS;
    if constexpr (G::DEAL) {   // loader + FFT warps: one budget over both leading warpgroups
        if (warp < SCM_WARP0) set_maxnreg<G::REG_FFT, G::REG_LAUNCH>();
    }
    if (warp < G::LEAD_WARPS) {
        if (G::REALLOC && !G::DEAL) set_maxnreg<G::REG_LEAD, G::REG_LAUNCH>();
        if (warp != 0) return;
        // =========================================================== LOADER (+ Nyquist bin)
        // Per tile `it`: stage tile it + NSTG - 1, then the Nyquist work of tile it.  Nothing on this chain divides by
        // the tile count or waits for a global load: two tile cursors (the next tile to stage, the Nyquist tile) walk
        // the range, the Nyquist masks are loaded a tile ahead and the Nyquist filter taps when the staging enters a
        // group.  (Staging as soon as samp_empty allows instead, ahead of the Nyquist work, was slower: DESIGN.md 4.1.)
        RoleClocks rc;
        const int grp_lo = (int)(lo / tiles_per_grp), tg_lo = (int)(lo % tiles_per_grp);
        auto stage_tile = [&](int it, int grp, int t0) {
            const int nfr = min(TT, T - t0), s = it % NSTG, c_valid = min(C, p.n_sig - grp * C);
            rc.wait(RC_SAMP_EMPTY, &samp_empty[s], ((it / NSTG) & 1) ^ 1);
            const float* xg = p.x + (size_t)grp * C * L;
            float* dst = samp + s * SAMP;
            const int s0 = t0 * H - H;
            // the in-range part [k_lo, k_hi) of the tile's samples comes by TMA; the FFT warps fill the
            // mirrored samples of edge tiles (at most one hop per side) themselves
            const int cnt = (nfr + 1) * H;
            const int k_lo = max(0, -s0), k_hi = min(cnt, L - s0);
            if (lane == 0) {
                if (p.use_tma && k_hi > k_lo) {
                    fence_proxy_async();
                    mbar_expect_tx(&samp_full[s], (uint32_t)(c_valid * (k_hi - k_lo) * sizeof(float)));
                    for (int c = 0; c < c_valid; ++c)
                        tma_load_1d(dst + c * (TT + 1) * H + k_lo, xg + (size_t)c * L + s0 + k_lo,
                                    (uint32_t)((k_hi - k_lo) * sizeof(float)), &samp_full[s]);
                } else {
                    mbar_arrive(&samp_full[s]);
                }
            }
        };
        // Nyquist bin: the spectrum is real there, so an SCM entry is a plain product y_i y_j.
        // lane l <-> (frame l / C, channel l % C) for the un-mixing and the Y store,
        // lane p <-> channel pair p (and p + 32 when C = 8) for the accumulation.
        constexpr int NP = C * (C + 1) / 2;
        constexpr int NSLOT = NP > 32 ? 2 : 1;
        int pi[NSLOT], pj[NSLOT], row[NSLOT];
#pragma unroll
        for (int u = 0; u < NSLOT; ++u) {
            const int pp = min(lane + 32 * u, NP - 1);
            if (pp < C) {
                pi[u] = pj[u] = pp;
                row[u] = pp;
            } else {
                int o = pp - C, i = 0, n = C - 1;
                while (o >= n) {
                    o -= n;
                    --n;
                    ++i;
                }
                pi[u] = i;
                pj[u] = i + 1 + o;
                row[u] = C + 2 * (pp - C);
            }
        }
        float as[NMX][NSLOT], an[NMX][NSLOT];
        auto nyq_reset = [&]() {
#pragma unroll
            for (int q = 0; q < NMX; ++q)
#pragma unroll
                for (int u = 0; u < NSLOT; ++u) as[q][u] = an[q][u] = 0.f;
        };
        nyq_reset();
        int st_grp = grp_lo, st_tg = tg_lo;       // the next tile to stage
        int ny_grp = grp_lo, ny_tg = tg_lo;       // the Nyquist tile `it` below
        // filter consumer: the Nyquist-bin taps of the Nyquist tile's group (nw), and those of the last staged tile's
        // group (pw), loaded when the staging enters the group, a tile before the Nyquist work needs them; lane <-> frame
        constexpr int NW = FILT ? C : 1;
        float2 nw1[NW], nw2[NW], pw1[NW], pw2[NW];
        int nw_grp = grp_lo, pw_grp = grp_lo;
        static_assert(NSTG == 2, "a new group's Nyquist taps are those of the last staged tile");
        auto load_taps = [&](float2 (&w1)[NW], float2 (&w2)[NW], int grp) {
            if constexpr (FILT) {
#pragma unroll
                for (int c = 0; c < C; ++c) {
                    w1[c] = p.W1[((size_t)grp * F + F - 1) * C + c];
                    w2[c] = p.W2[((size_t)grp * F + F - 1) * C + c];
                }
            }
        };
        auto stage_next = [&](int it) {
            if (FILT && st_grp != pw_grp) {
                load_taps(pw1, pw2, st_grp);
                pw_grp = st_grp;
            }
            stage_tile(it, st_grp, st_tg * TT);
            next_tile(st_grp, st_tg);
        };
        // pass 1: the Nyquist tile's mask values (lane <-> frame), loaded one tile ahead of their use
        float mq[NMX];
        auto load_masks = [&]() {
            const int t0 = ny_tg * TT, nfr = min(TT, T - t0);
#pragma unroll
            for (int q = 0; q < NMX; ++q) mq[q] = (SCM && lane < nfr) ? mask_at(q, ny_grp, t0 + lane, F - 1) : 0.f;
        };
        for (int i = 0; i < NSTG - 1; ++i)
            if (i < n_it) stage_next(i);
        if constexpr (FILT)
            load_taps(nw1, nw2, grp_lo);
        else
            load_masks();
        int ny_slot = SCM ? seg_slot(grp_lo) : 0;   // the CTA's partial-sum slot of the Nyquist tile's group (0 for a later group)
        for (int it = 0; it < n_it; ++it) {
            const int s = it % NSTG;
            const uint32_t ph = (it / NSTG) & 1;
            if constexpr (FILT) {
                if (ny_grp != nw_grp) {   // a CTA's tile range may cross groups; tile it was the last one staged
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        nw1[c] = pw1[c];
                        nw2[c] = pw2[c];
                    }
                    nw_grp = ny_grp;
                }
            }
            if (it + NSTG - 1 < n_it) stage_next(it + NSTG - 1);
            const int grp = ny_grp, t0 = ny_tg * TT;
            const int nfr = min(TT, T - t0), c_valid = min(C, p.n_sig - grp * C);
            if constexpr (FILT) {
                rc.wait(RC_SPEC_FULL, &spec_full[s], ph);
                if (lane < nfr) {
                    // the Nyquist spectrum is real; it goes through the complex helpers as (yv, 0), the value
                    // disco_stft stores there, so z, zn, yf match filter_dual on a stored Y bit for bit
                    float2 y[C];
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        const float2 z = spec[s * G::SPEC + (size_t)(lane * P + c / 2) * ROWP + N / 2];
                        y[c] = make_float2(stft_nyquist(z, c & 1), 0.f);
                    }
                    float2 z, zn, yf;
                    dual_filter<C>(nw1, nw2, y, p.ref, z, zn, yf);
                    const size_t o = FT ? ((size_t)grp * F + F - 1) * T + t0 + lane : ((size_t)grp * T + t0 + lane) * F + (F - 1);
                    __stcs(p.z + o, z);
                    if (p.zn) __stcs(p.zn + o, zn);
                    __stcs(p.yf + o, yf);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&spec_empty[s]);
            } else {
                rc.wait(RC_SPEC_FULL, &spec_full[s], ph);
#pragma unroll
                for (int r = lane; r < TT * C; r += 32) {
                    const int tl_l = r / C, c_l = r % C;
                    float yv = 0.f;
                    if (tl_l < nfr && c_l < c_valid) {
                        const float2 z = spec[s * G::SPEC + (size_t)(tl_l * P + c_l / 2) * ROWP + N / 2];
                        // stft_nyquist(z, c_l & 1), written out: the helper changes this path's machine code
                        yv = (c_l & 1) ? z.y + z.y : z.x + z.x;
                        if (STORE_Y) p.Y[(((size_t)grp * C + c_l) * T + t0 + tl_l) * F + (F - 1)] = make_float2(yv, 0.f);
                    }
                    nyq[r] = yv;
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&spec_empty[s]);
                if (SCM) {
#pragma unroll
                    for (int tl = 0; tl < TT; ++tl) {
                        if (tl < nfr) {   // warp-uniform
                            float pr[NSLOT];
#pragma unroll
                            for (int u = 0; u < NSLOT; ++u)
                                pr[u] = nyq[tl * C + pi[u]] * nyq[tl * C + pj[u]];
#pragma unroll
                            for (int q = 0; q < NM; ++q) {
                                const float m = __shfl_sync(0xffffffffu, mq[q], tl), om = 1.f - m;
                                const float a = m * m, b = om * om;
#pragma unroll
                                for (int u = 0; u < NSLOT; ++u) {
                                    as[q][u] = fmaf(a, pr[u], as[q][u]);
                                    an[q][u] = fmaf(b, pr[u], an[q][u]);
                                }
                            }
                        }
                    }
                    const bool seg_end = (it + 1 == n_it) || (ny_tg + 1 == tiles_per_grp);
                    if (seg_end) {
                        float* out = p.part + ((size_t)grp * p.slots_per_grp + ny_slot) * NACC * F + (F - 1);
#pragma unroll
                        for (int u = 0; u < NSLOT; ++u) {
                            const int pp = lane + 32 * u;
                            if (pp < NP) {
#pragma unroll
                                for (int q = 0; q < NM; ++q) {
                                    float* os = out + (size_t)(q * 2 * C * C) * F;
                                    float* on = os + (size_t)(C * C) * F;
                                    os[(size_t)row[u] * F] = as[q][u];
                                    on[(size_t)row[u] * F] = an[q][u];
                                    if (pp >= C) {
                                        os[(size_t)(row[u] + 1) * F] = 0.f;
                                        on[(size_t)(row[u] + 1) * F] = 0.f;
                                    }
                                }
                            }
                        }
                        nyq_reset();
                        ny_slot = 0;   // this CTA holds the first tile of every later group in its range
                    }
                }
                __syncwarp();   // nyq[] is rewritten by the next tile
            }
            rc.tile();
            next_tile(ny_grp, ny_tg);
            if constexpr (!FILT) {
                if (it + 1 < n_it) load_masks();
            }
        }
        rc.done(RC_ROLE_LOADER);
    } else if (is_fft) {
        if (G::REALLOC && !G::DEAL) set_maxnreg<G::REG_FFT, G::REG_LAUNCH>();
        // =========================================================== FFT warps
        // f0 = wf / FFT_WARPS is always 0 and w = wf % FFT_WARPS always wf.  They stay runtime values on purpose: with
        // a constant first tile and a constant barrier id nvcc schedules the FFT loop differently, and the cfg2 / cfg3
        // steps ran 0.4 % / 0.3 % slower (stft_scm<512,4,1> 1 %) on an H100 SXM (700 W)
        const int wf = warp - FFT_WARP0, f0 = wf / G::FFT_WARPS, w = wf % G::FFT_WARPS;
        constexpr bool WINREG = (RA <= 16);
        float win[WINREG ? RA : 1];   // window for n = lane + 32 j (pre-scaled by 1/2 for the two-for-one split)
        if (WINREG) {
#pragma unroll
            for (int j = 0; j < RA; ++j) win[j] = p.window[lane + 32 * j];
        }
        RoleClocks rc;
        // the tile an FFT warp is working on: its stages and extent
        struct FftTile {
            int s, nfr, c_valid;
            const float* sm;
            bool full;
        };
        // start tile `it`: wait for its samples, fill the reflect padding of edge tiles (every FFT warp takes part),
        // wait for its spectrum stage
        auto enter_tile = [&](int it) {
            int grp, t0;
            tile_of(it, grp, t0);
            const int nfr = min(TT, T - t0), s = it % NSTG, c_valid = min(C, p.n_sig - grp * C);
            const uint32_t ph = (it / NSTG) & 1;
            const float* sm = samp + s * SAMP;
            rc.wait(RC_SAMP_FULL, &samp_full[s], ph);
            {
                const int s0 = t0 * H - H;
                const int cnt = (nfr + 1) * H;
                int k_lo = max(0, -s0), k_hi = min(cnt, L - s0);   // [k_lo, k_hi) arrived by TMA
                if (!p.use_tma || k_hi <= k_lo) k_lo = k_hi = 0;
                const int n_fill = cnt - (k_hi - k_lo);
                if (n_fill > 0) {   // CTA-uniform: cooperative scalar fill (reflect padding) by the FFT warps
                    const float* xg = p.x + (size_t)grp * C * L;
                    float* dst = samp + s * SAMP;
                    named_bar_sync(1 + f0, 32 * G::FFT_WARPS);        // every FFT warp is done with this stage
                    // (DEAL: not unrolled, which helps keep the 104-register FFT warps free of spills; edge tiles only)
                    for (int c = 0; c < c_valid; ++c)
#pragma unroll(G::DEAL ? 1 : 4)
                        for (int q = w * 32 + lane; q < n_fill; q += 32 * G::FFT_WARPS) {
                            const int k = q < k_lo ? q : q + (k_hi - k_lo);
                            const int sidx = reflect_index(s0 + k, L);
                            float v = 0.f;
                            if (sidx >= 0 && sidx < L) v = xg[(size_t)c * L + sidx];
                            dst[c * (TT + 1) * H + k] = v;
                        }
                    named_bar_sync(1 + f0, 32 * G::FFT_WARPS);
                }
            }
            rc.wait(RC_SPEC_EMPTY, &spec_empty[s], ph ^ 1);   // spectrum stage s free (tile it-2 consumed)
            const bool full = (nfr == TT && c_valid == C && (C % 2 == 0) && (G::ITEMS % P == 0));
            return FftTile{s, nfr, c_valid, sm, full};
        };
        // job jb of tile tc; `release`: the warp's last job of the tile, after which it signals samp_empty
        auto run_job = [&](const FftTile& tc, int jb, bool release) {
            const int s = tc.s, nfr = tc.nfr, c_valid = tc.c_valid;
            const float* sm = tc.sm;
            const bool full = tc.full;
            float2* job = spec + s * G::SPEC + (size_t)jb * NB * ROWP;
            // inter-pass twiddles W_N^(lane k1): fetched once per job, shared by its transforms
            constexpr bool TWREG = (RA <= 16);
            float2 twr[TWREG ? RA : 1];
            if (TWREG) {
#pragma unroll
                for (int k1 = 1; k1 < RA; ++k1) twr[k1] = tw[k1 * 32 + lane];
            }
#pragma unroll
            for (int q = 0; q < NB; ++q) {
                const int item = jb * NB + q;
                const int tl = item / P, pr = item % P;
                const int ca = 2 * pr, cb = 2 * pr + 1;
                const float* xa = sm + ca * (TT + 1) * H + tl * H + lane;
                const float* xb = sm + cb * (TT + 1) * H + tl * H + lane;
                float2 v[RA];
                if (full || (tl < nfr && cb < c_valid)) {
#pragma unroll
                    for (int j = 0; j < RA; ++j) {
                        const float wj = WINREG ? win[j] : p.window[lane + 32 * j];
                        v[j] = fmul2(make_float2(xa[32 * j], xb[32 * j]), make_float2(wj, wj));
                    }
                } else if (tl < nfr && ca < c_valid) {
#pragma unroll
                    for (int j = 0; j < RA; ++j) {
                        const float wj = WINREG ? win[j] : p.window[lane + 32 * j];
                        v[j] = make_float2(xa[32 * j] * wj, 0.f);
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < RA; ++j) v[j] = make_float2(0.f, 0.f);
                }
                if (release && q == NB - 1) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&samp_empty[s]);   // all samples of this warp are in registers
                }
                stft_pass1<RA, TWREG>(v, job, q, lane, twr, tw);
            }
            stft_pass2<RA>(job, lane);
            rc.job();
        };
        if constexpr (G::DEAL) {
            // job j of the CTA's tile stream (tile j / JOBS, job j % JOBS of it) runs on warp j mod FFT_WARPS; with
            // JOBS >= FFT_WARPS every warp has a job in every tile, so each enters every tile (and its fill) in order.
            // samp_empty and spec_full count job arrivals.
            FftTile tc{};
            int cur = -1;
#pragma unroll 1
            for (int j = w; j < n_it * G::JOBS; j += G::FFT_WARPS) {
                const int it = j / G::JOBS;
                if (it != cur) {
                    tc = enter_tile(it);
                    cur = it;
                    rc.tile();
                }
                run_job(tc, j % G::JOBS, true);
                __syncwarp();
                if (lane == 0) mbar_arrive(&spec_full[tc.s]);
            }
        } else {
            for (int it = f0; it < n_it; ++it) {
                const FftTile tc = enter_tile(it);
#pragma unroll 1
                for (int jj = 0; jj < G::JPW; ++jj) run_job(tc, w * G::JPW + jj, jj == G::JPW - 1);
                __syncwarp();
                if (lane == 0) mbar_arrive(&spec_full[tc.s]);
                rc.tile();
            }
        }
        rc.done(RC_ROLE_FFT);
    } else {
        if (G::REALLOC) set_maxnreg<G::REG_SCM, G::REG_LAUNCH>();
        // =========================================================== SCM warps: thread <-> bin f
        const int f = (warp - SCM_WARP0) * 32 + lane;   // 0 .. N/2 - 1
        const int fn = (N - f) & (N - 1);
        RoleClocks rc;
        if constexpr (FILT) {
            // =========================================================== filter consumer: thread <-> bin f
            float2 w1[C], w2[C];
            int w_grp = -1, grp = (int)(lo / tiles_per_grp), tg = (int)(lo % tiles_per_grp);
            for (int it = 0; it < n_it; ++it, next_tile(grp, tg)) {
                const int t0 = tg * TT;
                const int nfr = min(TT, T - t0), s = it % NSTG;
                if (grp != w_grp) {   // a CTA's tile range may cross groups
#pragma unroll
                    for (int c = 0; c < C; ++c) {
                        w1[c] = p.W1[((size_t)grp * F + f) * C + c];
                        w2[c] = p.W2[((size_t)grp * F + f) * C + c];
                    }
                    w_grp = grp;
                }
                const float2* stage = spec + s * G::SPEC;
                // un-mix as below and filter frame tl of bin f
                auto point = [&](int tl, float2& z, float2& zn, float2& yf) {
                    float2 y[C];
#pragma unroll
                    for (int pr = 0; pr < P; ++pr) {
                        const float2* row = stage + (size_t)(tl * P + pr) * ROWP;
                        float2 ya, yb;
                        stft_unmix(row[f], row[fn], ya, yb);
                        y[2 * pr] = ya;
                        if (2 * pr + 1 < C) y[2 * pr + 1] = yb;
                    }
                    dual_filter<C>(w1, w2, y, p.ref, z, zn, yf);
                };
                rc.wait(RC_SPEC_FULL, &spec_full[s], (it / NSTG) & 1);
                if constexpr (!FT) {
                    // frame-major rows, coalesced over the bins of a warp
                    const size_t o = ((size_t)grp * T + t0) * F + f;
#pragma unroll 8
                    for (int tl = 0; tl < TT; ++tl) {
                        if (tl < nfr) {
                            float2 z, zn, yf;
                            point(tl, z, zn, yf);
                            __stcs(p.z + o + (size_t)tl * F, z);
                            if (p.zn) __stcs(p.zn + o + (size_t)tl * F, zn);
                            __stcs(p.yf + o + (size_t)tl * F, yf);
                        }
                    }
                } else {
                    // (F, T) layout: 8 frames at a time, one output after the other through the warp's staging rows,
                    // then lanes <-> (frame lane % 8, bin lane / 8 + 4 k): 64 contiguous bytes per bin and store
                    float2* st = ft_stage + (warp - SCM_WARP0) * 8 * G::FT_PITCH;
                    const int fw = (warp - SCM_WARP0) * 32, jl = lane & 7;
                    auto flush = [&](float2* out, int c8) {
                        __syncwarp();
                        if (c8 + jl < nfr) {
#pragma unroll
                            for (int k = 0; k < 8; ++k) {
                                const int i = (lane >> 3) + 4 * k;
                                __stcs(out + ((size_t)grp * F + fw + i) * T + t0 + c8 + jl, st[jl * G::FT_PITCH + i]);
                            }
                        }
                        __syncwarp();
                    };
#pragma unroll 1
                    for (int c8 = 0; c8 < nfr; c8 += 8) {
                        float2 znr[8], yfr[8];
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            float2 z = make_float2(0.f, 0.f);
                            znr[j] = yfr[j] = z;
                            if (c8 + j < nfr) point(c8 + j, z, znr[j], yfr[j]);
                            st[j * G::FT_PITCH + lane] = z;
                        }
                        flush(p.z, c8);
                        if (p.zn) {
#pragma unroll
                            for (int j = 0; j < 8; ++j) st[j * G::FT_PITCH + lane] = znr[j];
                            flush(p.zn, c8);
                        }
#pragma unroll
                        for (int j = 0; j < 8; ++j) st[j * G::FT_PITCH + lane] = yfr[j];
                        flush(p.yf, c8);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&spec_empty[s]);
                rc.tile();
            }
            rc.done(RC_ROLE_SCM);
            return;
        }
        ScmAcc<C, NM> acc;
        float mk[NMX][MC];
        // masks of chunk `ch` of the tile at frame t0 of group grp: one base pointer per mask, frame stride hoisted
        // (frame-major: F floats, (F, T) layout: 1).  A chunk whose frames all exist (every chunk but the last of a
        // group's last tile) loads with compile-time offsets and no per-frame bounds test.  That second copy of the
        // loads is kept to the variants of at most 512 points and 4 microphones, whose consumer warps have registers
        // to spare; the others load as before.
        constexpr bool MFAST = !G::WIDE && N <= 512;
        const int m_st = p.mask_ft ? 1 : F;
        const size_t m_f = p.mask_ft ? (size_t)f * T : (size_t)f;
        auto load_mask = [&](int grp, int t0, int ch) {
            const size_t base = (size_t)grp * T * F + m_f + (size_t)(t0 + ch * MC) * m_st;
            if (MFAST && (ch + 1) * MC <= TT && t0 + (ch + 1) * MC <= T) {
#pragma unroll
                for (int q = 0; q < NM; ++q) {
                    const float* mb = (q == 0 ? p.mask : p.mask2) + base;
                    if (p.mask_ft) {
#pragma unroll
                        for (int i = 0; i < MC; ++i) mk[q][i] = mb[i];
                    } else {
#pragma unroll
                        for (int i = 0; i < MC; ++i) mk[q][i] = mb[i * F];
                    }
                }
                return;
            }
#pragma unroll
            for (int q = 0; q < NM; ++q) {
                const float* mb = (q == 0 ? p.mask : p.mask2) + base;
#pragma unroll
                for (int i = 0; i < MC; ++i)
                    mk[q][i] = (ch * MC + i < TT && t0 + ch * MC + i < T) ? mb[i * m_st] : 0.f;
            }
        };
        int grp = (int)(lo / tiles_per_grp), tg = (int)(lo % tiles_per_grp);
        if (SCM) {
            acc.reset();
            load_mask(grp, tg * TT, 0);
        }
        // The 1024-point variants, whose FFT warps spill already, keep locating each tile by division: the cursor held
        // across their tile loop costs them spill traffic.
        constexpr bool CURSOR = N <= 512;
        for (int it = 0; it < n_it; ++it) {
            if constexpr (!CURSOR) {
                grp = (int)((lo + it) / tiles_per_grp);
                tg = (int)((lo + it) % tiles_per_grp);
            }
            const int t0 = tg * TT;
            const int nfr = min(TT, T - t0), s = it % NSTG, c_valid = min(C, p.n_sig - grp * C);
            const float2* stage = spec + s * G::SPEC;
            float2* ybase = p.Y + ((size_t)grp * C * T + t0) * F + f;
            const size_t cstride = (size_t)T * F;
            const bool full = (nfr == TT && c_valid == C);
#pragma unroll
            for (int ch = 0; ch < NCH; ++ch) {
                float mcur[NMX][MC];
#pragma unroll
                for (int q = 0; q < NMX; ++q)
#pragma unroll
                    for (int i = 0; i < MC; ++i) mcur[q][i] = SCM ? mk[q][i] : 0.f;
                if (SCM) {   // next chunk's masks (none past the CTA's last tile): in flight while this chunk is processed
                    if (ch + 1 < NCH)
                        load_mask(grp, t0, ch + 1);
                    else if (it + 1 < n_it)
                        load_mask(tg + 1 < tiles_per_grp ? grp : grp + 1, tg + 1 < tiles_per_grp ? (tg + 1) * TT : 0, 0);
                }
                if (ch == 0) rc.wait(RC_SPEC_FULL, &spec_full[s], (it / NSTG) & 1);
#pragma unroll
                for (int i = 0; i < MC; ++i) {
                    const int tl = ch * MC + i;
                    if (tl < TT && (full || tl < nfr)) {
                        // un-mix the two-for-one spectra
                        float2 y[C];
#pragma unroll
                        for (int pr = 0; pr < P; ++pr) {
                            const float2* row = stage + (size_t)(tl * P + pr) * ROWP;
                            float2 ya, yb;
                            stft_unmix(row[f], row[fn], ya, yb);
                            y[2 * pr] = ya;
                            if (2 * pr + 1 < C) y[2 * pr + 1] = yb;
                        }
                        if (STORE_Y) {
#pragma unroll
                            for (int c = 0; c < C; ++c)
                                if (full || c < c_valid) __stcs(ybase + c * cstride + tl * F, y[c]);
                        }
                        if (SCM) {
                            float m[NMX];
#pragma unroll
                            for (int q = 0; q < NMX; ++q) m[q] = mcur[q][i];
                            acc.step(y, m);
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&spec_empty[s]);
            const bool seg_end = (it + 1 == n_it) || (tg + 1 == tiles_per_grp);
            if (SCM && seg_end) {
                acc.flush(p.part + ((size_t)grp * p.slots_per_grp + seg_slot(grp)) * NACC * F + f, F);
                acc.reset();
            }
            rc.tile();
            next_tile(grp, tg);
        }
        rc.done(RC_ROLE_SCM);
    }
}

// Reduce the (group, CTA) segment partials of mask set `set` in fixed slot order, scale by 1/T, expand
// to full Hermitian matrices Rss, Rnn [n_grp][F][C][C] complex64 (R[i][j] = mean_t a_i conj(a_j),
// np.outer convention).  One block per group, one thread per bin: the loads of a thread are
// independent (coalesced over bins), so the kernel costs about one memory round trip.
template <int C>
__global__ void __launch_bounds__(288) scm_finalize_kernel(const float* __restrict__ part, float2* __restrict__ Rss,
                                                           float2* __restrict__ Rnn, int n_grp, int slots_per_grp,
                                                           int tiles_per_grp, int n_cta, int F, float inv_T, int n_set,
                                                           int set) {
    constexpr int NA = 2 * C * C;
    const int g = blockIdx.x;
    const long long total = (long long)n_grp * tiles_per_grp;
    const int n_slot = seg_slots(g, tiles_per_grp, total, n_cta).count();
    const size_t slot_stride = (size_t)n_set * NA * F;
    for (int f = threadIdx.x; f < F; f += blockDim.x) {
        const float* base = part + (size_t)g * slots_per_grp * slot_stride + (size_t)set * NA * F + f;
#pragma unroll 1
        for (int which = 0; which < 2; ++which) {
            float acc[C * C];
#pragma unroll
            for (int a = 0; a < C * C; ++a) acc[a] = 0.f;
            for (int sl = 0; sl < n_slot; ++sl) {
#pragma unroll
                for (int a = 0; a < C * C; ++a) acc[a] += __ldg(base + sl * slot_stride + (size_t)(which * C * C + a) * F);
            }
            float2* R = (which == 0 ? Rss : Rnn) + ((size_t)g * F + f) * C * C;
            int o = 0;
#pragma unroll
            for (int i = 0; i < C; ++i) {
                R[i * C + i] = make_float2(acc[i] * inv_T, 0.f);
#pragma unroll
                for (int j = i + 1; j < C; ++j) {
                    const float re = acc[C + 2 * o] * inv_T, im = acc[C + 2 * o + 1] * inv_T;
                    R[i * C + j] = make_float2(re, im);
                    R[j * C + i] = make_float2(re, -im);
                    ++o;
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------ host side
int stft_tiles_per_grp(int n_fft, int C, int T) {
    const int tt = stft_tile_frames(n_fft, C);
    return (T + tt - 1) / tt;
}

bool stft_scm_supported(int n_fft, int C, int n_mask) {
    if (C < 1 || C > 8 || n_mask < 0 || n_mask > 2) return false;
    if (n_fft != 256 && n_fft != 512 && n_fft != 1024) return false;
    if (C > 4 && (n_mask == 2 || n_fft == 1024)) return false;   // 128 accumulators per bin are the register limit
    if (n_mask == 2 && n_fft == 1024) return false;
    if (n_mask == 0 && C > 4) return false;   // the plain STFT (disco_stft) groups its signals by at most 4
    return true;
}

template <int N, int C, int NM, int OUT = OUT_Y>
static cudaError_t launch_one(const typename StftParam<OUT>::type& a, int n_cta, cudaStream_t st) {
    using G = StftCfg<N, C, NM, OUT>;
    auto kern = stft_scm_kernel<N, C, NM, OUT>;
    const size_t smem = smem_bytes<N, C, OUT>();
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (G::REALLOC) {   // setmaxnreg.inc would wait forever if the launch allocation were smaller than the budgets
        cudaFuncAttributes fa;
        e = cudaFuncGetAttributes(&fa, kern);
        if (e != cudaSuccess) return e;
        if ((long long)fa.numRegs * G::THREADS < G::REG_SUM) return cudaErrorLaunchOutOfResources;
    }
    kern<<<n_cta, G::THREADS, smem, st>>>(a);
    return cudaGetLastError();
}

template <int N, int C>
static cudaError_t launch_nm(const StftArgs& a, int nm, int n_cta, cudaStream_t st) {
    // the plain STFT (disco_stft) groups its signals by at most 4, so no group of 5..8 runs without a mask
    if constexpr (C <= 4) {
        if (nm == 0) return launch_one<N, C, 0>(a, n_cta, st);
    }
    if (nm == 1) return launch_one<N, C, 1>(a, n_cta, st);
    if constexpr (C <= 4 && N <= 512) {
        if (nm == 2) return a.Y ? launch_one<N, C, 2>(a, n_cta, st) : launch_one<N, C, 2, OUT_NONE>(a, n_cta, st);
    }
    return cudaErrorInvalidValue;
}

template <int N>
static cudaError_t launch_c(const StftArgs& a, int C, int nm, int n_cta, cudaStream_t st) {
    switch (C) {
        case 1: return launch_nm<N, 1>(a, nm, n_cta, st);
        case 2: return launch_nm<N, 2>(a, nm, n_cta, st);
        case 3: return launch_nm<N, 3>(a, nm, n_cta, st);
        case 4: return launch_nm<N, 4>(a, nm, n_cta, st);
        default: break;
    }
    if constexpr (N <= 512) {
        switch (C) {
            case 5: return launch_nm<N, 5>(a, nm, n_cta, st);
            case 6: return launch_nm<N, 6>(a, nm, n_cta, st);
            case 7: return launch_nm<N, 7>(a, nm, n_cta, st);
            case 8: return launch_nm<N, 8>(a, nm, n_cta, st);
            default: break;
        }
    }
    return cudaErrorInvalidValue;
}

cudaError_t launch_stft_scm(const StftArgs& a, int n_fft, int C, int n_cta, int n_mask, cudaStream_t st) {
    if (!stft_scm_supported(n_fft, C, n_mask)) return cudaErrorInvalidValue;
    switch (n_fft) {
        case 256: return launch_c<256>(a, C, n_mask, n_cta, st);
        case 512: return launch_c<512>(a, C, n_mask, n_cta, st);
        case 1024: return launch_c<1024>(a, C, n_mask, n_cta, st);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_stft_filter_dual(const StftFilterArgs& a, int n_fft, int C, int n_cta, cudaStream_t st) {
    if (!stft_scm_supported(n_fft, C, 2)) return cudaErrorInvalidValue;   // the coverage of the two-mask pass
#define DISCO_SFD(NN, CC)                                                                                  \
    if (n_fft == NN && C == CC)                                                                            \
        return a.out_ft ? launch_one<NN, CC, 0, OUT_FILTER_FT>(a, n_cta, st) : launch_one<NN, CC, 0, OUT_FILTER>(a, n_cta, st);
    DISCO_SFD(256, 1) DISCO_SFD(256, 2) DISCO_SFD(256, 3) DISCO_SFD(256, 4)
    DISCO_SFD(512, 1) DISCO_SFD(512, 2) DISCO_SFD(512, 3) DISCO_SFD(512, 4)
#undef DISCO_SFD
    return cudaErrorInvalidValue;
}

cudaError_t launch_scm_finalize(const float* part, float2* Rss, float2* Rnn, int n_grp, int slots_per_grp,
                                int tiles_per_grp, int n_cta, int C, int F, int T, int n_set, int set, cudaStream_t st) {
    const float inv_T = 1.0f / (float)T;
#define DISCO_FIN(CC)                                                                                              \
    case CC:                                                                                                       \
        scm_finalize_kernel<CC><<<n_grp, 288, 0, st>>>(part, Rss, Rnn, n_grp, slots_per_grp, tiles_per_grp, n_cta, \
                                                       F, inv_T, n_set, set);                                      \
        break;
    switch (C) {
        DISCO_FIN(1)
        DISCO_FIN(2)
        DISCO_FIN(3)
        DISCO_FIN(4)
        DISCO_FIN(5)
        DISCO_FIN(6)
        DISCO_FIN(7)
        DISCO_FIN(8)
        default: return cudaErrorInvalidValue;
    }
#undef DISCO_FIN
    return cudaGetLastError();
}

}  // namespace disco

#ifdef DISCO_ROLE_CLOCKS
// Measurement build only: the layout of the role-clock buffer, [max_ctas][32 warps][slots] unsigned 64-bit values.
extern "C" __attribute__((visibility("default"))) void disco_role_clocks_layout(int* max_ctas, int* slots) {
    *max_ctas = disco::RC_MAX_CTAS;
    *slots = disco::RC_SLOTS;
}
// Measurement build only: copy the role clocks of the last stft_scm_kernel launch to host memory `dst` (at most
// `bytes`) and, with reset != 0, zero them.  Returns the number of bytes copied, or -1 on a CUDA error.
extern "C" __attribute__((visibility("default"))) long long disco_role_clocks(void* dst, size_t bytes, int reset) {
    const size_t n = sizeof(disco::g_role_clocks) < bytes ? sizeof(disco::g_role_clocks) : bytes;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    if (n && cudaMemcpyFromSymbol(dst, disco::g_role_clocks, n) != cudaSuccess) return -1;
    if (reset) {
        void* a = nullptr;
        if (cudaGetSymbolAddress(&a, disco::g_role_clocks) != cudaSuccess ||
            cudaMemset(a, 0, sizeof(disco::g_role_clocks)) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess)
            return -1;
    }
    return (long long)n;
}
#endif
