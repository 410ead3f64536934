// Shared pieces of the wide-channel SCM kernels (scm_wide.cu, mid_multi.cu): everything a CTA that owns
// (group, 32-bin block) needs to stream tiles of spectra through shared memory and accumulate the
// Hermitian pairs of  sum_t m^2 x x^H  and  sum_t (1-m)^2 x x^H  in registers.  The pair index
// (tri_i / tri_j) also serves scm.cu, and the matrix store (store_pairs) online.cu.
//
//  * cp.async (LDGSTS) 8-byte copies fill a ring of shared-memory stages; out-of-range frames and bins
//    are zero-filled by the copy itself (src-size 0), so the accumulation loops carry no predicates
//    and every operand address is `base + immediate`.
//  * F = n_fft/2 + 1 is always 1 (mod 32): the last 32-bin block holds only the Nyquist bin.  In that
//    block the lanes are mapped to FRAMES instead of bins (32 frames of bin F-1 per tile slot), and a
//    butterfly sum over the lanes closes the accumulation -- instead of 31 idle lanes walking all T frames.
//  * the pairs (i, j), i <= j, are dealt round-robin to NPART warp-uniform partitions; diagonal pairs
//    accumulate only the real part |x_i|^2.
#pragma once
#include "common.cuh"

namespace disco {

DISCO_DEV void cp_async8(void* dst_smem, const void* src, bool valid) {
    const uint32_t n = valid ? 8u : 0u;   // src-size 0: nothing is read, 8 zero bytes are written
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(n)
                 : "memory");
}
DISCO_DEV void cp_async4(void* dst_smem, const void* src, bool valid) {
    const uint32_t n = valid ? 4u : 0u;
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(smem_u32(dst_smem)), "l"(src), "r"(n)
                 : "memory");
}
DISCO_DEV void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
DISCO_DEV void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Which (bin, frame) a lane touches in slot `ts` of tile `i` (TS slots per tile):
//   frame = (i * TS + ts) * tmul + tl,   bin = fcol
struct LaneGeom {
    int fcol, tl, tmul;
    bool ok;    // the lane owns a bin at all
    bool nyq;   // Nyquist block: lanes <-> frames
};
DISCO_DEV LaneGeom lane_geom(int blk, int lane, int F) {
    LaneGeom g;
    const int f = blk * 32 + lane;
    g.nyq = (F % 32 == 1) && (blk == F / 32);
    g.ok = g.nyq || f < F;
    g.fcol = (g.nyq || f >= F) ? F - 1 : f;
    g.tl = g.nyq ? lane : 0;
    g.tmul = g.nyq ? 32 : 1;
    return g;
}

// pair index -> (i, j), i <= j, row-major over the upper triangle (compile-time)
template <int D>
__host__ __device__ constexpr int tri_i(int p) {
    int i = 0, n = D;
    while (p >= n) {
        p -= n;
        --n;
        ++i;
    }
    return i;
}
template <int D>
__host__ __device__ constexpr int tri_j(int p) {
    int i = 0, n = D;
    while (p >= n) {
        p -= n;
        --n;
        ++i;
    }
    return i + p;
}

template <int D, int NPART>
struct PairGeom {
    static constexpr int NPAIR = D * (D + 1) / 2;
    static constexpr int NPP = (NPAIR + NPART - 1) / NPART;   // accumulator slots per partition
};

// a * conj(b) with the swapped operand precomputed: one fmul2 + one ffma2 (bit-identical to cmulc);
// a_sw = (a.y, -a.x)
DISCO_DEV float2 cmulc_packed(float2 a, float2 a_sw, float2 b) {
    const float2 t = fmul2(a_sw, make_float2(b.y, b.y));
    return ffma2(a, make_float2(b.x, b.x), t);
}

template <int D, int NPART, int PART, int Q = 0>
struct WidePairAcc {
    using G = PairGeom<D, NPART>;
    static DISCO_DEV void run(const float2 (&x)[D], const float2 (&xs)[D], float wa, float wb, float2 (&ps)[G::NPP],
                              float2 (&pn)[G::NPP]) {
        if constexpr (Q < G::NPP) {
            constexpr int pidx = Q * NPART + PART;
            if constexpr (pidx < G::NPAIR) {
                constexpr int i = tri_i<D>(pidx), j = tri_j<D>(pidx);
                if constexpr (i == j) {
                    const float p = fmaf(x[i].x, x[i].x, x[i].y * x[i].y);
                    ps[Q].x = fmaf(wa, p, ps[Q].x);
                    pn[Q].x = fmaf(wb, p, pn[Q].x);
                } else {
                    const float2 op = cmulc_packed(x[i], xs[i], x[j]);
                    ps[Q] = cfma_r(wa, op, ps[Q]);
                    pn[Q] = cfma_r(wb, op, pn[Q]);
                }
            }
            WidePairAcc<D, NPART, PART, Q + 1>::run(x, xs, wa, wb, ps, pn);
        }
    }
};

template <int D, int NPART, int PART>
DISCO_DEV void wide_point(const float2 (&x)[D], float m, bool has_mask, float2 (&ps)[PairGeom<D, NPART>::NPP],
                          float2 (&pn)[PairGeom<D, NPART>::NPP]) {
    float2 xs[D];
#pragma unroll
    for (int i = 0; i < D; ++i) xs[i] = make_float2(x[i].y, -x[i].x);   // unused ones are eliminated
    const float wa = m * m, wb = has_mask ? (1.f - m) * (1.f - m) : 0.f;
    WidePairAcc<D, NPART, PART>::run(x, xs, wa, wb, ps, pn);
}

// Nyquist block: every lane holds the partial sums of its frames -> all lanes get the total (fixed order)
template <int NPP>
DISCO_DEV void lane_butterfly(float2 (&ps)[NPP], float2 (&pn)[NPP]) {
#pragma unroll
    for (int q = 0; q < NPP; ++q) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            ps[q].x += __shfl_xor_sync(0xffffffffu, ps[q].x, o);
            ps[q].y += __shfl_xor_sync(0xffffffffu, ps[q].y, o);
            pn[q].x += __shfl_xor_sync(0xffffffffu, pn[q].x, o);
            pn[q].y += __shfl_xor_sync(0xffffffffu, pn[q].y, o);
        }
    }
}

// scale by 1/T and store one partition's pairs with their conjugate mirrors; `chan(r)` maps the
// accumulation channel index to the output channel index
template <int D, int NPART, class Map>
DISCO_DEV void store_pairs(const float2 (&ps)[PairGeom<D, NPART>::NPP], const float2 (&pn)[PairGeom<D, NPART>::NPP],
                           int part, float inv_T, float2* Rs, float2* Rn, Map chan) {
    using G = PairGeom<D, NPART>;
#pragma unroll
    for (int q = 0; q < G::NPP; ++q) {
        const int pidx = q * NPART + part;   // `part` is runtime here (tiny epilogue)
        if (pidx < G::NPAIR) {
            int i = 0, n = D, pp = pidx;
            while (pp >= n) {
                pp -= n;
                --n;
                ++i;
            }
            const int ri = chan(i), rj = chan(i + pp);
            float2 s = cscale(ps[q], inv_T), nn = cscale(pn[q], inv_T);
            if (ri == rj) s.y = 0.f, nn.y = 0.f;
            Rs[ri * D + rj] = s;
            Rn[ri * D + rj] = nn;
            if (ri != rj) {
                Rs[rj * D + ri] = cconj(s);
                Rn[rj * D + ri] = cconj(nn);
            }
        }
    }
}

}  // namespace disco
