// Per-bin multichannel-Wiener-filter solve: replaces intern_filter
// (reference se_utils/internal_formulas.py:31-81) for a whole batch of bins in one launch.
//
//   'gevd'   (:56-73)  rank-r GEVD-MWF.  Closed form of Q D (D + mu I)^-1 Q^-1 [:, 0]:
//            with (lambda_i, q_i) the generalised eigenpairs of (Rss, Rnn), q_i^H Rnn q_i = 1,
//            lambda clamped to [eps, 1e6] and sorted descending,
//                w  = sum_{i<r} q_i * lambda_i / (lambda_i + mu) * conj((Rnn q_i)[0])
//                t1 = q_0 * conj((Rnn q_0)[0])
//            computed as: Cholesky Rnn = L L^H, A = L^-1 Rss L^-H, cyclic complex Jacobi on A,
//            q = L^-H v.  (scipy.linalg.eig / cggev in the reference; same pairs for a
//            Hermitian-definite pencil.)
//   'r1-mwf' (:45-54)  w = l u conj(v_0) / (mu + l v^H u), (l, v) top eigenpair of Rss, u = Rnn^-1 v
//   'mwf'    (:74-76)  w = (Rnn + Rss)^-1 Rss e_0
//
// Float64 throughout (the SCMs arrive as complex64): the flop count is negligible next to the
// streaming kernels and double precision keeps the result far inside the 1e-5 parity budget even
// for ill-conditioned bins.  The work is latency-bound, so it is organised for short dependency
// chains: a GROUP of G = 2/4/8/16 lanes (>= D) owns one matrix, 32/G matrices share a warp, the
// matrices live in shared memory (no local-memory traffic), and every O(D) loop of the textbook
// algorithms (column / row updates of a Jacobi rotation, the columns of a triangular solve, ...)
// is spread over the group's lanes.  Groups synchronise with __syncwarp(group mask) only.
// Degenerate bins (DESIGN.md section 2; oracle/solve_f64.py states the policy executably): both matrices are
// scaled by one exact power of two (common.cuh solve_scale), a Cholesky pivot below 1e-13 * trace/D is floored
// there with the column below it set to zero, so the output stays finite at any scale where LAPACK would return
// inf/NaN eigenvalues.
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace disco {

struct cd {
    double x, y;
};
DISCO_DEV cd mk(double x, double y) { return cd{x, y}; }
DISCO_DEV cd operator+(cd a, cd b) { return cd{a.x + b.x, a.y + b.y}; }
DISCO_DEV cd operator-(cd a, cd b) { return cd{a.x - b.x, a.y - b.y}; }
DISCO_DEV cd operator*(cd a, cd b) { return cd{a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x}; }
DISCO_DEV cd operator*(double s, cd a) { return cd{s * a.x, s * a.y}; }
DISCO_DEV cd conj(cd a) { return cd{a.x, -a.y}; }
DISCO_DEV double norm2(cd a) { return a.x * a.x + a.y * a.y; }
// 1 / z without forming |z|^2 when that would overflow or underflow (z = mu + l v^H u reaches ~1e300 when
// Rnn == 0 puts u = Rnn^-1 v at 1e300 v); the plain form otherwise, so ordinary bins keep their bits.
DISCO_DEV cd crecip(cd z) {
    const double n2 = norm2(z);
    if (n2 > 1e-290 && n2 < 1e290) {
        const double dn = 1.0 / n2;
        return cd{z.x * dn, -z.y * dn};
    }
    const double s = 1.0 / fmax(fabs(z.x), fabs(z.y));
    const double a = s * z.x, b = s * z.y, dn = s / (a * a + b * b);
    return cd{a * dn, -b * dn};
}

constexpr double kEps = 2.220446049250313e-16;  // sys.float_info.epsilon (internal_formulas.py:6)
constexpr double kEta = 1e6;                    // internal_formulas.py:7

template <int D>
struct SolveGeom {
    static constexpr int G = D <= 2 ? 2 : (D <= 4 ? 4 : (D <= 8 ? 8 : 16));  // lanes per matrix
    static constexpr int MPW = 32 / G;                                       // matrices per warp
    static constexpr int P = (D % 2 == 0) ? D + 1 : D;   // odd row pitch (x16 B): conflict-free columns
    static constexpr int MAT = D * P;                     // cd elements per matrix
    static constexpr int WARPS = D <= 8 ? 4 : 2;
    static constexpr int THREADS = 32 * WARPS;
    static constexpr int MPB = MPW * WARPS;               // matrices per block
    static constexpr int NROT = (D + 1) / 2;              // rotations per Jacobi round
    static constexpr size_t SMEM = (size_t)MPB * (3 * MAT * sizeof(cd) + NROT * 48);
    // Where shared memory alone caps residency so low that >= 128 registers per thread would still fit (D = 8 and
    // D >= 12: 3..7 blocks per SM), the launch bounds tell the compiler so; left to itself it picks ~80 registers
    // and spills at D = 16.  (228 KB of shared memory per SM, 1 KB reserved per block.)
    static constexpr int SMEM_BLOCKS = (int)(233472 / (SMEM + 1024));
    static constexpr int MINB = 65536 / (THREADS * SMEM_BLOCKS) >= 128 ? SMEM_BLOCKS : 0;   // 0: no bound
};

// group-wide sum over the G lanes of a group (xor butterfly: fixed order, every lane gets the total)
template <int G>
DISCO_DEV double gsum(double v, unsigned gm) {
#pragma unroll
    for (int off = G / 2; off >= 1; off >>= 1) v += __shfl_xor_sync(gm, v, off, G);
    return v;
}
template <int G>
DISCO_DEV cd gsum(cd v, unsigned gm) {
    v.x = gsum<G>(v.x, gm);
    v.y = gsum<G>(v.y, gm);
    return v;
}

// In-place lower Cholesky of the Hermitian matrix M (lower triangle used) in shared memory.
// Lane j computes pivot j, lanes i > j their entry of column j.  A running pivot below `floor_` marks a null
// direction of M (Rnn == 0, a dead or duplicated microphone, a bin with a single noise frame): the pivot is
// floored and the column below it set to zero.  Dividing that column by the floored pivot instead would
// amplify the rounding noise of a numerically singular, slightly indefinite M (float32 statistics) by
// 1/sqrt(floor) per column, up to inf at D = 16.
template <int D>
DISCO_DEV void g_cholesky(cd* M, int l, unsigned gm, double floor_) {
    constexpr int P = SolveGeom<D>::P, G = SolveGeom<D>::G;
    for (int j = 0; j < D; ++j) {
        double inv = 0.0;
        if (l == j) {
            double d = M[j * P + j].x;
            for (int k = 0; k < j; ++k) d -= norm2(M[j * P + k]);
            const bool null_dir = !(d >= floor_);
            d = fmax(d, floor_);
            inv = rsqrt(d);
            M[j * P + j] = mk(d * inv, 0.0);
            if (null_dir) inv = 0.0;
        }
        inv = __shfl_sync(gm, inv, j, G);
        if (l > j && l < D) {
            cd s = M[l * P + j];
            for (int k = 0; k < j; ++k) s = s - M[l * P + k] * conj(M[j * P + k]);
            M[l * P + j] = inv * s;
        }
        __syncwarp(gm);
    }
}

// One Jacobi rotation (c, st) for the pivot pair (p, q); p < 0 marks "no rotation".
struct Rot {
    int p, q;
    double c;
    cd st;
};

// Parallel-order Jacobi of the Hermitian matrix A (destroyed) in shared memory; V <- eigenvectors
// (columns).  Round-robin tournament: every sweep is N-1 rounds (N = D rounded up to even) of N/2
// rotations on DISJOINT index pairs, so the N/2 expensive parameter computations of a round run
// on N/2 different lanes at once (three float64 special functions each: rsqrt, sqrt+div, rsqrt),
// then lane k applies all of them to row k of A and V (A <- A G, V <- V G), then to column k
// (A <- G^H A).  The latency of a sweep is that of N-1 parameter chains instead of D(D-1)/2.
template <int D>
DISCO_DEV void g_jacobi(cd* A, cd* V, Rot* rot, int l, unsigned gm) {
    constexpr int P = SolveGeom<D>::P, G = SolveGeom<D>::G;
    constexpr int N = D + (D & 1), NP = N / 2;
    const bool act = l < D;
    double mine = 0.0;
    if (act) {
        for (int j = 0; j < D; ++j) {
            V[l * P + j] = mk(j == l ? 1.0 : 0.0, 0.0);
            mine += norm2(A[l * P + j]);
        }
    }
    const double tot = gsum<G>(mine, gm);
    __syncwarp(gm);
    // Converged when the off-diagonal energy is below 1e-26 of the total AND every pair is small next to its own
    // diagonal: |a_pq|^2 <= 1e-26 |a_pp a_qq| + 1e-32 ||A||_F^2.  The first rule alone leaves entries of 1e-13 ||A||,
    // an absolute error of every eigenpair; where an ill-conditioned Rnn puts ||A|| near 1e9, the small eigenpairs that
    // 'full' and rank > 1 sum were off by 1e-4.  The pair rule gives them relative accuracy; its 1e-32 floor (1e-16
    // ||A||, the float64 rounding of A) ends the sweeps on the rounding noise of a singular A.  Entries below 1e-300,
    // which no rotation touches, never hold the sweeps.  tot = inf (Rnn == 0 puts A near 1e300 Rss, so norm2
    // overflows) stops before the first sweep, as it always did: both rules hold with inf on the right.
    for (int sweep = 0; sweep < 40; ++sweep) {
        double offm = 0.0;
        bool loose = false;
        if (act)
            for (int j = l + 1; j < D; ++j) {
                const double n2 = norm2(A[l * P + j]);
                offm += n2;
                loose |= n2 >= 1e-300 && n2 > 1e-26 * fabs(A[l * P + l].x) * fabs(A[j * P + j].x) + 1e-32 * tot;
            }
        const double off = gsum<G>(offm, gm);
        if (off <= 1e-26 * tot && !__any_sync(gm, loose)) break;   // group-uniform
        for (int r = 0; r < N - 1; ++r) {
            if (l < NP) {                        // lane l owns pair l of this round (circle method)
                int a0, b0;
                if (l == 0) {
                    a0 = N - 1;
                    b0 = r;
                } else {
                    a0 = (r + l) % (N - 1);
                    b0 = (r - l + (N - 1)) % (N - 1);
                }
                const int p = a0 < b0 ? a0 : b0, q = a0 < b0 ? b0 : a0;
                Rot ro;
                ro.p = -1;
                ro.q = 0;
                ro.c = 1.0;
                ro.st = mk(0.0, 0.0);
                if (q < D) {                     // q >= D: the dummy player of an odd D
                    const cd b = A[p * P + q];
                    const double n2 = norm2(b);
                    if (n2 >= 1e-300 && n2 <= 1.7976931348623157e308) {   // inf: ab = n2 rsqrt(n2) is inf * 0
                        const double inv_ab = rsqrt(n2), ab = n2 * inv_ab;
                        const cd ph = inv_ab * b;
                        const double d = 0.5 * (A[q * P + q].x - A[p * P + p].x);
                        const double t = copysign(ab, d) / (fabs(d) + sqrt(d * d + n2));
                        const double c = rsqrt(1.0 + t * t);
                        ro.p = p;
                        ro.q = q;
                        ro.c = c;
                        ro.st = (t * c) * ph;
                    }
                }
                rot[l] = ro;
            }
            __syncwarp(gm);
            if (act) {                          // A <- A G, V <- V G : row l, all pairs of the round
#pragma unroll
                for (int j = 0; j < NP; ++j) {
                    const Rot ro = rot[j];
                    if (ro.p < 0) continue;
                    const cd st = ro.st, stc = conj(ro.st);
                    const double c = ro.c;
                    const cd akp = A[l * P + ro.p], akq = A[l * P + ro.q];
                    A[l * P + ro.p] = c * akp - stc * akq;
                    A[l * P + ro.q] = st * akp + c * akq;
                    const cd vkp = V[l * P + ro.p], vkq = V[l * P + ro.q];
                    V[l * P + ro.p] = c * vkp - stc * vkq;
                    V[l * P + ro.q] = st * vkp + c * vkq;
                }
            }
            __syncwarp(gm);
            if (act) {                          // A <- G^H A : column l of the rows of every pair
#pragma unroll
                for (int j = 0; j < NP; ++j) {
                    const Rot ro = rot[j];
                    if (ro.p < 0) continue;
                    const cd st = ro.st, stc = conj(ro.st);
                    const double c = ro.c;
                    const cd apk = A[ro.p * P + l], aqk = A[ro.q * P + l];
                    cd np_ = c * apk - st * aqk, nq_ = stc * apk + c * aqk;
                    if (l == ro.q) {
                        np_ = mk(0.0, 0.0);     // the annihilated element and its mirror
                        nq_.y = 0.0;
                    }
                    if (l == ro.p) {
                        nq_ = mk(0.0, 0.0);
                        np_.y = 0.0;
                    }
                    A[ro.p * P + l] = np_;
                    A[ro.q * P + l] = nq_;
                }
            }
            __syncwarp(gm);
        }
    }
    __syncwarp(gm);
}

// Eigenpair of the LARGEST eigenvalue of the Hermitian matrix A (shared memory, preserved) by repeated squaring:
// B_0 = A / tr A, B_{k+1} = B_k^2 / tr(B_k^2) converges to v v^H with the eigenvalue ratio raised to the power
// 2^k, i.e. 10 squarings resolve a 3 % gap to 1e-14 and 24 squarings a 1e-5 gap -- a dozen small matrix products
// instead of ~50 Jacobi rounds with their float64 special functions.  Rank-1 is detected by ||B||_F^2 = 1
// (tr B = 1); at most 40 squarings, after which B spans the eigenvectors of (nearly) tied eigenvalues and any of
// its columns is a valid answer.  Lane l owns row l.  Returns this lane's component of the unit eigenvector (in
// *v_out) and the eigenvalue v^H A v.
// Squaring finds the eigenvalue of largest MAGNITUDE.  For a PSD matrix (every bin of an SCM pair) that is the
// largest one.  An indefinite A (user input such as Rss = Ryy - Rnn) whose most negative eigenvalue dominates, or
// which has eigenvalues +-rho, ends with a v that is not an eigenvector of a positive eigenvalue:
// ||A v||^2 != (v^H A v)^2 or v^H A v <= 0.  Then *ok is false and the caller takes the Jacobi path, which picks
// the largest signed eigenvalue.  A PSD matrix with a positive eigenvalue always passes.  tr A <= 1e-300 (the zero
// matrix, or an indefinite one with zero or negative trace) also goes to the Jacobi path.
// Used for the rank-1 GEVD-MWF (the only form Tango calls, tango.py:367, :443); rank > 1 keeps Jacobi.
template <int D>
DISCO_DEV double g_top_eigpair(const cd* A, cd* B, int l, unsigned gm, cd* v_out, bool* ok) {
    constexpr int P = SolveGeom<D>::P, G = SolveGeom<D>::G;
    const bool act = l < D;
    const double tr = gsum<G>(act ? A[l * P + l].x : 0.0, gm);
    *ok = false;
    if (!(tr > 1e-300)) return 0.0;             // group-uniform
    if (act) {
        const double it = 1.0 / tr;
        for (int j = 0; j < D; ++j) B[l * P + j] = it * A[l * P + j];
    }
    __syncwarp(gm);
    // B is Hermitian, so is B^2: only the entries i <= j are computed, each stored with its conjugate mirror.  Lane l
    // owns the H = D/2 + 1 entries (l, (l + s) mod D) of its row (every unordered pair has an owner; for even D the
    // pairs at distance D/2 have two owners that compute and store the same numbers).
    constexpr int H = D / 2 + 1;
    int col[H];
#pragma unroll
    for (int s = 0; s < H; ++s) col[s] = (l + s) % D;
    for (int iter = 0; iter < 40; ++iter) {
        cd c[H];
        double fro = 0.0, dg = 0.0;
        if (act) {
#pragma unroll
            for (int s = 0; s < H; ++s) c[s] = mk(0.0, 0.0);
            for (int k = 0; k < D; ++k) {
                const cd blk = B[l * P + k];
#pragma unroll
                for (int s = 0; s < H; ++s) c[s] = c[s] + blk * B[k * P + col[s]];
            }
            dg = c[0].x;
            fro = c[0].x * c[0].x;                  // the diagonal of a Hermitian square is real
#pragma unroll
            for (int s = 1; s < H; ++s) {
                // off-diagonal entries count twice (mirror); for even D the distance-D/2 pairs are owned twice
                const double wgt = (D % 2 == 0 && s == D / 2) ? 1.0 : 2.0;
                fro += wgt * norm2(c[s]);
            }
        }
        const double trc = gsum<G>(dg, gm);      // tr(B^2) = ||B||_F^2 of the previous iterate (<= 1)
        const double fr2 = gsum<G>(fro, gm);     // ||B^2||_F^2
        __syncwarp(gm);                          // everyone has finished reading B
        if (act) {
            const double it = 1.0 / trc;
            B[l * P + l] = mk(it * c[0].x, 0.0);
#pragma unroll
            for (int s = 1; s < H; ++s) {
                const cd v = it * c[s];
                B[l * P + col[s]] = v;
                B[col[s] * P + l] = conj(v);
            }
        }
        __syncwarp(gm);
        if (1.0 - fr2 / (trc * trc) <= 1e-14) break;   // new iterate is rank one (group-uniform)
    }
    // B ~ v v^H: take the column with the largest diagonal, normalise
    int jm = 0;
    double dmax = B[0].x;
    for (int j = 1; j < D; ++j)
        if (B[j * P + j].x > dmax) {
            dmax = B[j * P + j].x;
            jm = j;
        }
    cd v = act ? B[l * P + jm] : mk(0.0, 0.0);
    const double nv = gsum<G>(norm2(v), gm);
    v = rsqrt(nv) * v;
    __syncwarp(gm);
    if (act) B[l] = v;                           // row 0 of B as a scratch vector (B is dead now)
    __syncwarp(gm);
    cd av = mk(0.0, 0.0);
    if (act)
        for (int j = 0; j < D; ++j) av = av + A[l * P + j] * B[j];
    const cd lam = gsum<G>(conj(v) * av, gm);
    const double av2 = gsum<G>(norm2(av), gm);
    *ok = lam.x > 0.0 && lam.x * lam.x >= (1.0 - 1e-8) * av2;   // group-uniform
    *v_out = v;
    return lam.x;
}

// Lane l builds row l of the Hermitian-symmetrised matrix from a complex64 [D][D] array; returns the largest
// |Re| or |Im| of that row (0 for idle lanes).
template <int D>
DISCO_DEV double g_load_herm(const float2* __restrict__ R, cd* M, int l) {
    constexpr int P = SolveGeom<D>::P;
    double m = 0.0;
    if (l < D)
        for (int j = 0; j < D; ++j) {
            const float2 a = R[l * D + j], b = R[j * D + l];
            const cd v = mk(0.5 * ((double)a.x + (double)b.x), 0.5 * ((double)a.y - (double)b.y));
            M[l * P + j] = v;
            m = fmax(m, fmax(fabs(v.x), fabs(v.y)));
        }
    return m;
}

template <int D>
__global__ void __launch_bounds__(SolveGeom<D>::THREADS, SolveGeom<D>::MINB) mwf_solve_kernel(SolveArgs a) {
    using SG = SolveGeom<D>;
    constexpr int P = SG::P, G = SG::G;
    extern __shared__ __align__(16) unsigned char solve_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp_in_warp = lane / G, l = lane % G;
    const unsigned gm = (G == 32 ? 0xffffffffu : ((1u << G) - 1u)) << (grp_in_warp * G);
    const int slot = warp * SG::MPW + grp_in_warp;
    int idx = blockIdx.x * SG::MPB + slot;
    const bool live = idx < a.n_mat;       // group-uniform; dead groups mirror the last matrix (no stores)
    if (!live) idx = a.n_mat - 1;
    Rot* rot = reinterpret_cast<Rot*>(solve_smem + (size_t)SG::MPB * 3 * SG::MAT * sizeof(cd)) + (size_t)slot * SG::NROT;
    cd* S = reinterpret_cast<cd*>(solve_smem) + (size_t)slot * 3 * SG::MAT;   // Rss, then A
    cd* Lm = S + SG::MAT;                                                      // Rnn, then its Cholesky factor
    cd* V = Lm + SG::MAT;                                                      // eigenvectors
    const bool act = l < D;

    double m = g_load_herm<D>(a.Rss + (size_t)idx * D * D, S, l);
    m = fmax(m, g_load_herm<D>(a.Rnn + (size_t)idx * D * D, Lm, l));
    {   // one exact power-of-two scale for both matrices (common.cuh solve_scale)
        double t = act ? fabs(S[l * P + l].x) + fabs(Lm[l * P + l].x) : 0.0;
#pragma unroll
        for (int off = G / 2; off >= 1; off >>= 1) {   // one butterfly for the sum and the maximum
            t += __shfl_xor_sync(gm, t, off, G);
            m = fmax(m, __shfl_xor_sync(gm, m, off, G));
        }
        const double sc = solve_scale(fmax(t, m));
        if (act)
            for (int j = 0; j < D; ++j) {
                S[l * P + j] = sc * S[l * P + j];
                Lm[l * P + j] = sc * Lm[l * P + j];
            }
    }
    __syncwarp(gm);
    // first row of Rnn (for conj((Rnn q)[0])) and the traces, before the matrices are overwritten
    const cd n0 = act ? Lm[0 * P + l] : mk(0.0, 0.0);
    const double trn = gsum<G>(act ? Lm[l * P + l].x : 0.0, gm);
    const double trs = gsum<G>(act ? S[l * P + l].x : 0.0, gm);
    cd w = mk(0.0, 0.0), t1 = mk((l == 0) ? 1.0 : 0.0, 0.0);   // t1 = e_0 (internal_formulas.py:43)

    if (a.type == 0) {  // ------------------------------------------------------------ gevd
        g_cholesky<D>(Lm, l, gm, 1e-13 * trn / D + 1e-300);
        if (act) {      // M = L^-1 Rss : lane = column
            for (int i = 0; i < D; ++i) {
                cd s = S[i * P + l];
                for (int k = 0; k < i; ++k) s = s - Lm[i * P + k] * S[k * P + l];
                S[i * P + l] = (1.0 / Lm[i * P + i].x) * s;
            }
        }
        __syncwarp(gm);
        if (act) {      // A = M L^-H : lane = row
            for (int j = 0; j < D; ++j) {
                cd s = S[l * P + j];
                for (int k = 0; k < j; ++k) s = s - S[l * P + k] * conj(Lm[j * P + k]);
                S[l * P + j] = (1.0 / Lm[j * P + j].x) * s;
            }
        }
        __syncwarp(gm);
        if (act) {      // exact Hermitian symmetry: lane l owns the pairs (l, j < l)
            for (int j = 0; j < l; ++j) {
                const cd v = 0.5 * (S[l * P + j] + conj(S[j * P + l]));
                S[l * P + j] = v;
                S[j * P + l] = conj(v);
            }
            S[l * P + l].y = 0.0;
        }
        __syncwarp(gm);
        bool top_ok = false;   // rank 1 by squaring; Jacobi for rank > 1 and for the bins squaring cannot settle
        if (a.rank == 1) {
            // rank-1 GEVD-MWF: only the principal pair is needed
            cd v;
            const double lam1 = g_top_eigpair<D>(S, V, l, gm, &v, &top_ok);
            if (top_ok) {
                // q = L^-H v : column-oriented back substitution, one broadcast per step
                cd q = v;
                for (int i = D - 1; i >= 0; --i) {
                    cd qi = mk(0.0, 0.0);
                    if (l == i) {
                        q = (1.0 / Lm[i * P + i].x) * q;
                        qi = q;
                    }
                    qi.x = __shfl_sync(gm, qi.x, i, G);
                    qi.y = __shfl_sync(gm, qi.y, i, G);
                    if (l < i) q = q - conj(Lm[i * P + l]) * qi;
                }
                if (!act) q = mk(0.0, 0.0);
                const double lam = fmin(fmax(lam1, kEps), kEta);
                const cd c0 = gsum<G>(n0 * q, gm);            // (Rnn q)[0] = sum_j Rnn[0][j] q[j]
                const cd qc = q * conj(c0);
                w = (lam / (lam + a.mu)) * qc;
                t1 = qc;
            }
        }
        if (!top_ok) {
            __syncwarp(gm);                      // the squaring's scratch in V is dead
            g_jacobi<D>(S, V, rot, l, gm);
            if (act) {      // Q = L^-H V : lane = eigenvector (column), back substitution
                for (int i = D - 1; i >= 0; --i) {
                    cd s = V[i * P + l];
                    for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k * P + i]) * V[k * P + l];
                    V[i * P + l] = (1.0 / Lm[i * P + i].x) * s;
                }
            }
            __syncwarp(gm);
            const int rank = (a.rank <= 0 || a.rank > D) ? D : a.rank;
            unsigned used = 0;
            for (int r = 0; r < rank; ++r) {   // r-th largest eigenvalue (every lane makes the same choice)
                int best = -1;
                double lbest = 0.0;
                for (int i = 0; i < D; ++i) {
                    const double li = S[i * P + i].x;
                    if (!((used >> i) & 1u) && (best < 0 || li > lbest)) {
                        best = i;
                        lbest = li;
                    }
                }
                used |= 1u << best;
                const double lam = fmin(fmax(lbest, kEps), kEta);
                const cd qi = act ? V[l * P + best] : mk(0.0, 0.0);
                const cd c0 = gsum<G>(n0 * qi, gm);           // (Rnn q)[0] = sum_j Rnn[0][j] q[j]
                const cd qc = qi * conj(c0);
                w = w + (lam / (lam + a.mu)) * qc;
                if (r == 0) t1 = qc;
            }
        }
    } else if (a.type == 1) {  // -------------------------------------------------- r1-mwf
        g_jacobi<D>(S, V, rot, l, gm);            // eigen-decomposition of Rss itself
        int best = 0;
        for (int i = 1; i < D; ++i)
            if (S[i * P + i].x > S[best * P + best].x) best = i;
        const double lmax = fabs(S[best * P + best].x);
        g_cholesky<D>(Lm, l, gm, 1e-13 * trn / D + 1e-300);
        __syncwarp(gm);
        cd* u = S;                            // A is no longer needed: its first row is scratch for u = Rnn^-1 v
        if (l == 0) {
            for (int i = 0; i < D; ++i) {
                cd s = V[i * P + best];
                for (int k = 0; k < i; ++k) s = s - Lm[i * P + k] * u[k];
                u[i] = (1.0 / Lm[i * P + i].x) * s;
            }
            for (int i = D - 1; i >= 0; --i) {
                cd s = u[i];
                for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k * P + i]) * u[k];
                u[i] = (1.0 / Lm[i * P + i].x) * s;
            }
        }
        __syncwarp(gm);
        const cd vl = act ? V[l * P + best] : mk(0.0, 0.0);
        const cd ul = act ? u[l] : mk(0.0, 0.0);
        const cd vhu = gsum<G>(conj(vl) * ul, gm);
        const cd den = mk(a.mu + lmax * vhu.x, lmax * vhu.y);   // real for Hermitian Rnn up to rounding
        const cd inv = crecip(den);
        w = ul * ((lmax * conj(V[0 * P + best])) * inv);
    } else {  // ------------------------------------------------------------------------ mwf
        if (act)
            for (int j = 0; j < D; ++j) Lm[l * P + j] = Lm[l * P + j] + S[l * P + j];
        __syncwarp(gm);
        g_cholesky<D>(Lm, l, gm, 1e-13 * (trn + trs) / D + 1e-300);
        cd* u = V;                            // scratch: first row of V
        if (l == 0) {
            for (int i = 0; i < D; ++i) {     // L y = Rss[:, 0]
                cd s = S[i * P + 0];
                for (int k = 0; k < i; ++k) s = s - Lm[i * P + k] * u[k];
                u[i] = (1.0 / Lm[i * P + i].x) * s;
            }
            for (int i = D - 1; i >= 0; --i) {
                cd s = u[i];
                for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k * P + i]) * u[k];
                u[i] = (1.0 / Lm[i * P + i].x) * s;
            }
        }
        __syncwarp(gm);
        if (act) w = u[l];
    }
    if (live && act) {
        a.W[(size_t)idx * D + l] = make_float2((float)w.x, (float)w.y);
        if (a.T1) a.T1[(size_t)idx * D + l] = make_float2((float)t1.x, (float)t1.y);
    }
}

template <int D>
static cudaError_t launch_d(const SolveArgs& a, cudaStream_t st) {
    using SG = SolveGeom<D>;
    const int blocks = (a.n_mat + SG::MPB - 1) / SG::MPB;
    auto kern = mwf_solve_kernel<D>;
    if (SG::SMEM > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SG::SMEM);
        if (e != cudaSuccess) return e;
    }
    kern<<<blocks, SG::THREADS, SG::SMEM, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_mwf_solve_small(const SolveArgs& a, cudaStream_t st);   // solve_small.cu (D <= 4, registers)

cudaError_t launch_mwf_solve(const SolveArgs& a, cudaStream_t st) {
    if (a.n_mat <= 0) return cudaSuccess;
    if (a.D <= 4) return launch_mwf_solve_small(a, st);
    if (a.part != nullptr) return cudaErrorInvalidValue;   // only the D <= 4 solver reads the partial sums
    switch (a.D) {
        case 5: return launch_d<5>(a, st);
        case 6: return launch_d<6>(a, st);
        case 7: return launch_d<7>(a, st);
        case 8: return launch_d<8>(a, st);
        case 9: return launch_d<9>(a, st);
        case 10: return launch_d<10>(a, st);
        case 11: return launch_d<11>(a, st);
        case 12: return launch_d<12>(a, st);
        case 13: return launch_d<13>(a, st);
        case 14: return launch_d<14>(a, st);
        case 15: return launch_d<15>(a, st);
        case 16: return launch_d<16>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
