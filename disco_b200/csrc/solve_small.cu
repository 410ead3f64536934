// Thread-per-matrix variant of the per-bin MWF solve for SMALL matrices (D <= 4): every loop is fully
// unrolled so the 4x4 complex float64 matrices live in registers (no shared or local memory traffic);
// with C <= 4 microphones per node this is the step-1 solve of every Tango configuration.  Same
// mathematics and degenerate-bin policy as solve.cu (see there for the formulas and references).
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"

namespace disco {
namespace small {

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
DISCO_DEV double cmaxabs(cd a, cd b) { return fmax(fmax(fabs(a.x), fabs(a.y)), fmax(fabs(b.x), fabs(b.y))); }
// 1 / z without forming |z|^2 when that would overflow or underflow (see solve.cu crecip)
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

// Row pitch of the per-thread matrices.  D = 16 is padded to 17: with a power-of-two pitch nvcc 12.9
// miscompiles the 'gevd' branch (the same source built for the host is correct; see DESIGN.md).
template <int D>
struct Ld {
    static constexpr int v = (D == 16) ? 17 : D;
};

// In-place lower Cholesky of the Hermitian matrix M (uses the lower triangle); returns L in M's
// lower triangle with real positive diagonal.  Pivots are floored at `floor_`, and the column below a floored
// pivot is set to zero (solve.cu g_cholesky).
template <int D>
DISCO_DEV void cholesky(cd (&M)[D][Ld<D>::v], double floor_) {
    constexpr int U = (D <= 4) ? D : 1;   // small matrices: fully unrolled, register resident
#pragma unroll U
    for (int j = 0; j < D; ++j) {
        double d = M[j][j].x;
        for (int k = 0; k < j; ++k) d -= norm2(M[j][k]);
        const bool null_dir = !(d >= floor_);
        d = fmax(d, floor_);
        const double inv = rsqrt(d), l = d * inv, sc = null_dir ? 0.0 : inv;
        M[j][j] = mk(l, 0.0);
        for (int i = j + 1; i < D; ++i) {
            cd s = M[i][j];
            for (int k = 0; k < j; ++k) s = s - M[i][k] * conj(M[j][k]);
            M[i][j] = sc * s;
        }
    }
}

// One Jacobi rotation annihilating A[p][q] (and A[q][p]); A <- G^H A G, V <- V G.
// Three expensive float64 operations per rotation (rsqrt, sqrt + div, rsqrt) instead of six.
template <int D>
DISCO_DEV void jacobi_rotate(cd (&A)[D][Ld<D>::v], cd (&V)[D][Ld<D>::v], int p, int q) {
    const cd b = A[p][q];
    const double n2 = norm2(b);
    if (n2 < 1e-300 || n2 > 1.7976931348623157e308) return;   // inf: ab = n2 rsqrt(n2) is inf * 0
    const double inv_ab = rsqrt(n2), ab = n2 * inv_ab;
    const cd ph = inv_ab * b;
    const double d = 0.5 * (A[q][q].x - A[p][p].x);
    const double t = copysign(ab, d) / (fabs(d) + sqrt(d * d + n2));   // tan of the rotation angle
    const double c = rsqrt(1.0 + t * t), s = t * c;
    const cd st = s * ph, stc = conj(st);
#pragma unroll
    for (int k = 0; k < D; ++k) {  // A <- A G
        const cd akp = A[k][p], akq = A[k][q];
        A[k][p] = c * akp - stc * akq;
        A[k][q] = st * akp + c * akq;
    }
#pragma unroll
    for (int k = 0; k < D; ++k) {  // A <- G^H A
        const cd apk = A[p][k], aqk = A[q][k];
        A[p][k] = c * apk - st * aqk;
        A[q][k] = stc * apk + c * aqk;
    }
    A[p][q] = mk(0.0, 0.0);
    A[q][p] = mk(0.0, 0.0);
    A[p][p].y = 0.0;
    A[q][q].y = 0.0;
#pragma unroll
    for (int k = 0; k < D; ++k) {  // V <- V G
        const cd vkp = V[k][p], vkq = V[k][q];
        V[k][p] = c * vkp - stc * vkq;
        V[k][q] = st * vkp + c * vkq;
    }
}

// Cyclic Jacobi for a Hermitian matrix A (destroyed); V receives the eigenvectors (columns),
// lam the eigenvalues (unsorted).  Converged when the off-diagonal energy is below 1e-26 of the
// total (the inputs carry float32 rounding, ~1e-14 relative energy) and every pair is small next to its own diagonal,
// |a_pq|^2 <= 1e-26 |a_pp a_qq| + 1e-32 ||A||_F^2, which gives the small eigenpairs relative accuracy (solve.cu
// g_jacobi).  For D <= 4 the (p, q) loops are
// fully unrolled so that A and V live in registers; larger matrices index local memory.
template <int D>
DISCO_DEV void jacobi(cd (&A)[D][Ld<D>::v], cd (&V)[D][Ld<D>::v], double (&lam)[D]) {
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) V[i][j] = mk(i == j ? 1.0 : 0.0, 0.0);
    double tot = 0.0;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) tot += norm2(A[i][j]);
#pragma unroll 1
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0;
        bool loose = false;
#pragma unroll
        for (int p = 0; p < D; ++p)
#pragma unroll
            for (int q = p + 1; q < D; ++q) {
                const double n2 = norm2(A[p][q]);
                off += n2;
                loose |= n2 >= 1e-300 && n2 > 1e-26 * fabs(A[p][p].x) * fabs(A[q][q].x) + 1e-32 * tot;
            }
        if (off <= 1e-26 * tot && !loose) break;
        if constexpr (D <= 4) {
#pragma unroll
            for (int p = 0; p < D - 1; ++p)
#pragma unroll
                for (int q = p + 1; q < D; ++q) jacobi_rotate<D>(A, V, p, q);
        } else {
#pragma unroll 1
            for (int p = 0; p < D - 1; ++p)
#pragma unroll 1
                for (int q = p + 1; q < D; ++q) jacobi_rotate<D>(A, V, p, q);
        }
    }
#pragma unroll
    for (int i = 0; i < D; ++i) lam[i] = A[i][i].x;
}

// Eigenpair of the LARGEST eigenvalue of the Hermitian matrix A by repeated squaring (see solve.cu g_top_eigpair):
// B <- B^2 / tr(B^2) until ||B||_F^2 = 1 (rank one).  Fully unrolled: B and its square live in registers.
// v receives the unit eigenvector, the return value is v^H A v.  When v is not an eigenvector of a positive
// eigenvalue (indefinite A, see solve.cu), the squaring is repeated on A - shift I with shift = -1.5 D max |A_ij|
// below the smallest eigenvalue: that matrix is PSD with the same top eigenvector.  (The cooperative solver takes
// its Jacobi path instead; a second squaring run there costs registers and spills.)
template <int D>
DISCO_DEV double top_eigpair(const cd (&A)[D][Ld<D>::v], cd (&v)[D]) {
    double tr = 0.0, amax = 0.0;
#pragma unroll
    for (int i = 0; i < D; ++i) tr += A[i][i].x;
#pragma unroll
    for (int i = 0; i < D; ++i)
#pragma unroll
        for (int j = 0; j < D; ++j) amax = fmax(amax, fmax(fabs(A[i][j].x), fabs(A[i][j].y)));
    if (!(amax > 1e-300)) {
#pragma unroll
        for (int i = 0; i < D; ++i) v[i] = mk(i == 0 ? 1.0 : 0.0, 0.0);
        return 0.0;
    }
    double shift = 0.0, nrm = (tr >= 0.5 * amax) ? tr : amax, lam = 0.0;   // tr A >= max |A_ij| for PSD A
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {
        cd B[D][D];
        {
            const double it = 1.0 / nrm;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = 0; j < D; ++j) B[i][j] = it * A[i][j];
#pragma unroll
            for (int i = 0; i < D; ++i) B[i][i].x = it * (A[i][i].x - shift);
        }
#pragma unroll 1
        for (int iter = 0; iter < 40; ++iter) {
            cd C[D][D];
            double trc = 0.0, fr2 = 0.0;
#pragma unroll
            for (int i = 0; i < D; ++i)
#pragma unroll
                for (int j = i; j < D; ++j) {           // Hermitian: upper triangle only
                    cd c = B[i][0] * B[0][j];
#pragma unroll
                    for (int k = 1; k < D; ++k) c = c + B[i][k] * B[k][j];
                    C[i][j] = c;
                    if (i == j) {
                        trc += c.x;
                        fr2 += c.x * c.x;
                    } else {
                        fr2 += 2.0 * norm2(c);
                    }
                }
            const double it = 1.0 / trc;
#pragma unroll
            for (int i = 0; i < D; ++i) {
                B[i][i] = mk(it * C[i][i].x, 0.0);
#pragma unroll
                for (int j = i + 1; j < D; ++j) {
                    B[i][j] = it * C[i][j];
                    B[j][i] = conj(B[i][j]);
                }
            }
            if (1.0 - fr2 * it * it <= 1e-14) break;
        }
        int jm = 0;
#pragma unroll
        for (int j = 1; j < D; ++j)
            if (B[j][j].x > B[jm][jm].x) jm = j;
        double nv = 0.0;
#pragma unroll
        for (int i = 0; i < D; ++i) {
            cd c = B[i][0];
#pragma unroll
            for (int j = 1; j < D; ++j)
                if (j == jm) c = B[i][j];
            v[i] = c;
            nv += norm2(c);
        }
        const double inv = rsqrt(nv);
        double av2 = 0.0;
        lam = 0.0;
#pragma unroll
        for (int i = 0; i < D; ++i) v[i] = inv * v[i];
#pragma unroll
        for (int i = 0; i < D; ++i) {
            cd av = A[i][0] * v[0];
#pragma unroll
            for (int j = 1; j < D; ++j) av = av + A[i][j] * v[j];
            lam += (conj(v[i]) * av).x;
            av2 += norm2(av);
        }
        if (lam > 0.0 && lam * lam >= (1.0 - 1e-8) * av2) break;   // an eigenvector of a positive eigenvalue
        shift = -1.5 * D * amax;
        nrm = tr - D * shift;
    }
    return lam;
}

template <int D>
DISCO_DEV void load_herm(const float2* __restrict__ R, cd (&M)[D][Ld<D>::v]) {
    // Hermitian-symmetrise: the SCM kernels write exact conjugate mirrors, user input may not
    for (int i = 0; i < D; ++i)
        for (int j = 0; j <= i; ++j) {
            const float2 a = R[i * D + j], b = R[j * D + i];
            const cd v = mk(0.5 * ((double)a.x + (double)b.x), 0.5 * ((double)a.y - (double)b.y));
            M[i][j] = v;
            M[j][i] = conj(v);
        }
}

// Rebuild one Hermitian matrix from the fused STFT+SCM kernel's partial sums: accumulator layout
// [D diagonals][D(D-1)/2 x (re, im) upper pairs, row-major], slots summed in order, scaled by 1/T
// (same arithmetic as scm_finalize_kernel, so both routes give bit-identical matrices).
template <int D>
DISCO_DEV void load_part(const float* __restrict__ q, int n_slot, size_t slot_stride, int F, float inv_T,
                         cd (&M)[D][Ld<D>::v]) {
    float acc[D * D];
#pragma unroll
    for (int a = 0; a < D * D; ++a) acc[a] = 0.f;
    for (int sl = 0; sl < n_slot; ++sl) {
#pragma unroll
        for (int a = 0; a < D * D; ++a) acc[a] += __ldg(q + sl * slot_stride + (size_t)a * F);
    }
    int o = 0;
#pragma unroll
    for (int i = 0; i < D; ++i) {
        M[i][i] = mk((double)(acc[i] * inv_T), 0.0);
#pragma unroll
        for (int j = i + 1; j < D; ++j) {
            const cd v = mk((double)(acc[D + 2 * o] * inv_T), (double)(acc[D + 2 * o + 1] * inv_T));
            M[i][j] = v;
            M[j][i] = conj(v);
            ++o;
        }
    }
}

template <int D, int MINB, bool PART>
__global__ void __launch_bounds__(64, MINB) mwf_solve_kernel(SolveArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.n_mat) return;
    constexpr int LD = Ld<D>::v;
    cd S[D][LD], Nn[D][LD], V[D][LD];
    cd w[D], t1[D];
    for (int i = 0; i < D; ++i) t1[i] = mk(i == 0 ? 1.0 : 0.0, 0.0);   // e_0 (internal_formulas.py:43)
    if (PART) {
        const int n_set = a.n_set > 0 ? a.n_set : 1;
        const int n_grp = a.n_mat / (a.F * n_set);
        const int set = idx / (n_grp * a.F), g = (idx / a.F) % n_grp, f = idx % a.F;
        const long long total = (long long)n_grp * a.tiles_per_grp;
        const int n_slot = seg_slots(g, a.tiles_per_grp, total, a.n_cta).count();
        const size_t slot_stride = (size_t)n_set * 2 * D * D * a.F;
        const float* q = a.part + (size_t)g * a.slots_per_grp * slot_stride + (size_t)set * 2 * D * D * a.F + f;
        load_part<D>(q, n_slot, slot_stride, a.F, a.inv_T, S);
        load_part<D>(q + (size_t)D * D * a.F, n_slot, slot_stride, a.F, a.inv_T, Nn);
        if (a.Rss) {   // optionally also materialise the matrices (API output of the fused op)
            float2* Rs = const_cast<float2*>(a.Rss) + (size_t)idx * D * D;
            float2* Rn = const_cast<float2*>(a.Rnn) + (size_t)idx * D * D;
            for (int i = 0; i < D; ++i)
                for (int j = 0; j < D; ++j) {
                    Rs[i * D + j] = make_float2((float)S[i][j].x, (float)S[i][j].y);
                    Rn[i * D + j] = make_float2((float)Nn[i][j].x, (float)Nn[i][j].y);
                }
        }
    } else {
        load_herm<D>(a.Rss + (size_t)idx * D * D, S);
        load_herm<D>(a.Rnn + (size_t)idx * D * D, Nn);
    }
    {   // one exact power-of-two scale for both matrices (common.cuh solve_scale)
        double t = 0.0, m = 0.0;
        for (int i = 0; i < D; ++i) t += fabs(S[i][i].x) + fabs(Nn[i][i].x);
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) m = fmax(m, cmaxabs(S[i][j], Nn[i][j]));
        const double sc = solve_scale(fmax(t, m));
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) {
                S[i][j] = sc * S[i][j];
                Nn[i][j] = sc * Nn[i][j];
            }
    }
    double trn = 0.0, trs = 0.0;
    for (int i = 0; i < D; ++i) trn += Nn[i][i].x, trs += S[i][i].x;

    if (a.type == 0) {  // ------------------------------------------------------------ gevd
        cd Lm[D][LD];
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) Lm[i][j] = Nn[i][j];
        cholesky<D>(Lm, 1e-13 * trn / D + 1e-300);
        // M = L^-1 S  (forward substitution, column by column), stored in S
        for (int col = 0; col < D; ++col)
            for (int i = 0; i < D; ++i) {
                cd s = S[i][col];
                for (int k = 0; k < i; ++k) s = s - Lm[i][k] * S[k][col];
                S[i][col] = (1.0 / Lm[i][i].x) * s;
            }
        // A = M L^-H  <=>  A^H = L^-1 M^H ; do it row-wise: for each row r of M solve x L^H = M[r]
        for (int r = 0; r < D; ++r)
            for (int j = 0; j < D; ++j) {
                cd s = S[r][j];
                for (int k = 0; k < j; ++k) s = s - S[r][k] * conj(Lm[j][k]);
                S[r][j] = (1.0 / Lm[j][j].x) * s;
            }
        for (int i = 0; i < D; ++i)   // enforce exact Hermitian symmetry
            for (int j = 0; j < i; ++j) {
                cd v = 0.5 * (S[i][j] + conj(S[j][i]));
                S[i][j] = v;
                S[j][i] = conj(v);
            }
        if (a.rank == 1) {   // rank-1 GEVD-MWF (tango.py:367, :443): principal pair only, by repeated squaring
            cd q[D];
            const double lam1 = top_eigpair<D>(S, q);
            for (int i = D - 1; i >= 0; --i) {       // q = L^-H v
                cd sacc = q[i];
                for (int k = i + 1; k < D; ++k) sacc = sacc - conj(Lm[k][i]) * q[k];
                q[i] = (1.0 / Lm[i][i].x) * sacc;
            }
            const double l = fmin(fmax(lam1, kEps), kEta);
            cd c0 = mk(0.0, 0.0);                    // (Rnn q)[0]
            for (int j = 0; j < D; ++j) c0 = c0 + Nn[0][j] * q[j];
            const cd cc = conj(c0);
            const double g = l / (l + a.mu);
            for (int i = 0; i < D; ++i) {
                const cd qc = q[i] * cc;
                w[i] = g * qc;
                t1[i] = qc;
            }
        } else {
        double lam[D];
            jacobi<D>(S, V, lam);
            // Q = L^-H V : back substitution on each eigenvector
            for (int col = 0; col < D; ++col)
                for (int i = D - 1; i >= 0; --i) {
                    cd s = V[i][col];
                    for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k][i]) * V[k][col];
                    V[i][col] = (1.0 / Lm[i][i].x) * s;
                }
            for (int i = 0; i < D; ++i) w[i] = mk(0.0, 0.0);
            const int rank = (a.rank <= 0 || a.rank > D) ? D : a.rank;
            bool used[D];
            for (int i = 0; i < D; ++i) used[i] = false;
            for (int r = 0; r < rank; ++r) {  // r-th largest eigenvalue (selection, stable for ties)
                int best = -1;
                for (int i = 0; i < D; ++i)
                    if (!used[i] && (best < 0 || lam[i] > lam[best])) best = i;
                used[best] = true;
                const double l = fmin(fmax(lam[best], kEps), kEta);
                cd c0 = mk(0.0, 0.0);  // (Rnn q)[0]
                for (int j = 0; j < D; ++j) c0 = c0 + Nn[0][j] * V[j][best];
                const cd cc = conj(c0);
                const double g = l / (l + a.mu);
                for (int i = 0; i < D; ++i) {
                    const cd qc = V[i][best] * cc;
                    w[i] = w[i] + g * qc;
                    if (r == 0) t1[i] = qc;
                }
            }
        }
    } else if (a.type == 1) {  // -------------------------------------------------- r1-mwf
        cd Lm[D][LD];
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) Lm[i][j] = Nn[i][j];
        double lam[D];
        jacobi<D>(S, V, lam);
        int best = 0;
        for (int i = 1; i < D; ++i)
            if (lam[i] > lam[best]) best = i;
        const double l = fabs(lam[best]);
        cholesky<D>(Lm, 1e-13 * trn / D + 1e-300);
        cd u[D];
        for (int i = 0; i < D; ++i) {  // L y = v
            cd s = V[i][best];
            for (int k = 0; k < i; ++k) s = s - Lm[i][k] * u[k];
            u[i] = (1.0 / Lm[i][i].x) * s;
        }
        for (int i = D - 1; i >= 0; --i) {  // L^H u = y
            cd s = u[i];
            for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k][i]) * u[k];
            u[i] = (1.0 / Lm[i][i].x) * s;
        }
        cd vhu = mk(0.0, 0.0);
        for (int i = 0; i < D; ++i) vhu = vhu + conj(V[i][best]) * u[i];
        // w = l u conj(v0) / (mu + l v^H u); the denominator is real for Hermitian Rnn
        const cd den = mk(a.mu + l * vhu.x, l * vhu.y);
        const cd inv = crecip(den);
        const cd sc = (l * conj(V[0][best])) * inv;
        for (int i = 0; i < D; ++i) w[i] = u[i] * sc;
    } else {  // ------------------------------------------------------------------------ mwf
        cd Lm[D][LD];
        for (int i = 0; i < D; ++i)
            for (int j = 0; j < D; ++j) Lm[i][j] = Nn[i][j] + S[i][j];
        cholesky<D>(Lm, 1e-13 * (trn + trs) / D + 1e-300);
        for (int i = 0; i < D; ++i) {  // L y = Rss[:, 0]
            cd s = S[i][0];
            for (int k = 0; k < i; ++k) s = s - Lm[i][k] * w[k];
            w[i] = (1.0 / Lm[i][i].x) * s;
        }
        for (int i = D - 1; i >= 0; --i) {
            cd s = w[i];
            for (int k = i + 1; k < D; ++k) s = s - conj(Lm[k][i]) * w[k];
            w[i] = (1.0 / Lm[i][i].x) * s;
        }
    }
    for (int i = 0; i < D; ++i) {
        a.W[(size_t)idx * D + i] = make_float2((float)w[i].x, (float)w[i].y);
        if (a.T1) a.T1[(size_t)idx * D + i] = make_float2((float)t1[i].x, (float)t1[i].y);
    }
}

template <int D>
static cudaError_t launch_d(const SolveArgs& a, cudaStream_t st) {
    if (a.part != nullptr)
        mwf_solve_kernel<D, 1, true><<<(a.n_mat + 63) / 64, 64, 0, st>>>(a);
    else
        mwf_solve_kernel<D, 1, false><<<(a.n_mat + 63) / 64, 64, 0, st>>>(a);
    return cudaGetLastError();
}

}  // namespace small

cudaError_t launch_mwf_solve_small(const SolveArgs& a, cudaStream_t st) {
    switch (a.D) {
        case 1: return small::launch_d<1>(a, st);
        case 2: return small::launch_d<2>(a, st);
        case 3: return small::launch_d<3>(a, st);
        case 4: return small::launch_d<4>(a, st);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace disco
