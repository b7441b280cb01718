// Relative pose on the device: `estimate_pose` (romatch/utils/utils.py:30-51), i.e. cv2.findEssentialMat (plain RANSAC over
// Nister's five-point solver, OpenCV's E error and stopping rule) followed by cv2.recoverPose, for a batch of pairs.
// The estimator is OpenCV's; only the stream of minimal samples differs (Philox4x32-10, documented in include/romab200.h).
//   norm       xn = inv(K[:2,:2]) (x - K[:2,2]) in float64 (closed-form 2x2 inverse), one thread per point;
//   solve      one warp per hypothesis.  Lane j owns column j of the 5x9 epipolar system (its null space is orthonormalised by
//              modified Gram-Schmidt) and then of Nister's 10x20 constraint matrix, so Gauss-Jordan with partial pivoting runs on registers with shuffles (no spill); the constraint rows
//              (det E = 0, 2 E E^T E - tr(E E^T) E = 0) are expanded by lanes 0-9 into shared memory.  Lane 0 then forms the
//              degree-10 polynomial in z, isolates its real roots with a Sturm sequence (bisection on sign-change counts),
//              refines each by bisection and Newton, and back-substitutes x, y: up to 10 E per sample;
//   score      one thread per (hypothesis, solution slot), the model in registers, the pair's points streamed through shared
//              memory; grid.y cuts the points into slices whose integer partial counts `select` adds in a fixed order;
//   select     one thread per pair replays OpenCV's sequential loop over (hypothesis, solution);
//   recover    one CTA per pair: 3x3 SVD of E (Jacobi on E^T E), linear (DLT) triangulation of every point for the four
//              (R, +-t) with the smallest eigenvector of A^T A (4x4 Jacobi), OpenCV's chirality / distance tests.
// Everything is deterministic: no atomics, no order-dependent sums.
#include "geometry.cuh"

namespace rb {

constexpr int PS_ROUND = RB_POSE_ROUND;
constexpr int PS_SOL = RB_POSE_MAX_SOL;
constexpr int PS_WARPS = 4;                       // hypotheses per CTA of the solver
constexpr int PS_THREADS = 128;                   // score: hypotheses per CTA
constexpr int PS_TILE = 256;                      // score: points per shared-memory tile (8 KB)
constexpr int PS_RECOVER_THREADS = 256;
enum { ST_ITER = 0, ST_NITERS, ST_BEST, ST_HYP, ST_SOL, ST_NE, ST_RUN, ST_N };
constexpr unsigned FULL = 0xffffffffu;

// ---------------------------------------------------------------------------------------------------------------- norm
__global__ void __launch_bounds__(256) pose_norm_kernel(rb_pose_args a) {
    rb::pdl_wait();
    const int b = blockIdx.y;
    const int64_t o0 = a.offsets[b], o1 = a.offsets[b + 1];
    for (int64_t i = o0 + (int64_t)blockIdx.x * 256 + threadIdx.x; i < o1; i += (int64_t)gridDim.x * 256) {
#pragma unroll
        for (int cam = 0; cam < 2; ++cam) {
            const double* K = a.K + (int64_t)b * 18 + cam * 9;
            const double det = __dsub_rn(__dmul_rn(K[0], K[4]), __dmul_rn(K[1], K[3]));
            const double i00 = __ddiv_rn(K[4], det), i01 = __ddiv_rn(-K[1], det), i10 = __ddiv_rn(-K[3], det), i11 = __ddiv_rn(K[0], det);
            const double* x = cam ? a.x1 : a.x0;
            const double dx = __dsub_rn(x[2 * i], K[2]), dy = __dsub_rn(x[2 * i + 1], K[5]);
            a.xn[4 * i + 2 * cam] = __dadd_rn(__dmul_rn(i00, dx), __dmul_rn(i01, dy));
            a.xn[4 * i + 2 * cam + 1] = __dadd_rn(__dmul_rn(i10, dx), __dmul_rn(i11, dy));
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------- solve
// Gauss-Jordan with partial pivoting (first largest |pivot|) of an R x (<= 32) matrix held by columns, lane c owning column c:
// reduces the first R columns to the identity, every operation rounded separately.  Returns false (warp-uniform) on a
// non-finite pivot or one below 1e-12 of the first: a rank-deficient sample (e.g. repeated points) yields no model.
template <int R>
__device__ __forceinline__ bool gauss_jordan_cols(double (&a)[R], int lane) {
    double p0 = 0.0;
#pragma unroll
    for (int k = 0; k < R; ++k) {
        int piv = k;
        double best = -1.0;
#pragma unroll
        for (int r = k; r < R; ++r) {
            const double v = fabs(a[r]);
            if (v > best) { best = v; piv = r; }
        }
        piv = __shfl_sync(FULL, piv, k);
#pragma unroll
        for (int r = k + 1; r < R; ++r)
            if (r == piv) { const double t = a[k]; a[k] = a[r]; a[r] = t; }
        const double p = __shfl_sync(FULL, a[k], k);
        if (k == 0) p0 = fabs(p);
        if (!(fabs(p) > 1e-12 * p0) || !isfinite(p)) return false;
        a[k] = __ddiv_rn(a[k], p);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            if (r == k) continue;
            const double f = __shfl_sync(FULL, a[r], k);
            a[r] = __dsub_rn(a[r], __dmul_rn(f, a[k]));
        }
    }
    return true;
}

// monomials: degree 1 over (x, y, z, 1) -> 0..3; degree <= 2 as sorted pairs (u <= v) -> 0..9; degree <= 3 in Nister's column
// order x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy | xz^2 xz x yz^2 yz y z^3 z^2 z 1
__host__ __device__ constexpr int mono2(int u, int v) { return (u == 0 ? 0 : u == 1 ? 4 : u == 2 ? 7 : 9) + (v - u); }
__host__ __device__ constexpr int mono3_exp(int key) {          // key = 16 ex + 4 ey + ez
    switch (key) {
        case 48: return 0; case 12: return 1; case 36: return 2; case 24: return 3; case 33: return 4; case 32: return 5;
        case 9: return 6; case 8: return 7; case 21: return 8; case 20: return 9; case 18: return 10; case 17: return 11;
        case 16: return 12; case 6: return 13; case 5: return 14; case 4: return 15; case 3: return 16; case 2: return 17;
        case 1: return 18; default: return 19;
    }
}
// the product of variables u, v, w (3 = the constant)
__host__ __device__ constexpr int mono3(int u, int v, int w) {
    return mono3_exp(16 * ((u == 0) + (v == 0) + (w == 0)) + 4 * ((u == 1) + (v == 1) + (w == 1)) + ((u == 2) + (v == 2) + (w == 2)));
}

// out2 += s * a * b (degree-1 polynomials)
__device__ __forceinline__ void mul11(const double* a, const double* b, double s, double (&out)[10]) {
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) out[mono2(u < v ? u : v, u < v ? v : u)] += s * (a[u] * b[v]);
}
// out3 += s * p2 * b
__device__ __forceinline__ void mul21(const double (&p)[10], const double* b, double s, double (&out)[20]) {
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = u; v < 4; ++v)
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                const int x = u, y = v, z = w;
                const int s0 = z < x ? z : x, s2 = z > y ? z : y, s1 = x + y + z - s0 - s2;
                out[mono3(s0, s1, s2)] += s * (p[mono2(u, v)] * b[w]);
            }
}

template <int NA, int NB>
__device__ __forceinline__ void polymul(const double (&a)[NA], const double (&b)[NB], double (&out)[NA + NB - 1]) {
#pragma unroll
    for (int i = 0; i < NA + NB - 1; ++i) out[i] = 0.0;
#pragma unroll
    for (int i = 0; i < NA; ++i)
#pragma unroll
        for (int j = 0; j < NB; ++j) out[i + j] += a[i] * b[j];
}

template <int N>
__device__ __forceinline__ double horner_n(const double (&p)[N], double x) {
    double v = p[N - 1];
#pragma unroll
    for (int i = N - 2; i >= 0; --i) v = v * x + p[i];
    return v;
}

__device__ __forceinline__ double horner(const double* p, int deg, double x) {
    double v = p[deg];
    for (int i = deg - 1; i >= 0; --i) v = v * x + p[i];
    return v;
}

// per-warp shared scratch of the solver
struct SolveSmem {
    double basis[4][9];           // null vectors X, Y, Z, W of the 5x9 system: E = x X + y Y + z Z + W
    double M[10][20];             // constraint matrix, then (after elimination) its right half
    double sturm[11][12];         // Sturm sequence, ascending coefficients
    int deg[11];
};

// number of sign changes of the Sturm sequence at x
__device__ __forceinline__ int sturm_changes(const SolveSmem& S, int ns, double x) {
    int changes = 0, last = 0;
    for (int k = 0; k < ns; ++k) {
        const double v = horner(S.sturm[k], S.deg[k], x);
        const int sg = v > 0.0 ? 1 : (v < 0.0 ? -1 : 0);
        if (sg != 0) {
            if (last != 0 && sg != last) ++changes;
            last = sg;
        }
    }
    return changes;
}

__global__ void __launch_bounds__(PS_WARPS * 32) pose_solve_kernel(rb_pose_args a) {
    rb::pdl_wait();
    __shared__ SolveSmem smem[PS_WARPS];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SolveSmem& S = smem[w];
    const int b = blockIdx.y, hl = blockIdx.x * PS_WARPS + w;
    const int64_t h = (int64_t)a.round * PS_ROUND + hl;
    const int64_t slot = (int64_t)b * PS_ROUND + hl;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    if (!(ransac_drawn<5>(n, h, a.max_iters) && (a.round == 0 || a.state[b * RB_POSE_STATE + ST_RUN] != 0))) {
        if (lane == 0) a.nsol[slot] = 0;
        return;
    }
    // ---- draw 5 distinct indices (lane 0), broadcast
    int id[5] = {0, 1, 2, 3, 4};
    if (n > 5 && lane == 0) ransac_draw(id, n, a.seed, [&](uint32_t sub) { return make_uint4((uint32_t)h, (uint32_t)b, sub, 0u); });
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        id[k] = __shfl_sync(FULL, id[k], 0);
        if (lane == k) a.sample[slot * 5 + k] = id[k];
    }
    // ---- 5x9 system q . e = 0, e = E row-major, q = (x1 x0, x1 y0, x1, y1 x0, y1 y0, y1, x0, y0, 1); lane j owns column j
    double q[5];
#pragma unroll
    for (int r = 0; r < 5; ++r) {
        const double* p = a.xn + 4 * (off + id[r]);
        const double x0 = p[0], y0 = p[1], x1 = p[2], y1 = p[3];
        const int c = lane < 9 ? lane : 8;
        const double u = c < 3 ? x1 : (c < 6 ? y1 : 1.0);
        const int m = c % 3;
        const double v = m == 0 ? x0 : (m == 1 ? y0 : 1.0);
        q[r] = lane < 9 ? u * v : 0.0;
    }
    bool ok = gauss_jordan_cols<5>(q, lane);
    double* out_E = a.E + slot * PS_SOL * 9;
    if (!ok) {
        if (lane == 0) a.nsol[slot] = 0;
        return;
    }
    if (lane >= 5 && lane < 9) {                // free column c: null vector v[r] = -F[r][c] (r < 5), v[c] = 1
#pragma unroll
        for (int r = 0; r < 5; ++r) S.basis[lane - 5][r] = -q[r];
#pragma unroll
        for (int c = 5; c < 9; ++c) S.basis[lane - 5][c] = c == lane ? 1.0 : 0.0;
    }
    __syncwarp();
    if (lane < 9) {                             // modified Gram-Schmidt, lane k owning entry k: an orthonormal basis conditions the solver
#pragma unroll
        for (int i = 0; i < 4; ++i) {
#pragma unroll
            for (int j = 0; j < i; ++j) {
                double d = 0.0;
                for (int k = 0; k < 9; ++k) d += S.basis[i][k] * S.basis[j][k];
                __syncwarp(0x1ffu);
                S.basis[i][lane] -= d * S.basis[j][lane];
                __syncwarp(0x1ffu);
            }
            double nn = 0.0;
            for (int k = 0; k < 9; ++k) nn += S.basis[i][k] * S.basis[i][k];
            __syncwarp(0x1ffu);
            S.basis[i][lane] /= sqrt(nn);
            __syncwarp(0x1ffu);
        }
    }
    __syncwarp();
    // ---- constraint rows: lane 0 det(E), lanes 1..9 entry (i, j) of 2 E E^T E - tr(E E^T) E, as cubics in (x, y, z)
    if (lane < 10) {
        double row[20];
#pragma unroll
        for (int c = 0; c < 20; ++c) row[c] = 0.0;
        auto ld = [&](int k, double* e) {
#pragma unroll
            for (int c = 0; c < 4; ++c) e[c] = S.basis[c][k];
        };
        if (lane == 0) {
            const int cof[3][5] = {{0, 4, 8, 5, 7}, {1, 3, 8, 5, 6}, {2, 3, 7, 4, 6}};   // e_0j * (e_a e_b - e_c e_d)
            const double sgn[3] = {1.0, -1.0, 1.0};
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                double m2[10];
#pragma unroll
                for (int c = 0; c < 10; ++c) m2[c] = 0.0;
                double ea[4], eb[4], e0[4];
                ld(cof[j][1], ea); ld(cof[j][2], eb); mul11(ea, eb, 1.0, m2);
                ld(cof[j][3], ea); ld(cof[j][4], eb); mul11(ea, eb, -1.0, m2);
                ld(cof[j][0], e0);
                mul21(m2, e0, sgn[j], row);
            }
        } else {
            const int i = (lane - 1) / 3, j = (lane - 1) % 3;
            double tr[10];
#pragma unroll
            for (int c = 0; c < 10; ++c) tr[c] = 0.0;
#pragma unroll
            for (int k = 0; k < 9; ++k) { double e[4]; ld(k, e); mul11(e, e, 1.0, tr); }
            double eij[4];
            ld(3 * i + j, eij);
            mul21(tr, eij, -1.0, row);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                double A[10];
#pragma unroll
                for (int c = 0; c < 10; ++c) A[c] = 0.0;
#pragma unroll
                for (int l = 0; l < 3; ++l) { double ea[4], eb[4]; ld(3 * i + l, ea); ld(3 * k + l, eb); mul11(ea, eb, 1.0, A); }
                double ekj[4];
                ld(3 * k + j, ekj);
                mul21(A, ekj, 2.0, row);
            }
        }
#pragma unroll
        for (int c = 0; c < 20; ++c) S.M[lane][c] = row[c];
    }
    __syncwarp();
    double col[10];
#pragma unroll
    for (int r = 0; r < 10; ++r) col[r] = lane < 20 ? S.M[r][lane] : 0.0;
    __syncwarp();
    ok = gauss_jordan_cols<10>(col, lane);
    if (!ok) {
        if (lane == 0) a.nsol[slot] = 0;
        return;
    }
    if (lane >= 10 && lane < 20) {
#pragma unroll
        for (int r = 0; r < 10; ++r) S.M[r][lane] = col[r];
    }
    __syncwarp();
    if (lane != 0) return;
    // ---- lane 0: rows 4-9 express x^2z, x^2, y^2z, y^2, xyz, xy in the last 10 monomials; <k> = row4 - z row5, <l> = row6 - z row7,
    // <m> = row8 - z row9 are linear in (x, y, 1) with polynomial coefficients in z (degrees 3, 3, 4)
    double px[3][4], py[3][4], p1[3][5];
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        const int ra = 4 + 2 * e, rb = ra + 1;
#pragma unroll
        for (int c = 0; c < 4; ++c) { px[e][c] = 0.0; py[e][c] = 0.0; }
#pragma unroll
        for (int c = 0; c < 5; ++c) p1[e][c] = 0.0;
#pragma unroll
        for (int p = 0; p < 3; ++p) {            // columns 10..12: x z^2, x z, x; 13..15: y z^2, y z, y
            px[e][2 - p] -= S.M[ra][10 + p]; px[e][3 - p] += S.M[rb][10 + p];
            py[e][2 - p] -= S.M[ra][13 + p]; py[e][3 - p] += S.M[rb][13 + p];
        }
#pragma unroll
        for (int p = 0; p < 4; ++p) {            // columns 16..19: z^3, z^2, z, 1
            p1[e][3 - p] -= S.M[ra][16 + p]; p1[e][4 - p] += S.M[rb][16 + p];
        }
    }
    // det [[kx ky k1] [lx ly l1] [mx my m1]] = kx (ly m1 - l1 my) - ky (lx m1 - l1 mx) + k1 (lx my - ly mx)
    double poly[11];
    {
        double t7a[8], t7b[8], t6a[7], t6b[7], c10[11];
#pragma unroll
        for (int i = 0; i < 11; ++i) poly[i] = 0.0;
        polymul(py[1], p1[2], t7a); polymul(p1[1], py[2], t7b);
        double m0[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) m0[i] = t7a[i] - t7b[i];
        polymul(px[0], m0, c10);
#pragma unroll
        for (int i = 0; i < 11; ++i) poly[i] += c10[i];
        polymul(px[1], p1[2], t7a); polymul(p1[1], px[2], t7b);
#pragma unroll
        for (int i = 0; i < 8; ++i) m0[i] = t7a[i] - t7b[i];
        polymul(py[0], m0, c10);
#pragma unroll
        for (int i = 0; i < 11; ++i) poly[i] -= c10[i];
        polymul(px[1], py[2], t6a); polymul(py[1], px[2], t6b);
        double m2[7];
#pragma unroll
        for (int i = 0; i < 7; ++i) m2[i] = t6a[i] - t6b[i];
        polymul(p1[0], m2, c10);
#pragma unroll
        for (int i = 0; i < 11; ++i) poly[i] += c10[i];
    }
    // ---- Sturm sequence: p0 = poly (scaled to max |coef| = 1), p1 = p0', p_{k+1} = -rem(p_{k-1}, p_k), each rescaled
    int deg0 = 10;
    while (deg0 > 0 && poly[deg0] == 0.0) --deg0;
    double scale = 0.0;
    for (int i = 0; i <= deg0; ++i) scale = fmax(scale, fabs(poly[i]));
    int nsol = 0;
    if (deg0 >= 1 && scale > 0.0 && isfinite(scale)) {
        for (int i = 0; i <= deg0; ++i) S.sturm[0][i] = poly[i] / scale;
        S.deg[0] = deg0;
        for (int i = 1; i <= deg0; ++i) S.sturm[1][i - 1] = i * S.sturm[0][i];
        S.deg[1] = deg0 - 1;
        int ns = 2;
        while (ns < 11 && S.deg[ns - 1] > 0) {
            double* r = S.sturm[ns];
            const double* u = S.sturm[ns - 2];
            const double* v = S.sturm[ns - 1];
            const int du = S.deg[ns - 2], dv = S.deg[ns - 1];
            for (int i = 0; i <= du; ++i) r[i] = u[i];
            for (int i = du; i >= dv; --i) {
                const double f = r[i] / v[dv];
                for (int j = 0; j <= dv; ++j) r[i - dv + j] -= f * v[j];
            }
            int dr = dv - 1;
            double mx = 0.0;
            for (int i = 0; i <= dr; ++i) mx = fmax(mx, fabs(r[i]));
            if (!(mx > 0.0) || !isfinite(mx)) break;
            while (dr > 0 && r[dr] == 0.0) --dr;
            for (int i = 0; i <= dr; ++i) r[i] = -r[i] / mx;
            S.deg[ns] = dr;
            ++ns;
        }
        // Cauchy bound on the real roots
        double bound = 0.0;
        const double lead = S.sturm[0][deg0];
        for (int i = 0; i < deg0; ++i) bound = fmax(bound, fabs(S.sturm[0][i] / lead));
        bound = 1.0 + bound;
        if (isfinite(bound)) {
            const double lo0 = -bound, hi0 = bound;
            const int v_lo0 = sturm_changes(S, ns, lo0), v_hi0 = sturm_changes(S, ns, hi0);
            const int nroots = v_lo0 - v_hi0;       // distinct real roots in (lo0, hi0]
            double lo = lo0;
            int k = 1;                              // root k in ascending order: N(lo) < k <= N(hi), N(x) = v_lo0 - V(x)
            while (k <= nroots && nsol < PS_SOL) {
                double hi = hi0;
                int nlo = v_lo0 - sturm_changes(S, ns, lo), nhi = nroots;
                for (int it = 0; it < 200 && nhi - nlo > 1; ++it) {   // isolate: exactly one root in (lo, hi]
                    const double mid = 0.5 * (lo + hi);
                    if (!(mid > lo && mid < hi)) break;
                    const int nm = v_lo0 - sturm_changes(S, ns, mid);
                    if (nm >= k) { hi = mid; nhi = nm; } else { lo = mid; nlo = nm; }
                }
                // refine: bisection on the sign of p0, then Newton
                const double* p = S.sturm[0];
                double a0 = lo, b0 = hi, fa = horner(p, deg0, a0);
                const double fb = horner(p, deg0, b0);
                double z = 0.5 * (a0 + b0);
                if ((fa < 0.0) != (fb < 0.0)) {
                    for (int it = 0; it < 120; ++it) {
                        const double mid = 0.5 * (a0 + b0);
                        if (!(mid > a0 && mid < b0)) break;
                        const double fm = horner(p, deg0, mid);
                        if ((fm < 0.0) == (fa < 0.0)) { a0 = mid; fa = fm; } else b0 = mid;
                    }
                    z = 0.5 * (a0 + b0);
                }
#pragma unroll 1
                for (int it = 0; it < 2; ++it) {
                    double f = p[deg0], d = 0.0;
                    for (int i = deg0 - 1; i >= 0; --i) { d = d * z + f; f = f * z + p[i]; }
                    const double zn = z - f / d;
                    if (isfinite(zn) && zn >= lo && zn <= hi) z = zn;
                }
                // back-substitution: (x, y, 1) is the null vector of B(z); take the cross product of two rows with the largest |third component|
                double B[3][3];
#pragma unroll
                for (int e = 0; e < 3; ++e) {
                    B[e][0] = horner_n(px[e], z); B[e][1] = horner_n(py[e], z); B[e][2] = horner_n(p1[e], z);
                }
                double cx = 0.0, cy = 0.0, cz = 0.0;
#pragma unroll
                for (int pr = 0; pr < 3; ++pr) {
                    const int r0 = pr == 2 ? 1 : 0, r1 = pr == 0 ? 1 : 2;
                    const double vx = B[r0][1] * B[r1][2] - B[r0][2] * B[r1][1];
                    const double vy = B[r0][2] * B[r1][0] - B[r0][0] * B[r1][2];
                    const double vz = B[r0][0] * B[r1][1] - B[r0][1] * B[r1][0];
                    if (fabs(vz) > fabs(cz)) { cx = vx; cy = vy; cz = vz; }
                }
                const double x = cx / cz, y = cy / cz;
                double E[9], ss = 0.0;
#pragma unroll
                for (int i = 0; i < 9; ++i) {
                    E[i] = x * S.basis[0][i] + y * S.basis[1][i] + z * S.basis[2][i] + S.basis[3][i];
                    ss += E[i] * E[i];
                }
                const double nrm = sqrt(ss);
                bool fin = nrm > 0.0 && isfinite(nrm);
                double emax = E[0];              // the first entry of largest magnitude
#pragma unroll
                for (int i = 1; i < 9; ++i)
                    if (fabs(E[i]) > fabs(emax)) emax = E[i];
                const double sgn = emax < 0.0 ? -1.0 : 1.0;
                if (fin) {
#pragma unroll
                    for (int i = 0; i < 9; ++i) {
                        E[i] = sgn * (E[i] / nrm);
                        fin &= isfinite(E[i]);
                    }
                }
                if (fin) {
#pragma unroll
                    for (int i = 0; i < 9; ++i) out_E[nsol * 9 + i] = E[i];
                    ++nsol;
                }
                // the next root lies above hi; a cluster that could not be isolated counts once
                k = nhi + 1;
                lo = hi;
            }
        }
    }
    a.nsol[slot] = nsol;
}

// ---------------------------------------------------------------------------------------------------------------- score
// OpenCV's EMEstimatorCallback::computeError in float64 with every operation rounded separately, then rounded to float and
// compared with (float)(thresh^2).  A NaN error (NaN point, 0/0) is never an inlier.
__device__ __forceinline__ bool pose_inlier(const double (&e)[9], double x0, double y0, double x1, double y1, float t) {
    const double ex0 = __dadd_rn(__dadd_rn(__dmul_rn(e[0], x0), __dmul_rn(e[1], y0)), e[2]);
    const double ex1 = __dadd_rn(__dadd_rn(__dmul_rn(e[3], x0), __dmul_rn(e[4], y0)), e[5]);
    const double ex2 = __dadd_rn(__dadd_rn(__dmul_rn(e[6], x0), __dmul_rn(e[7], y0)), e[8]);
    const double et0 = __dadd_rn(__dadd_rn(__dmul_rn(e[0], x1), __dmul_rn(e[3], y1)), e[6]);
    const double et1 = __dadd_rn(__dadd_rn(__dmul_rn(e[1], x1), __dmul_rn(e[4], y1)), e[7]);
    const double v = __dadd_rn(__dadd_rn(__dmul_rn(x1, ex0), __dmul_rn(y1, ex1)), ex2);
    const double den = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(ex0, ex0), __dmul_rn(ex1, ex1)), __dmul_rn(et0, et0)), __dmul_rn(et1, et1));
    const float err = __double2float_rn(__ddiv_rn(__dmul_rn(v, v), den));
    return err <= t;
}

__device__ __forceinline__ float pose_thresh(double th) { return __double2float_rn(__dmul_rn(th, th)); }

// grid (RB_POSE_ROUND / 128, splits, batch * RB_POSE_MAX_SOL): thread = hypothesis, blockIdx.z % 10 = solution slot
__global__ void __launch_bounds__(PS_THREADS) pose_score_kernel(rb_pose_args a, int per_split) {
    rb::pdl_wait();
    __shared__ __align__(16) double4 tile[PS_TILE];
    const int b = blockIdx.z / PS_SOL, s = blockIdx.z % PS_SOL;
    const int hl = blockIdx.x * PS_THREADS + threadIdx.x;
    const int64_t slot = (int64_t)b * PS_ROUND + hl;
    const bool act = s < a.nsol[slot];
    if (!__syncthreads_or(act)) return;
    double e[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) e[i] = act ? a.E[(slot * PS_SOL + s) * 9 + i] : 0.0;
    const float t = pose_thresh(a.thresh);
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const double4* pts = reinterpret_cast<const double4*>(a.xn) + off;
    const int cnt = ransac_count<PS_THREADS>(tile, n, per_split, act, [&](int64_t j) { return pts[j]; },
                                             [&](const double4& p) { return pose_inlier(e, p.x, p.y, p.z, p.w, t); });
    if (act) a.counts[(((int64_t)b * RB_POSE_MAX_SPLITS + blockIdx.y) * PS_SOL + s) * PS_ROUND + hl] = cnt;
}

// ---------------------------------------------------------------------------------------------------------------- select
__global__ void __launch_bounds__(128) pose_select_kernel(rb_pose_args a, int splits) {
    rb::pdl_wait();
    const int b = blockIdx.x * 128 + threadIdx.x;
    if (b >= a.batch) return;
    int* st = a.state + (int64_t)b * RB_POSE_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const int64_t slot0 = (int64_t)b * PS_ROUND;
    if (a.round == 0) {
        st[ST_ITER] = 0; st[ST_NITERS] = a.max_iters; st[ST_BEST] = 0; st[ST_HYP] = -1; st[ST_SOL] = -1; st[ST_NE] = 0;
        st[ST_RUN] = n >= 5; st[ST_N] = (int)n;
        if (n == 5) {                    // OpenCV's count == modelPoints case: every solution, all points inliers
            const int ns = a.nsol[slot0];
            for (int i = 0; i < ns * 9; ++i) a.best_E[(int64_t)b * PS_SOL * 9 + i] = a.E[slot0 * PS_SOL * 9 + i];
            st[ST_NE] = ns; st[ST_BEST] = ns > 0 ? 5 : 0; st[ST_HYP] = ns > 0 ? 0 : -1; st[ST_SOL] = ns > 0 ? 0 : -1;
            st[ST_RUN] = 0;
            return;
        }
    }
    if (!st[ST_RUN]) return;
    int iter = st[ST_ITER], niters = st[ST_NITERS], best = st[ST_BEST];
    const int64_t per_split_stride = (int64_t)PS_SOL * PS_ROUND;
    for (int hl = 0; hl < PS_ROUND && iter < niters; ++hl, ++iter) {
        const int ns = a.nsol[slot0 + hl];
        for (int s = 0; s < ns; ++s) {
            int cnt = 0;
            const int32_t* c = a.counts + (int64_t)b * RB_POSE_MAX_SPLITS * per_split_stride + (int64_t)s * PS_ROUND + hl;
            for (int y = 0; y < splits; ++y) cnt += c[y * per_split_stride];
            if (cnt > max(best, 4)) {
                best = cnt;
                st[ST_HYP] = iter; st[ST_SOL] = s;
                for (int i = 0; i < 9; ++i) a.best_E[(int64_t)b * PS_SOL * 9 + i] = a.E[((slot0 + hl) * PS_SOL + s) * 9 + i];
                niters = ransac_update_num_iters<5>(a.conf, (double)(n - cnt) / (double)n, niters);
            }
        }
    }
    st[ST_ITER] = iter; st[ST_NITERS] = niters; st[ST_BEST] = best; st[ST_NE] = best > 0 ? 1 : 0;
    st[ST_RUN] = iter < niters;
    if (iter < niters) a.running[0] = 1;
}

// ---------------------------------------------------------------------------------------------------------------- recover
// cv::decomposeEssentialMat: E = U diag V^T with det U = det V = 1, R1 = U W V^T, R2 = U W^T V^T, t = U[:, 2]
__device__ void decompose_essential(const double* E, double (&R1)[9], double (&R2)[9], double (&tv)[3]) {
    double v[3][3], u[3][3], sv[2];             // v[k] = k-th right singular vector
    svd3(E, u, v, sv);
    // U W V^T with W = [[0 1 0] [-1 0 0] [0 0 1]]: columns of U W are (-u1, u0, u2); of U W^T: (u1, -u0, u2)
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            R1[3 * i + j] = -u[1][i] * v[0][j] + u[0][i] * v[1][j] + u[2][i] * v[2][j];
            R2[3 * i + j] = u[1][i] * v[0][j] - u[0][i] * v[1][j] + u[2][i] * v[2][j];
        }
#pragma unroll
    for (int i = 0; i < 3; ++i) tv[i] = u[2][i];
}

// cv::recoverPose's test for one candidate P1 = [R | t] (P0 = [I | 0]): DLT triangulation (dlt_two_view), Q.z Q.w > 0, Q.z / Q.w < dist, 0 < (P1 Q / Q.w).z < dist
__device__ __forceinline__ bool chirality(const double* R, const double* t, double x0, double y0, double x1, double y1) {
    constexpr double dist = 1e9;
    double Q[4];
    dlt_two_view(R, t, x0, y0, x1, y1, Q);
    if (!(Q[2] * Q[3] > 0.0)) return false;
    const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
    if (!(Z < dist)) return false;
    const double z2 = R[6] * X + R[7] * Y + R[8] * Z + t[2];
    return z2 > 0.0 && z2 < dist;
}

__global__ void __launch_bounds__(PS_RECOVER_THREADS, 1) pose_recover_kernel(rb_pose_args a) {
    rb::pdl_wait();
    __shared__ double cand[4][12];      // R (9) and t (3) of the four candidates
    __shared__ int good[PS_RECOVER_THREADS / 32][4];
    __shared__ double bestRt[12];
    __shared__ uint8_t snap[5];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int* st = a.state + (int64_t)b * RB_POSE_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const int nE = n >= 5 ? st[ST_NE] : 0;
    const float thr = pose_thresh(a.thresh);
    const double* bestE = a.best_E + (int64_t)b * PS_SOL * 9;
    int best_n = 0;
    if (tid < 12) bestRt[tid] = 0.0;
    for (int e = 0; e < nE; ++e) {
        const double* E = bestE + e * 9;
        if (tid == 0) {
            double R1[9], R2[9], tv[3];
            decompose_essential(E, R1, R2, tv);
            for (int i = 0; i < 9; ++i) { cand[0][i] = R1[i]; cand[1][i] = R2[i]; cand[2][i] = R1[i]; cand[3][i] = R2[i]; }
            for (int i = 0; i < 3; ++i) { cand[0][9 + i] = tv[i]; cand[1][9 + i] = tv[i]; cand[2][9 + i] = -tv[i]; cand[3][9 + i] = -tv[i]; }
        }
        __syncthreads();
        double ev[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) ev[i] = E[i];
        int g[4] = {0, 0, 0, 0};
        for (int64_t i = tid; i < n; i += PS_RECOVER_THREADS) {
            const double* p = a.xn + 4 * (off + i);
            const double x0 = p[0], y0 = p[1], x1 = p[2], y1 = p[3];
            bool in;
            if (e > 0) in = a.mask[off + i] != 0;
            else if (st[ST_N] == 5) in = true;
            else in = pose_inlier(ev, x0, y0, x1, y1, thr);
            uint8_t code = 0;
            if (in) {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (chirality(cand[c], cand[c] + 9, x0, y0, x1, y1)) { code |= (uint8_t)(1u << c); ++g[c]; }
            }
            a.mask[off + i] = code;
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
#pragma unroll
            for (int d = 16; d; d >>= 1) g[c] += __shfl_xor_sync(FULL, g[c], d);
            if ((tid & 31) == 0) good[tid >> 5][c] = g[c];
        }
        __syncthreads();
        int G[4] = {0, 0, 0, 0};
        for (int w = 0; w < PS_RECOVER_THREADS / 32; ++w)
#pragma unroll
            for (int c = 0; c < 4; ++c) G[c] += good[w][c];
        int c;
        if (G[0] >= G[1] && G[0] >= G[2] && G[0] >= G[3]) c = 0;
        else if (G[1] >= G[0] && G[1] >= G[2] && G[1] >= G[3]) c = 1;
        else if (G[2] >= G[0] && G[2] >= G[1] && G[2] >= G[3]) c = 2;
        else c = 3;
        for (int64_t i = tid; i < n; i += PS_RECOVER_THREADS) a.mask[off + i] = (a.mask[off + i] >> c) & 1u;
        if (G[c] > best_n) {
            best_n = G[c];
            if (tid < 12) bestRt[tid] = cand[c][tid];
            if (nE > 1 && tid < 5) snap[tid] = a.mask[off + tid];       // n == 5: the reference keeps the mask of its best call
        }
        __syncthreads();
    }
    if (nE == 0)
        for (int64_t i = tid; i < n; i += PS_RECOVER_THREADS) a.mask[off + i] = 0;
    if (nE > 1 && tid < 5) a.mask[off + tid] = best_n > 0 ? snap[tid] : 0;
    __syncthreads();
    if (tid < 9) a.R[(int64_t)b * 9 + tid] = bestRt[tid];
    if (tid < 3) a.t[(int64_t)b * 3 + tid] = bestRt[9 + tid];
    if (tid == 0) a.ok[b] = best_n > 0;
}

static int pose_check(const rb_pose_args* a, const char* what) {
    if (ransac_check(a, what, 4096, PS_ROUND)) return 1;
    RB_REQUIRE(a->x0 && a->x1 && a->K && a->xn, "%s: null argument", what);
    return 0;
}

static int pose_splits(int64_t max_n) { return ransac_splits(max_n, 1024, RB_POSE_MAX_SPLITS); }

}  // namespace rb

using namespace rb;

extern "C" int romab200_pose_hypotheses(const rb_pose_args* a, void* stream) {
    if (pose_check(a, "pose_hypotheses")) return 1;
    RB_REQUIRE(a->sample && a->E && a->nsol && a->running, "pose_hypotheses: null output");
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(cudaMemsetAsync(a->running, 0, sizeof(int32_t), st) == cudaSuccess, "pose_hypotheses: memset failed");
    if (a->round == 0) {
        const int64_t g = (a->max_n + 255) / 256;
        const int gx = g < 1 ? 1 : (g > 64 ? 64 : (int)g);
        rb::launch_pdl(pose_norm_kernel, dim3(gx, a->batch), dim3(256), 0, st, *a);
        if (check_launch("pose_hypotheses(normalise)")) return 1;
    }
    rb::launch_pdl(pose_solve_kernel, dim3(PS_ROUND / PS_WARPS, a->batch), dim3(PS_WARPS * 32), 0, st, *a);
    return check_launch("pose_hypotheses(solve)");
}

extern "C" int romab200_pose_score(const rb_pose_args* a, void* stream) {
    if (pose_check(a, "pose_score")) return 1;
    RB_REQUIRE(a->E && a->nsol && a->counts, "pose_score: null argument");
    const int splits = pose_splits(a->max_n);
    const int per_split = (int)((a->max_n + splits - 1) / splits);
    rb::launch_pdl(pose_score_kernel, dim3(PS_ROUND / PS_THREADS, splits, a->batch * PS_SOL), dim3(PS_THREADS), 0, (cudaStream_t)stream, *a,
                   max(per_split, 1));
    return check_launch("pose_score");
}

extern "C" int romab200_pose_select(const rb_pose_args* a, void* stream) {
    if (pose_check(a, "pose_select")) return 1;
    RB_REQUIRE(a->E && a->nsol && a->counts && a->best_E && a->running, "pose_select: null argument");
    rb::launch_pdl(pose_select_kernel, dim3((a->batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, *a, pose_splits(a->max_n));
    return check_launch("pose_select");
}

extern "C" int romab200_pose_recover(const rb_pose_args* a, void* stream) {
    RB_REQUIRE(a && a->offsets && a->xn && a->state && a->best_E && a->R && a->t && a->ok && a->mask, "pose_recover: null argument");
    RB_REQUIRE(a->batch > 0 && a->batch <= 4096, "pose_recover: batch %d outside [1, 4096]", a->batch);
    rb::launch_pdl(pose_recover_kernel, dim3(a->batch), dim3(PS_RECOVER_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("pose_recover");
}
