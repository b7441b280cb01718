// Absolute pose on the device (include/romab200.h): batched P3P RANSAC and Gauss-Newton refinement, and the gather of image
// registration's correspondences against triangulated tracks.
//   hypotheses one thread per hypothesis: three bearings, Lambda Twist P3P, up to RB_ABS_MAX_SOL models (R, t);
//   score      one thread per (hypothesis, solution slot), the model folded into P = K [R | t] in registers, the item's points streamed
//              through shared memory; grid.y cuts the points into slices whose integer partial counts `select` adds;
//   select     one thread per item replays OpenCV's sequential loop over (hypothesis, solution);
//   refine     one CTA per item: Gauss-Newton on the best model's inliers, the 6 x 6 normal equations and the cost summed by cta_sum,
//              every thread solving the same system by Cholesky; then the final inlier mask.
//   register   a warp per track checks its element ids and keys the ok tracks' elements by image; radix_sort_hi32 orders them; the
//              listed images' segments are packed into the estimator's x / X / offsets layout.
// No float atomics and a fixed order in every reduction, so the result is bit-identical from run to run.
#include "geometry.cuh"

namespace rb {

constexpr int AB_ROUND = RB_ABS_ROUND;
constexpr int AB_SOL = RB_ABS_MAX_SOL;
constexpr int AB_HYP_THREADS = 128;
constexpr int AB_THREADS = 128;                   // score: hypotheses per CTA
constexpr int AB_TILE = 256;                      // score: points per shared-memory tile (10 KB)
constexpr int AB_REFINE_THREADS = 256;
constexpr int AB_SUMS = 29;                       // J^T J (21, upper triangle by rows), J^T r (6), cost, depths <= 0
enum { AS_ITER = 0, AS_NITERS, AS_BEST, AS_HYP, AS_SOL, AS_RUN, AS_N };
static_assert(AB_ROUND % AB_THREADS == 0 && AB_ROUND % AB_HYP_THREADS == 0, "a round is a whole number of CTAs");

// ---------------------------------------------------------------------------------------------------------------- helpers
__device__ __forceinline__ double det_cols(const double (&a)[3], const double (&b)[3], const double (&c)[3]) {
    return a[0] * (b[1] * c[2] - b[2] * c[1]) - a[1] * (b[0] * c[2] - b[2] * c[0]) + a[2] * (b[0] * c[1] - b[1] * c[0]);
}

// inverse of a row-major 3 x 3 matrix by cofactors over the determinant
__device__ __forceinline__ void inv3(const double* M, double (&I)[9]) {
    const double c00 = M[4] * M[8] - M[5] * M[7], c01 = M[5] * M[6] - M[3] * M[8], c02 = M[3] * M[7] - M[4] * M[6];
    const double det = M[0] * c00 + M[1] * c01 + M[2] * c02;
    I[0] = c00 / det; I[1] = (M[2] * M[7] - M[1] * M[8]) / det; I[2] = (M[1] * M[5] - M[2] * M[4]) / det;
    I[3] = c01 / det; I[4] = (M[0] * M[8] - M[2] * M[6]) / det; I[5] = (M[2] * M[3] - M[0] * M[5]) / det;
    I[6] = c02 / det; I[7] = (M[1] * M[6] - M[0] * M[7]) / det; I[8] = (M[0] * M[4] - M[1] * M[3]) / det;
}

// the real roots of g^3 + b g^2 + c g + d in descending order (Cardano or the trigonometric form, two Newton steps each); returns
// their number
__device__ __forceinline__ int cubic_roots(double b, double c, double d, double (&g)[3]) {
    const double p = c - b * b / 3.0, q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d;
    const double disc = q * q / 4.0 + p * p * p / 27.0;
    int nr;
    if (disc > 0.0) {
        const double s = sqrt(disc);
        g[0] = cbrt(-q / 2.0 + s) + cbrt(-q / 2.0 - s) - b / 3.0;
        nr = 1;
    } else {
        const double r = sqrt(fmax(-p / 3.0, 0.0));
        const double arg = r == 0.0 ? 0.0 : fmin(fmax(-q / (2.0 * r * r * r), -1.0), 1.0);
        const double phi = acos(arg);
#pragma unroll
        for (int k = 0; k < 3; ++k) g[k] = 2.0 * r * cospi((phi * (1.0 / CUDART_PI) - 2.0 * k) / 3.0) - b / 3.0;   // cospi: no stack
        nr = 3;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (k >= nr) break;
#pragma unroll 1
        for (int it = 0; it < 2; ++it) {
            const double f = ((g[k] + b) * g[k] + c) * g[k] + d, df = (3.0 * g[k] + 2.0 * b) * g[k] + c;
            if (df != 0.0) {
                const double g1 = g[k] - f / df;
                if (isfinite(g1)) g[k] = g1;
            }
        }
    }
    if (nr == 3) {                                 // descending
        if (g[1] > g[0]) { const double t = g[0]; g[0] = g[1]; g[1] = t; }
        if (g[2] > g[1]) { const double t = g[1]; g[1] = g[2]; g[2] = t; }
        if (g[1] > g[0]) { const double t = g[0]; g[0] = g[1]; g[1] = t; }
    }
    return nr;
}

// Lambda Twist's depth polish: Newton steps on l_i^2 + l_j^2 - 2 b_ij l_i l_j - a_ij, kept while the sum of squares falls
__device__ __forceinline__ void polish_depths(double (&l)[3], const double (&A)[3], const double (&B)[3]) {
    auto res = [&](const double (&v)[3], double (&r)[3]) {
        r[0] = v[0] * v[0] + v[1] * v[1] - 2.0 * B[0] * v[0] * v[1] - A[0];
        r[1] = v[0] * v[0] + v[2] * v[2] - 2.0 * B[1] * v[0] * v[2] - A[1];
        r[2] = v[1] * v[1] + v[2] * v[2] - 2.0 * B[2] * v[1] * v[2] - A[2];
    };
    double r[3];
    res(l, r);
#pragma unroll 1
    for (int it = 0; it < RB_ABS_POLISH_ITERS; ++it) {
        double J[9] = {2.0 * l[0] - 2.0 * B[0] * l[1], 2.0 * l[1] - 2.0 * B[0] * l[0], 0.0,
                       2.0 * l[0] - 2.0 * B[1] * l[2], 0.0, 2.0 * l[2] - 2.0 * B[1] * l[0],
                       0.0, 2.0 * l[1] - 2.0 * B[2] * l[2], 2.0 * l[2] - 2.0 * B[2] * l[1]};
        double Ji[9];
        inv3(J, Ji);
        double l1[3], r1[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) l1[i] = l[i] - (Ji[3 * i] * r[0] + Ji[3 * i + 1] * r[1] + Ji[3 * i + 2] * r[2]);
        if (!(isfinite(l1[0]) && isfinite(l1[1]) && isfinite(l1[2]))) break;
        res(l1, r1);
        if (!(r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2] < r[0] * r[0] + r[1] * r[1] + r[2] * r[2])) break;
#pragma unroll
        for (int i = 0; i < 3; ++i) { l[i] = l1[i]; r[i] = r1[i]; }
    }
}

// eigenvector column k of V, signed so that its first largest-magnitude entry is positive
__device__ __forceinline__ void canonical_col(const double (&V)[3][3], int k, double (&u)[3]) {
#pragma unroll
    for (int i = 0; i < 3; ++i) u[i] = k == 0 ? V[i][0] : (k == 1 ? V[i][1] : V[i][2]);
    double big = u[0];
    if (fabs(u[1]) > fabs(big)) big = u[1];
    if (fabs(u[2]) > fabs(big)) big = u[2];
    if (big < 0.0) { u[0] = -u[0]; u[1] = -u[1]; u[2] = -u[2]; }
}

// rule 3: Lambda Twist on bearings f and world points Xw (rows); writes up to RB_ABS_MAX_SOL models (R row-major, t) to out, returns
// their number
__device__ int lambda_twist(const double (&f)[3][3], const double (&Xw)[3][3], double* out) {
    double A[3], B[3];                             // a12, a13, a23 and b12, b13, b23
    {
        const int pi[3] = {0, 0, 1}, pj[3] = {1, 2, 2};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const double d0 = Xw[pi[k]][0] - Xw[pj[k]][0], d1 = Xw[pi[k]][1] - Xw[pj[k]][1], d2 = Xw[pi[k]][2] - Xw[pj[k]][2];
            A[k] = d0 * d0 + d1 * d1 + d2 * d2;
            B[k] = f[pi[k]][0] * f[pj[k]][0] + f[pi[k]][1] * f[pj[k]][1] + f[pi[k]][2] * f[pj[k]][2];
        }
    }
    const double a12 = A[0], a13 = A[1], a23 = A[2], b12 = B[0], b13 = B[1], b23 = B[2];
    // D1 = a23 M12 - a12 M23, D2 = a23 M13 - a13 M23 (symmetric: columns = rows)
    const double D1[3][3] = {{a23, -a23 * b12, 0.0}, {-a23 * b12, a23 - a12, a12 * b23}, {0.0, a12 * b23, -a12}};
    const double D2[3][3] = {{a23, 0.0, -a23 * b13}, {0.0, -a13, a13 * b23}, {-a23 * b13, a13 * b23, a23 - a13}};
    const double c3 = det_cols(D2[0], D2[1], D2[2]);
    const double c2 = det_cols(D1[0], D2[1], D2[2]) + det_cols(D2[0], D1[1], D2[2]) + det_cols(D2[0], D2[1], D1[2]);
    const double c1 = det_cols(D2[0], D1[1], D1[2]) + det_cols(D1[0], D2[1], D1[2]) + det_cols(D1[0], D1[1], D2[2]);
    const double c0 = det_cols(D1[0], D1[1], D1[2]);
    if (!(c3 != 0.0 && isfinite(c3))) return 0;
    double roots[3];
    const int nr = cubic_roots(c2 / c3, c1 / c3, c0 / c3, roots);
    // the root whose D0 is indefinite with the largest ratio |sigma2| / |sigma1| (ties to the first): far from a semidefinite D0,
    // whose two lines are complex and whose sign test rounding could flip
    double best_ratio = -1.0, s1 = 0.0, s2 = 0.0, u1[3] = {0.0, 0.0, 0.0}, u2[3] = {0.0, 0.0, 0.0};
#pragma unroll 1
    for (int r = 0; r < nr; ++r) {
        const double g = r == 0 ? roots[0] : (r == 1 ? roots[1] : roots[2]);
        double D0[3][3], V[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) D0[i][j] = D1[i][j] + g * D2[i][j];
        jacobi_eig<3>(D0, V, 10);
        // the two eigenvalues of largest magnitude, ties to the lower index
        const double e[3] = {D0[0][0], D0[1][1], D0[2][2]};
        int i0 = fabs(e[1]) > fabs(e[0]) ? 1 : 0;
        if (fabs(e[2]) > (i0 == 0 ? fabs(e[0]) : fabs(e[1]))) i0 = 2;
        const int i1 = i0 == 0 ? (fabs(e[2]) > fabs(e[1]) ? 2 : 1) : (i0 == 1 ? (fabs(e[2]) > fabs(e[0]) ? 2 : 0) : (fabs(e[1]) > fabs(e[0]) ? 1 : 0));
        const double a0 = i0 == 0 ? e[0] : (i0 == 1 ? e[1] : e[2]), a1 = i1 == 0 ? e[0] : (i1 == 1 ? e[1] : e[2]);
        if (!(a0 * a1 < 0.0)) continue;
        const double ratio = fabs(a1) / fabs(a0);
        if (!(ratio > best_ratio)) continue;
        best_ratio = ratio; s1 = a0; s2 = a1;
        canonical_col(V, i0, u1);
        canonical_col(V, i1, u2);
    }
    int nsol = 0;
    if (best_ratio >= 0.0) {
        if (s1 < 0.0) {
            const double t = s1; s1 = s2; s2 = t;
#pragma unroll
            for (int i = 0; i < 3; ++i) { const double v = u1[i]; u1[i] = u2[i]; u2[i] = v; }
        }
        const double s = sqrt(-s2 / s1);
#pragma unroll 1
        for (int line = 0; line < 2; ++line) {
            const double sg = line == 0 ? -s : s;
            const double n0 = u1[0] + sg * u2[0], n1 = u1[1] + sg * u2[1], n2 = u1[2] + sg * u2[2];
            if (n0 == 0.0) continue;
            const double w0 = -n1 / n0, w1 = -n2 / n0;
            // v = al + tau be, al = (w0, 1, 0), be = (w1, 0, 1): A tau^2 + B tau + C = v^T D2 v
            const double Da[3] = {D2[0][0] * w0 + D2[0][1], D2[1][0] * w0 + D2[1][1], D2[2][0] * w0 + D2[2][1]};
            const double Db[3] = {D2[0][0] * w1 + D2[0][2], D2[1][0] * w1 + D2[1][2], D2[2][0] * w1 + D2[2][2]};
            const double qa = w1 * Db[0] + Db[2], qb = 2.0 * (w0 * Db[0] + Db[1]), qc = w0 * Da[0] + Da[1];
            const double disc = qb * qb - 4.0 * qa * qc;
            if (!(qa != 0.0 && disc >= 0.0)) continue;
            const double qq = -0.5 * (qb + copysign(sqrt(disc), qb));
            if (qq == 0.0) continue;
            const double ta = qq / qa, tb = qc / qq, tau0 = fmin(ta, tb), tau1 = fmax(ta, tb);
#pragma unroll 1
            for (int k = 0; k < 2; ++k) {
                const double tk = k == 0 ? tau0 : tau1;
                if (!(tk > 0.0)) continue;
                const double l2 = sqrt(a23 / (tk * tk - 2.0 * b23 * tk + 1.0));
                double l[3] = {w0 * l2 + w1 * (tk * l2), l2, tk * l2};
                if (!(l[0] > 0.0)) continue;
                polish_depths(l, A, B);
                double Y[3][3];
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) Y[i][j] = l[i] * f[i][j];
                // R = Ym Xm^-1, columns (P1 - P2, P1 - P3, (P1 - P2) x (P1 - P3))
                double Xm[9], Ym[9];
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    Xm[3 * i] = Xw[0][i] - Xw[1][i]; Xm[3 * i + 1] = Xw[0][i] - Xw[2][i];
                    Ym[3 * i] = Y[0][i] - Y[1][i];   Ym[3 * i + 1] = Y[0][i] - Y[2][i];
                }
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    const int j = (i + 1) % 3, k2 = (i + 2) % 3;
                    Xm[3 * i + 2] = Xm[3 * j] * Xm[3 * k2 + 1] - Xm[3 * k2] * Xm[3 * j + 1];
                    Ym[3 * i + 2] = Ym[3 * j] * Ym[3 * k2 + 1] - Ym[3 * k2] * Ym[3 * j + 1];
                }
                double Xi[9], m[12];
                inv3(Xm, Xi);
                bool fin = true;
#pragma unroll
                for (int i = 0; i < 3; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) {
                        m[3 * i + j] = Ym[3 * i] * Xi[j] + Ym[3 * i + 1] * Xi[3 + j] + Ym[3 * i + 2] * Xi[6 + j];
                        fin &= isfinite(m[3 * i + j]);
                    }
#pragma unroll
                for (int i = 0; i < 3; ++i) {
                    m[9 + i] = Y[0][i] - (m[3 * i] * Xw[0][0] + m[3 * i + 1] * Xw[0][1] + m[3 * i + 2] * Xw[0][2]);
                    fin &= isfinite(m[9 + i]);
                }
                if (fin && nsol < AB_SOL) {
#pragma unroll
                    for (int i = 0; i < 12; ++i) out[nsol * 12 + i] = m[i];
                    ++nsol;
                }
            }
        }
    }
    return nsol;
}

// ---------------------------------------------------------------------------------------------------------------- hypotheses
__global__ void __launch_bounds__(AB_HYP_THREADS) abs_hyp_kernel(rb_abspose_args a) {
    pdl_wait();
    const int b = blockIdx.y, hl = blockIdx.x * AB_HYP_THREADS + threadIdx.x;
    const int64_t h = (int64_t)a.round * AB_ROUND + hl;
    const int64_t slot = (int64_t)b * AB_ROUND + hl;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    if (!(ransac_drawn<3>(n, h, a.max_iters) && (a.round == 0 || a.state[(int64_t)b * RB_ABS_STATE + AS_RUN] != 0))) {
        a.nsol[slot] = 0;
        return;
    }
    int id[3];
    ransac_draw<3>(id, n, a.seed, [&](uint32_t sub) { return make_uint4((uint32_t)h, sub, 0u, RB_ABS_CTR); });
    double Ki[9];
    inv3(a.K + (int64_t)b * 9, Ki);
    double f[3][3], Xw[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        a.sample[slot * 3 + k] = id[k];
        const int64_t j = off + id[k];
        const double x = a.x[2 * j], y = a.x[2 * j + 1];
        double nn = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            f[k][i] = Ki[3 * i] * x + Ki[3 * i + 1] * y + Ki[3 * i + 2];
            nn += f[k][i] * f[k][i];
        }
        nn = sqrt(nn);
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            f[k][i] /= nn;
            Xw[k][i] = a.X[3 * j + i];
        }
    }
    a.nsol[slot] = lambda_twist(f, Xw, a.models + slot * AB_SOL * 12);
}

// ---------------------------------------------------------------------------------------------------------------- score
struct AbsPt { double x, y, X0, X1, X2; };

// P = K [R | t] (12, row-major) and the depth row (R row 2, t_z) of a model (R row-major, t)
__device__ __forceinline__ void abs_projection(const double (&R)[9], const double (&t)[3], const double* K, double (&P)[16]) {
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double c0 = j < 3 ? R[j] : t[0], c1 = j < 3 ? R[3 + j] : t[1], c2 = j < 3 ? R[6 + j] : t[2];
            P[4 * i + j] = K[3 * i] * c0 + K[3 * i + 1] * c1 + K[3 * i + 2] * c2;
        }
    P[12] = R[6]; P[13] = R[7]; P[14] = R[8]; P[15] = t[2];
}

__device__ __forceinline__ void abs_load_model(const double* m, double (&R)[9], double (&t)[3]) {
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = m[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) t[i] = m[9 + i];
}

// rule 4
__device__ __forceinline__ bool abs_inlier(const double (&P)[16], const AbsPt& q, double max_error2) {
    const double p0 = P[0] * q.X0 + P[1] * q.X1 + P[2] * q.X2 + P[3];
    const double p1 = P[4] * q.X0 + P[5] * q.X1 + P[6] * q.X2 + P[7];
    const double p2 = P[8] * q.X0 + P[9] * q.X1 + P[10] * q.X2 + P[11];
    const double dz = P[12] * q.X0 + P[13] * q.X1 + P[14] * q.X2 + P[15];
    const double du = p0 / p2 - q.x, dv = p1 / p2 - q.y;
    return dz > 0.0 && du * du + dv * dv <= max_error2;
}

__device__ __forceinline__ AbsPt abs_point(const rb_abspose_args& a, int64_t j) {
    return {a.x[2 * j], a.x[2 * j + 1], a.X[3 * j], a.X[3 * j + 1], a.X[3 * j + 2]};
}

// grid (RB_ABS_ROUND / 128, splits, batch * RB_ABS_MAX_SOL): thread = hypothesis, blockIdx.z % RB_ABS_MAX_SOL = solution slot
__global__ void __launch_bounds__(AB_THREADS) abs_score_kernel(rb_abspose_args a, int per_split) {
    pdl_wait();
    __shared__ AbsPt tile[AB_TILE];
    const int b = blockIdx.z / AB_SOL, s = blockIdx.z % AB_SOL;
    const int hl = blockIdx.x * AB_THREADS + threadIdx.x;
    const int64_t slot = (int64_t)b * AB_ROUND + hl;
    const bool act = s < a.nsol[slot];
    if (!__syncthreads_or(act)) return;
    double P[16], R[9] = {}, t[3] = {};
    if (act) abs_load_model(a.models + (slot * AB_SOL + s) * 12, R, t);
    abs_projection(R, t, a.K + (int64_t)b * 9, P);
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const double e2 = a.max_error2;
    const int cnt = ransac_count<AB_THREADS>(tile, n, per_split, act, [&](int64_t j) { return abs_point(a, off + j); },
                                             [&](const AbsPt& q) { return abs_inlier(P, q, e2); });
    if (act) a.counts[(((int64_t)b * gridDim.y + blockIdx.y) * AB_SOL + s) * AB_ROUND + hl] = cnt;
}

// ---------------------------------------------------------------------------------------------------------------- select
__global__ void __launch_bounds__(128) abs_select_kernel(rb_abspose_args a, int splits) {
    pdl_wait();
    const int b = blockIdx.x * 128 + threadIdx.x;
    if (b >= a.batch) return;
    int* st = a.state + (int64_t)b * RB_ABS_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const int64_t slot0 = (int64_t)b * AB_ROUND;
    if (a.round == 0) {
        st[AS_ITER] = 0; st[AS_NITERS] = a.max_iters; st[AS_BEST] = 0; st[AS_HYP] = -1; st[AS_SOL] = -1;
        st[AS_RUN] = n >= 3; st[AS_N] = (int)n;
    }
    if (!st[AS_RUN]) return;
    int iter = st[AS_ITER], niters = st[AS_NITERS], best = st[AS_BEST];
    const int64_t per_split_stride = (int64_t)AB_SOL * AB_ROUND;
    for (int hl = 0; hl < AB_ROUND && iter < niters; ++hl, ++iter) {
        const int ns = a.nsol[slot0 + hl];
        for (int s = 0; s < ns; ++s) {
            int cnt = 0;
            const int32_t* c = a.counts + (int64_t)b * splits * per_split_stride + (int64_t)s * AB_ROUND + hl;
            for (int y = 0; y < splits; ++y) cnt += c[y * per_split_stride];
            if (cnt > max(best, 2)) {
                best = cnt;
                st[AS_HYP] = iter; st[AS_SOL] = s;
                for (int i = 0; i < 12; ++i) a.best[(int64_t)b * 12 + i] = a.models[((slot0 + hl) * AB_SOL + s) * 12 + i];
                niters = ransac_update_num_iters<3>(a.conf, (double)(n - cnt) / (double)n, niters);
            }
        }
    }
    // an item of exactly 3 points draws hypothesis 0 only
    const bool more = iter < niters && n > 3;
    st[AS_ITER] = iter; st[AS_NITERS] = niters; st[AS_BEST] = best; st[AS_RUN] = more;
    if (more) a.running[0] = 1;
}

// ---------------------------------------------------------------------------------------------------------------- refine
// this thread's share of the Gauss-Newton sums at (R, t) over the used points (mask set)
__device__ __forceinline__ void abs_gn_sums(const rb_abspose_args& a, int64_t off, int64_t n, const double (&R)[9], const double (&t)[3],
                                            const double* K, double (&v)[AB_SUMS]) {
#pragma unroll
    for (int k = 0; k < AB_SUMS; ++k) v[k] = 0.0;
    for (int64_t j = threadIdx.x; j < n; j += AB_REFINE_THREADS) {
        if (!a.mask[off + j]) continue;
        const AbsPt q = abs_point(a, off + j);
        double RX[3], Y[3], p[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            RX[i] = R[3 * i] * q.X0 + R[3 * i + 1] * q.X1 + R[3 * i + 2] * q.X2;
            Y[i] = RX[i] + t[i];
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) p[i] = K[3 * i] * Y[0] + K[3 * i + 1] * Y[1] + K[3 * i + 2] * Y[2];
        const double u = p[0] / p[2], w = p[1] / p[2], ru = u - q.x, rv = w - q.y;
        double J[2][6];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            J[0][3 + i] = (K[i] - u * K[6 + i]) / p[2];
            J[1][3 + i] = (K[3 + i] - w * K[6 + i]) / p[2];
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {                // d/d_omega of Exp(d_omega) R X is -[R X]x, so the row is (R X) x g
            const double* g = J[r] + 3;
            J[r][0] = RX[1] * g[2] - RX[2] * g[1];
            J[r][1] = RX[2] * g[0] - RX[0] * g[2];
            J[r][2] = RX[0] * g[1] - RX[1] * g[0];
        }
        int k = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int jj = i; jj < 6; ++jj) v[k++] += J[0][i] * J[0][jj] + J[1][i] * J[1][jj];
#pragma unroll
        for (int i = 0; i < 6; ++i) v[21 + i] += J[0][i] * ru + J[1][i] * rv;
        v[27] += ru * ru + rv * rv;
        v[28] += Y[2] > 0.0 ? 0.0 : 1.0;
    }
}

// (J^T J) d = -J^T r by Cholesky on the upper triangle of the sums; false on a pivot that is not > 0 and finite
__device__ __forceinline__ bool abs_solve6(const double* s, double (&d)[6]) {
    double L[6][6];
    int k = 0;
#pragma unroll
    for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = i; j < 6; ++j) L[j][i] = s[k++];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
        double dj = L[j][j];
#pragma unroll
        for (int q = 0; q < j; ++q) dj -= L[j][q] * L[j][q];
        if (!(dj > 0.0 && isfinite(dj))) return false;
        dj = sqrt(dj);
        L[j][j] = dj;
#pragma unroll
        for (int i = j + 1; i < 6; ++i) {
            double v = L[i][j];
#pragma unroll
            for (int q = 0; q < j; ++q) v -= L[i][q] * L[j][q];
            L[i][j] = v / dj;
        }
    }
    double y[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
        double v = -s[21 + i];
#pragma unroll
        for (int q = 0; q < i; ++q) v -= L[i][q] * y[q];
        y[i] = v / L[i][i];
    }
#pragma unroll
    for (int i = 5; i >= 0; --i) {
        double v = y[i];
#pragma unroll
        for (int q = i + 1; q < 6; ++q) v -= L[q][i] * d[q];
        d[i] = v / L[i][i];
    }
    return isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]) && isfinite(d[3]) && isfinite(d[4]) && isfinite(d[5]);
}

__global__ void __launch_bounds__(AB_REFINE_THREADS) abs_refine_kernel(rb_abspose_args a) {
    pdl_wait();
    __shared__ double red[AB_REFINE_THREADS / 32][AB_SUMS];
    __shared__ double tot[AB_SUMS], tot1[AB_SUMS];
    __shared__ int wcount[AB_REFINE_THREADS / 32];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const bool has = n >= 3 && a.state[(int64_t)b * RB_ABS_STATE + AS_BEST] >= 3;
    if (!has) {
        for (int64_t j = tid; j < n; j += AB_REFINE_THREADS) a.mask[off + j] = 0;
        if (tid < 9) a.R[(int64_t)b * 9 + tid] = 0.0;
        if (tid < 3) a.t[(int64_t)b * 3 + tid] = 0.0;
        if (tid == 0) { a.ok[b] = 0; a.num_inliers[b] = 0; }
        return;
    }
    const double* K = a.K + (int64_t)b * 9;
    double R[9], t[3], P[16];
    abs_load_model(a.best + (int64_t)b * 12, R, t);
    abs_projection(R, t, K, P);
    // the used points: the best model's inliers (each thread reads back only the entries it wrote)
    for (int64_t j = tid; j < n; j += AB_REFINE_THREADS) a.mask[off + j] = abs_inlier(P, abs_point(a, off + j), a.max_error2);
    double v[AB_SUMS];
    abs_gn_sums(a, off, n, R, t, K, v);
    cta_sum<AB_SUMS, AB_REFINE_THREADS>(v, red, tot);
#pragma unroll 1
    for (int it = 0; it < RB_ABS_GN_ITERS; ++it) {
        double d[6];
        if (!abs_solve6(tot, d)) break;
        const double w[3] = {d[0], d[1], d[2]};
        double E[3][3], R1[9], t1[3];
        so3_exp(w, E);
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) R1[3 * i + j] = E[i][0] * R[j] + E[i][1] * R[3 + j] + E[i][2] * R[6 + j];
#pragma unroll
        for (int i = 0; i < 3; ++i) t1[i] = t[i] + d[3 + i];
        abs_gn_sums(a, off, n, R1, t1, K, v);
        cta_sum<AB_SUMS, AB_REFINE_THREADS>(v, red, tot1);
        if (!(tot1[27] < tot[27] && tot1[28] == 0.0)) break;
#pragma unroll
        for (int i = 0; i < 9; ++i) R[i] = R1[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) t[i] = t1[i];
        __syncthreads();
        if (tid < AB_SUMS) tot[tid] = tot1[tid];
        __syncthreads();
    }
    // rule 4 once more against the refined pose
    abs_projection(R, t, K, P);
    int cnt = 0;
    for (int64_t j = tid; j < n; j += AB_REFINE_THREADS) {
        const bool in = abs_inlier(P, abs_point(a, off + j), a.max_error2);
        a.mask[off + j] = in;
        cnt += in;
    }
#pragma unroll
    for (int dd = 16; dd; dd >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, dd);
    if ((tid & 31) == 0) wcount[tid >> 5] = cnt;
    __syncthreads();
    if (tid == 0) {
#pragma unroll
        for (int i = 0; i < 9; ++i) a.R[(int64_t)b * 9 + i] = R[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) a.t[(int64_t)b * 3 + i] = t[i];
        int64_t total = 0;
        for (int w = 0; w < AB_REFINE_THREADS / 32; ++w) total += wcount[w];
        a.ok[b] = 1;
        a.num_inliers[b] = total;
    }
}

static int abs_check(const rb_abspose_args* a, const char* what) {
    if (ransac_check(a, what, RB_ABS_MAX_BATCH, AB_ROUND)) return 1;
    RB_REQUIRE(a->x && a->X && a->K, "%s: null argument", what);
    RB_REQUIRE(a->max_error2 > 0.0, "%s: bad max_error2 %g", what, a->max_error2);
    return 0;
}

static int abs_splits(int64_t max_n) { return ransac_splits(max_n, RB_ABS_SLICE, RB_ABS_MAX_SPLITS); }

// ---------------------------------------------------------------------------------------------------------------- register
constexpr int RG_THREADS = 128;
constexpr int RG_WARPS = RG_THREADS / 32;

__global__ void __launch_bounds__(RG_THREADS) reg_setup_kernel(rb_register_args a) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * RG_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * RG_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) {
        const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
        const bool ok = a.track_ok[k] != 0;
        bool bad = false;
        for (int64_t e = lane; e < L; e += 32) {
            const int64_t g = base + e;
            const int i = a.elements[2 * g], id = a.elements[2 * g + 1];
            const bool bad_e = i < 0 || i >= a.num_images || id < 0 || id >= a.kp_offsets[i + 1] - a.kp_offsets[i];
            bad |= bad_e;
            a.track[g] = (int32_t)k;
            const int img = ok && !bad_e ? i : a.num_images;
            a.keys[g] = ((unsigned long long)(uint32_t)img << 32) | (uint32_t)g;
        }
        if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr((unsigned long long*)a.info, (unsigned long long)RB_REG_BAD_ID);
    }
}

// image_offsets[i] = the first sorted key of image >= i; elem = the element ids in sorted order
__global__ void __launch_bounds__(256) reg_offsets_kernel(rb_register_args a, const uint64_t* __restrict__ sorted) {
    pdl_wait();
    const int64_t t0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, step = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i <= a.num_images; i += step) {
        int64_t lo = 0, hi = a.num_elements;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)(sorted[mid] >> 32) < i) lo = mid + 1;
            else hi = mid;
        }
        a.image_offsets[i] = lo;
    }
    for (int64_t q = t0; q < a.num_elements; q += step) a.elem[q] = (int32_t)(uint32_t)sorted[q];
}

// grid (ceil, num_list): item m of the chunk copies image images[m]'s correspondences to out_offsets[m]
__global__ void __launch_bounds__(256) reg_gather_kernel(rb_register_args a) {
    pdl_wait();
    const int m = blockIdx.y, i = a.images[m];
    const int64_t src = a.image_offsets[i], cnt = a.image_offsets[i + 1] - src, dst = a.out_offsets[m];
    for (int64_t q = (int64_t)blockIdx.x * 256 + threadIdx.x; q < cnt; q += (int64_t)gridDim.x * 256) {
        const int64_t e = a.elem[src + q];
        const int64_t r = a.kp_offsets[i] + a.elements[2 * e + 1];
        const int64_t k = a.track[e];
        a.x[2 * (dst + q)] = (double)a.keypoints[2 * r];
        a.x[2 * (dst + q) + 1] = (double)a.keypoints[2 * r + 1];
#pragma unroll
        for (int c = 0; c < 3; ++c) a.X[3 * (dst + q) + c] = a.points[3 * k + c];
    }
}

static int reg_check(const rb_register_args* a, const char* what) {
    RB_REQUIRE(a && a->track_offsets && a->elements && a->kp_offsets && a->keypoints && a->track_ok && a->points && a->info && a->keys &&
               a->keys_alt && a->hist && a->image_offsets && a->elem && a->track, "%s: null argument", what);
    RB_REQUIRE(a->num_tracks > 0 && a->num_images > 0 && a->num_elements > 0 && a->num_elements < (1ll << 31) && a->num_rows > 0,
               "%s: bad sizes num_tracks=%d num_images=%d num_elements=%lld num_rows=%lld", what, a->num_tracks, a->num_images,
               (long long)a->num_elements, (long long)a->num_rows);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_abspose_hypotheses(const rb_abspose_args* a, void* stream) {
    if (abs_check(a, "abspose_hypotheses")) return 1;
    RB_REQUIRE(a->sample && a->models && a->nsol && a->running, "abspose_hypotheses: null output");
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(cudaMemsetAsync(a->running, 0, sizeof(int32_t), st) == cudaSuccess, "abspose_hypotheses: memset failed");
    launch_pdl(abs_hyp_kernel, dim3(AB_ROUND / AB_HYP_THREADS, a->batch), dim3(AB_HYP_THREADS), 0, st, *a);
    return check_launch("abspose_hypotheses");
}

extern "C" int romab200_abspose_score(const rb_abspose_args* a, void* stream) {
    if (abs_check(a, "abspose_score")) return 1;
    RB_REQUIRE(a->models && a->nsol && a->counts, "abspose_score: null argument");
    const int splits = abs_splits(a->max_n);
    const int per_split = (int)((a->max_n + splits - 1) / splits);
    launch_pdl(abs_score_kernel, dim3(AB_ROUND / AB_THREADS, splits, a->batch * AB_SOL), dim3(AB_THREADS), 0, (cudaStream_t)stream, *a,
               max(per_split, 1));
    return check_launch("abspose_score");
}

extern "C" int romab200_abspose_select(const rb_abspose_args* a, void* stream) {
    if (abs_check(a, "abspose_select")) return 1;
    RB_REQUIRE(a->models && a->nsol && a->counts && a->best && a->running, "abspose_select: null argument");
    launch_pdl(abs_select_kernel, dim3((a->batch + 127) / 128), dim3(128), 0, (cudaStream_t)stream, *a, abs_splits(a->max_n));
    return check_launch("abspose_select");
}

extern "C" int romab200_abspose_refine(const rb_abspose_args* a, void* stream) {
    RB_REQUIRE(a && a->offsets && a->x && a->X && a->K && a->state && a->best && a->R && a->t && a->ok && a->num_inliers && a->mask,
               "abspose_refine: null argument");
    RB_REQUIRE(a->batch > 0 && a->batch <= RB_ABS_MAX_BATCH, "abspose_refine: batch %d outside [1, %d]", a->batch, RB_ABS_MAX_BATCH);
    launch_pdl(abs_refine_kernel, dim3(a->batch), dim3(AB_REFINE_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("abspose_refine");
}

extern "C" int romab200_register_setup(const rb_register_args* a, void* stream) {
    if (reg_check(a, "register_setup")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(a->info, 0, sizeof(int64_t), st) != cudaSuccess) return check_launch("register_setup(info)");
    launch_pdl(reg_setup_kernel, dim3(grid1d(a->num_tracks, RG_WARPS, 64 * 1024)), dim3(RG_THREADS), 0, st, *a);
    if (check_launch("register_setup(check)")) return 1;
    const int bits = 32 - __builtin_clz((unsigned)a->num_images);              // images lie in [0, num_images]
    uint64_t* sorted = nullptr;
    if (radix_sort_hi32<RB_TRACKS_TILE>(a->keys, a->keys_alt, a->hist, a->num_elements, bits, st, "register_setup(radix)", &sorted)) return 1;
    launch_pdl(reg_offsets_kernel, dim3(grid1d(a->num_elements, 256, 16 * 1024)), dim3(256), 0, st, *a, (const uint64_t*)sorted);
    return check_launch("register_setup(offsets)");
}

extern "C" int romab200_register_gather(const rb_register_args* a, void* stream) {
    if (reg_check(a, "register_gather")) return 1;
    RB_REQUIRE(a->images && a->out_offsets && a->x && a->X, "register_gather: null argument");
    RB_REQUIRE(a->num_list > 0 && a->num_list <= RB_ABS_MAX_BATCH, "register_gather: num_list %d outside [1, %d]", a->num_list,
               RB_ABS_MAX_BATCH);
    launch_pdl(reg_gather_kernel, dim3(64, a->num_list), dim3(256), 0, (cudaStream_t)stream, *a);
    return check_launch("register_gather");
}
