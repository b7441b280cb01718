// Fundamental matrix on the device: cv2.findFundamentalMat(kptsA, kptsB, ransacReprojThreshold, cv2.USAC_MAGSAC, confidence, maxIters)
// as the reference's usage example calls it (README.md:62-78, demo/demo_fundamental.py), for a batch of pairs.  The estimator is
// MAGSAC++ (Barath, Noskova, Ivashechkin, Matas, CVPR 2020) over seven-point samples, stated in include/romab200.h and DESIGN.md:
//   hypotheses  round 0 normalises each pair (one CTA per pair, fixed-order sums); then one thread per hypothesis: draw 7 indices,
//               the 7x9 system by Gauss-Jordan in registers, the real roots of the cubic by bisection, the oriented epipolar
//               constraint, up to 3 de-normalised models.  Every operation is rounded separately, so oracle/fundamental_ransac.py
//               reproduces the models bit for bit;
//   score       thread = (hypothesis, model slot), the model in registers, the pair's points streamed through shared memory in
//               slices of RB_FUND_SLICE points on grid.y: per slice a sequential float64 MAGSAC++ loss and an integer inlier count;
//   select      one warp per pair replays the sequential loop 32 hypotheses at a time: an exclusive prefix minimum of the
//               hypotheses' losses marks the records, and only those are walked in order;
//   refine      one CTA per pair, sigma-consensus++: MAGSAC++ weights, the weighted normalised eight-point fit (cyclic Jacobi on the
//               9x9 sums, one warp), rank 2 by a 3x3 SVD, kept while the loss decreases; then the Sampson mask.
// Everything is deterministic: no atomics, no order-dependent sums.
#include "geometry.cuh"

namespace rb {

constexpr int FM_ROUND = RB_FUND_ROUND;
constexpr int FM_MODELS = RB_FUND_MODELS;
constexpr int FM_SLOTS = FM_ROUND * FM_MODELS;   // (hypothesis, model) slots of a round
constexpr int FM_THREADS = 128;                   // hypotheses per CTA of the solver, slots per CTA of the score
constexpr int FM_TILE = 256;                      // score: points per shared-memory tile (8 KB)
constexpr int FM_NORM_THREADS = 256;
constexpr int FM_REFINE_THREADS = 256;
constexpr int FM_NSUMS = 45;                      // refine: distinct entries of the symmetric 9x9 sum
enum { FS_ITER = 0, FS_NITERS, FS_HYP, FS_SLOT, FS_RUN, FS_N };
constexpr unsigned FM_FULL = 0xffffffffu;

// ---------------------------------------------------------------------------------------------------------------- normalise
// grid (batch): centroid and mean distance over the rows whose four coordinates are finite, scale = sqrt(2) / mean distance
__global__ void __launch_bounds__(FM_NORM_THREADS) fund_norm_kernel(rb_fund_args a) {
    rb::pdl_wait();
    __shared__ double red[FM_NORM_THREADS / 32][5];
    __shared__ double tot[5];
    const int b = blockIdx.x, tid = threadIdx.x;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const double2* X0 = reinterpret_cast<const double2*>(a.x0) + off;
    const double2* X1 = reinterpret_cast<const double2*>(a.x1) + off;
    auto finite = [](double2 p, double2 q) { return isfinite(p.x) && isfinite(p.y) && isfinite(q.x) && isfinite(q.y); };
    double s[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (int64_t i = tid; i < n; i += FM_NORM_THREADS) {
        const double2 p = X0[i], q = X1[i];
        if (!finite(p, q)) continue;
        s[0] = __dadd_rn(s[0], p.x); s[1] = __dadd_rn(s[1], p.y); s[2] = __dadd_rn(s[2], q.x); s[3] = __dadd_rn(s[3], q.y);
        s[4] = __dadd_rn(s[4], 1.0);
    }
    cta_sum<5, FM_NORM_THREADS>(s, red, tot);
    const double cnt = tot[4];
    const double c0x = __ddiv_rn(tot[0], cnt), c0y = __ddiv_rn(tot[1], cnt), c1x = __ddiv_rn(tot[2], cnt), c1y = __ddiv_rn(tot[3], cnt);
    double d[2] = {0.0, 0.0};
    for (int64_t i = tid; i < n; i += FM_NORM_THREADS) {
        const double2 p = X0[i], q = X1[i];
        if (!finite(p, q)) continue;
        const double px = __dsub_rn(p.x, c0x), py = __dsub_rn(p.y, c0y), qx = __dsub_rn(q.x, c1x), qy = __dsub_rn(q.y, c1y);
        d[0] = __dadd_rn(d[0], __dsqrt_rn(__dadd_rn(__dmul_rn(px, px), __dmul_rn(py, py))));
        d[1] = __dadd_rn(d[1], __dsqrt_rn(__dadd_rn(__dmul_rn(qx, qx), __dmul_rn(qy, qy))));
    }
    cta_sum<2, FM_NORM_THREADS>(d, red, tot);
    constexpr double SQRT2 = 1.4142135623730951;
    const double s0 = __ddiv_rn(SQRT2, __ddiv_rn(tot[0], cnt)), s1 = __ddiv_rn(SQRT2, __ddiv_rn(tot[1], cnt));
    if (tid == 0) {
        double* nr = a.norm + (int64_t)b * 6;
        nr[0] = c0x; nr[1] = c0y; nr[2] = s0; nr[3] = c1x; nr[4] = c1y; nr[5] = s1;
    }
    double4* xn = reinterpret_cast<double4*>(a.xn) + off;
    for (int64_t i = tid; i < n; i += FM_NORM_THREADS) {
        const double2 p = X0[i], q = X1[i];
        xn[i] = make_double4(__dmul_rn(__dsub_rn(p.x, c0x), s0), __dmul_rn(__dsub_rn(p.y, c0y), s0), __dmul_rn(__dsub_rn(q.x, c1x), s1),
                             __dmul_rn(__dsub_rn(q.y, c1y), s1));
    }
}

// ---------------------------------------------------------------------------------------------------------------- solver
// cofactors of a row-major 3x3 matrix
__device__ __forceinline__ void cofactors(const double (&A)[9], double (&c)[9]) {
    c[0] = __dsub_rn(__dmul_rn(A[4], A[8]), __dmul_rn(A[5], A[7]));
    c[1] = __dsub_rn(__dmul_rn(A[5], A[6]), __dmul_rn(A[3], A[8]));
    c[2] = __dsub_rn(__dmul_rn(A[3], A[7]), __dmul_rn(A[4], A[6]));
    c[3] = __dsub_rn(__dmul_rn(A[2], A[7]), __dmul_rn(A[1], A[8]));
    c[4] = __dsub_rn(__dmul_rn(A[0], A[8]), __dmul_rn(A[2], A[6]));
    c[5] = __dsub_rn(__dmul_rn(A[1], A[6]), __dmul_rn(A[0], A[7]));
    c[6] = __dsub_rn(__dmul_rn(A[1], A[5]), __dmul_rn(A[2], A[4]));
    c[7] = __dsub_rn(__dmul_rn(A[2], A[3]), __dmul_rn(A[0], A[5]));
    c[8] = __dsub_rn(__dmul_rn(A[0], A[4]), __dmul_rn(A[1], A[3]));
}

// sum_i B[i] c[i], in index order
__device__ __forceinline__ double dot9(const double (&B)[9], const double (&c)[9]) {
    double s = __dmul_rn(B[0], c[0]);
#pragma unroll
    for (int i = 1; i < 9; ++i) s = __dadd_rn(s, __dmul_rn(B[i], c[i]));
    return s;
}

__device__ __forceinline__ double cubic(double c3, double c2, double c1, double c0, double x) {
    return __dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dadd_rn(__dmul_rn(c3, x), c2), x), c1), x), c0);
}

// the root of the cubic in [lo, hi], where its sign changes: bisection until lo and hi are adjacent doubles (at most 128 halvings)
__device__ __forceinline__ double bisect(double c3, double c2, double c1, double c0, double lo, double hi, bool neg_lo) {
#pragma unroll 1
    for (int it = 0; it < 128; ++it) {
        const double mid = __dmul_rn(__dadd_rn(lo, hi), 0.5);
        if (!(mid > lo && mid < hi)) break;
        if ((cubic(c3, c2, c1, c0, mid) < 0.0) == neg_lo) lo = mid;
        else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ void cross3(double a0, double a1, double a2, double b0, double b1, double b2, double (&c)[3]) {
    c[0] = __dsub_rn(__dmul_rn(a1, b2), __dmul_rn(a2, b1));
    c[1] = __dsub_rn(__dmul_rn(a2, b0), __dmul_rn(a0, b2));
    c[2] = __dsub_rn(__dmul_rn(a0, b1), __dmul_rn(a1, b0));
}

__device__ __forceinline__ double norm2_3(const double (&c)[3]) {
    return __dadd_rn(__dadd_rn(__dmul_rn(c[0], c[0]), __dmul_rn(c[1], c[1])), __dmul_rn(c[2], c[2]));
}

// The oriented epipolar constraint on the 7 normalised points p[i] = (x, y, x', y'): (e' x x'_i) . (F x_i) has the same strict sign
// for all of them, e' the largest (in squared norm, first on ties) of the cross products c0 x c2, c1 x c2, c0 x c1 of F's columns.
__device__ __forceinline__ bool oriented(const double (&F)[9], const double (&p)[7][4]) {
    double e[3], t[3];
    cross3(F[0], F[3], F[6], F[2], F[5], F[8], e);
    double ne = norm2_3(e);
    cross3(F[1], F[4], F[7], F[2], F[5], F[8], t);
    double nt = norm2_3(t);
    if (nt > ne) { e[0] = t[0]; e[1] = t[1]; e[2] = t[2]; ne = nt; }
    cross3(F[0], F[3], F[6], F[1], F[4], F[7], t);
    nt = norm2_3(t);
    if (nt > ne) { e[0] = t[0]; e[1] = t[1]; e[2] = t[2]; }
    int pos = 0, neg = 0;
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const double x = p[i][0], y = p[i][1], u = p[i][2], v = p[i][3];
        const double f0 = __dadd_rn(__dadd_rn(__dmul_rn(F[0], x), __dmul_rn(F[1], y)), F[2]);
        const double f1 = __dadd_rn(__dadd_rn(__dmul_rn(F[3], x), __dmul_rn(F[4], y)), F[5]);
        const double f2 = __dadd_rn(__dadd_rn(__dmul_rn(F[6], x), __dmul_rn(F[7], y)), F[8]);
        const double l0 = __dsub_rn(e[1], __dmul_rn(e[2], v)), l1 = __dsub_rn(__dmul_rn(e[2], u), e[0]);
        const double l2 = __dsub_rn(__dmul_rn(e[0], v), __dmul_rn(e[1], u));
        const double s = __dadd_rn(__dadd_rn(__dmul_rn(l0, f0), __dmul_rn(l1, f1)), __dmul_rn(l2, f2));
        pos += s > 0.0;
        neg += s < 0.0;
    }
    return pos == 7 || neg == 7;
}

// The seven-point solver on normalised points p[i] = (x, y, x', y'): rows (x'x, x'y, x', y'x, y'y, y', x, y, 1), Gauss-Jordan with
// partial pivoting (first largest |pivot|) to [I | N], the pencil F2 + l D with F1 = (-N[:, 0], 1, 0), F2 = (-N[:, 1], 0, 1),
// D = F1 - F2, and det(F2 + l D) = c3 l^3 + c2 l^2 + c1 l + c0.  Its real roots, ascending, give the models that pass `oriented`.
// Returns the number of models (0 when a pivot is not finite or below 1e-12 of the first, or the cubic has no finite bound).
__device__ __forceinline__ int seven_point(const double (&p)[7][4], double (&Fm)[FM_MODELS][9]) {
    double a[7][9];
#pragma unroll
    for (int i = 0; i < 7; ++i) {
        const double x = p[i][0], y = p[i][1], u = p[i][2], v = p[i][3];
        a[i][0] = __dmul_rn(u, x); a[i][1] = __dmul_rn(u, y); a[i][2] = u;
        a[i][3] = __dmul_rn(v, x); a[i][4] = __dmul_rn(v, y); a[i][5] = v;
        a[i][6] = x; a[i][7] = y; a[i][8] = 1.0;
    }
    double p0 = 0.0;
#pragma unroll
    for (int k = 0; k < 7; ++k) {
        int piv = k;
        double best = -1.0;
#pragma unroll
        for (int r = k; r < 7; ++r) {
            const double v = fabs(a[r][k]);
            if (v > best) { best = v; piv = r; }
        }
#pragma unroll
        for (int r = k + 1; r < 7; ++r)
            if (r == piv) {
#pragma unroll
                for (int c = k; c < 9; ++c) { const double t = a[k][c]; a[k][c] = a[r][c]; a[r][c] = t; }
            }
        const double pk = a[k][k];
        if (k == 0) p0 = fabs(pk);
        if (!(fabs(pk) > __dmul_rn(1e-12, p0)) || !isfinite(pk)) return 0;
#pragma unroll
        for (int c = k; c < 9; ++c) a[k][c] = __ddiv_rn(a[k][c], pk);
#pragma unroll
        for (int r = 0; r < 7; ++r) {
            if (r == k) continue;
            const double f = a[r][k];
#pragma unroll
            for (int c = k; c < 9; ++c) a[r][c] = __dsub_rn(a[r][c], __dmul_rn(f, a[k][c]));
        }
    }
    double F2[9], D[9], cf[9];
#pragma unroll
    for (int i = 0; i < 7; ++i) { F2[i] = -a[i][8]; D[i] = __dsub_rn(-a[i][7], F2[i]); }
    F2[7] = 0.0; F2[8] = 1.0; D[7] = 1.0; D[8] = -1.0;
    cofactors(F2, cf);
    const double c0 = __dadd_rn(__dadd_rn(__dmul_rn(F2[0], cf[0]), __dmul_rn(F2[1], cf[1])), __dmul_rn(F2[2], cf[2]));
    const double c1 = dot9(D, cf);
    cofactors(D, cf);
    const double c3 = __dadd_rn(__dadd_rn(__dmul_rn(D[0], cf[0]), __dmul_rn(D[1], cf[1])), __dmul_rn(D[2], cf[2]));
    const double c2 = dot9(F2, cf);
    const double B = __dadd_rn(1.0, __ddiv_rn(fmax(fmax(fabs(c2), fabs(c1)), fabs(c0)), fabs(c3)));
    if (!isfinite(B)) return 0;
    // the edges of the monotone pieces: -B, the critical points (when real, clamped to [-B, B]), B
    double edge[4] = {-B, B, B, B};
    int ne = 2;
    const double c33 = __dmul_rn(3.0, c3);
    const double disc = __dsub_rn(__dmul_rn(c2, c2), __dmul_rn(c33, c1));
    if (disc > 0.0) {
        const double q = __dsqrt_rn(disc);
        const double t0 = __ddiv_rn(__dsub_rn(-c2, q), c33), t1 = __ddiv_rn(__dadd_rn(-c2, q), c33);
        edge[1] = fmin(fmax(fmin(t0, t1), -B), B);
        edge[2] = fmin(fmax(fmax(t0, t1), -B), B);
        ne = 4;
    }
    int nm = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (k + 1 >= ne) break;
        const bool na = cubic(c3, c2, c1, c0, edge[k]) < 0.0, nb = cubic(c3, c2, c1, c0, edge[k + 1]) < 0.0;
        if (na == nb) continue;
        const double l = bisect(c3, c2, c1, c0, edge[k], edge[k + 1], na);
        double F[9];
        bool fin = true;
#pragma unroll
        for (int i = 0; i < 9; ++i) { F[i] = __dadd_rn(F2[i], __dmul_rn(l, D[i])); fin &= isfinite(F[i]); }
        if (!fin || !oriented(F, p)) continue;
#pragma unroll
        for (int m = 0; m < FM_MODELS; ++m)
            if (m == nm) {
#pragma unroll
                for (int i = 0; i < 9; ++i) Fm[m][i] = F[i];
            }
        ++nm;
    }
    return nm;
}

// T1^T Fn T0 with T = [[s, 0, -(s cx)], [0, s, -(s cy)], [0, 0, 1]] (nr = (cx0, cy0, s0, cx1, cy1, s1)), scaled to unit Frobenius norm
// (the squares summed in index order).  Returns false when the result is not finite.
__device__ __forceinline__ bool fund_denormalise(const double* Fn, const double* nr, double (&F)[9]) {
    const double T0[9] = {nr[2], 0.0, -__dmul_rn(nr[2], nr[0]), 0.0, nr[2], -__dmul_rn(nr[2], nr[1]), 0.0, 0.0, 1.0};
    const double T1[9] = {nr[5], 0.0, -__dmul_rn(nr[5], nr[3]), 0.0, nr[5], -__dmul_rn(nr[5], nr[4]), 0.0, 0.0, 1.0};
    double A[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            A[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(Fn[3 * i], T0[j]), __dmul_rn(Fn[3 * i + 1], T0[3 + j])), __dmul_rn(Fn[3 * i + 2], T0[6 + j]));
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            F[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(T1[i], A[j]), __dmul_rn(T1[3 + i], A[3 + j])), __dmul_rn(T1[6 + i], A[6 + j]));
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < 9; ++i) s = __dadd_rn(s, __dmul_rn(F[i], F[i]));
    s = __dsqrt_rn(s);
    bool fin = true;
#pragma unroll
    for (int i = 0; i < 9; ++i) { F[i] = __ddiv_rn(F[i], s); fin &= isfinite(F[i]); }
    return fin;
}

__global__ void __launch_bounds__(FM_THREADS) fund_hypotheses_kernel(rb_fund_args a) {
    rb::pdl_wait();
    const int b = blockIdx.y, hl = blockIdx.x * FM_THREADS + threadIdx.x;
    const int64_t h = (int64_t)a.round * FM_ROUND + hl;
    const int64_t slot = (int64_t)b * FM_ROUND + hl;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    if (!(ransac_drawn<7>(n, h, a.max_iters) && (a.round == 0 || a.state[b * RB_FUND_STATE + FS_RUN] != 0))) {
        a.nmod[slot] = 0;
        return;
    }
    int id[7] = {0, 1, 2, 3, 4, 5, 6};
    if (n > 7) ransac_draw(id, n, a.seed, [&](uint32_t sub) { return make_uint4((uint32_t)h, sub, 0u, RB_FUND_CTR); });
    const double4* xn = reinterpret_cast<const double4*>(a.xn) + off;
    double p[7][4];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
        a.sample[slot * 7 + k] = id[k];
        const double4 q = xn[id[k]];
        p[k][0] = q.x; p[k][1] = q.y; p[k][2] = q.z; p[k][3] = q.w;
    }
    double Fm[FM_MODELS][9];
    const int nm = seven_point(p, Fm);
    const double* nr = a.norm + (int64_t)b * 6;
    int kept = 0;
#pragma unroll
    for (int m = 0; m < FM_MODELS; ++m) {
        if (m >= nm) break;
        double F[9];
        if (!fund_denormalise(Fm[m], nr, F)) continue;
#pragma unroll
        for (int i = 0; i < 9; ++i) a.F[(slot * FM_MODELS + kept) * 9 + i] = F[i];
        ++kept;
    }
    a.nmod[slot] = kept;
}

// ---------------------------------------------------------------------------------------------------------------- score
// squared Sampson distance of (x, y) <-> (u, v) under F, every operation rounded separately
__device__ __forceinline__ double sampson2(const double (&f)[9], double x, double y, double u, double v) {
    const double a0 = __dadd_rn(__dadd_rn(__dmul_rn(f[0], x), __dmul_rn(f[1], y)), f[2]);
    const double a1 = __dadd_rn(__dadd_rn(__dmul_rn(f[3], x), __dmul_rn(f[4], y)), f[5]);
    const double a2 = __dadd_rn(__dadd_rn(__dmul_rn(f[6], x), __dmul_rn(f[7], y)), f[8]);
    const double b0 = __dadd_rn(__dadd_rn(__dmul_rn(f[0], u), __dmul_rn(f[3], v)), f[6]);
    const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(f[1], u), __dmul_rn(f[4], v)), f[7]);
    const double e = __dadd_rn(__dadd_rn(__dmul_rn(u, a0), __dmul_rn(v, a1)), a2);
    const double den = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, a0), __dmul_rn(a1, a1)), __dmul_rn(b0, b0)), __dmul_rn(b1, b1));
    return __ddiv_rn(__dmul_rn(e, e), den);
}

// table t[0..RB_FUND_TABLE] interpolated linearly at p in [0, RB_FUND_TABLE]
__device__ __forceinline__ double table_at(const double* t, double p) {
    const int i = min((int)p, RB_FUND_TABLE - 1);
    const double fr = __dsub_rn(p, (double)i);
    return __dadd_rn(t[i], __dmul_rn(fr, __dsub_rn(t[i + 1], t[i])));
}

struct FundThresh {
    double t2, l2, sc;         // thresh^2 (inliers), k^2 thresh^2 (end of the loss), RB_FUND_TABLE / (k^2 thresh^2)
};

__device__ __forceinline__ FundThresh fund_thresh(double th) {
    const double t2 = __dmul_rn(th, th), l2 = __dmul_rn(RB_FUND_K2, t2);
    return {t2, l2, __ddiv_rn((double)RB_FUND_TABLE, l2)};
}

// grid (FM_SLOTS / 128, splits, batch): thread = slot (hypothesis, model)
__global__ void __launch_bounds__(FM_THREADS) fund_score_kernel(rb_fund_args a, int splits) {
    rb::pdl_wait();
    __shared__ double tab[RB_FUND_TABLE + 1];
    __shared__ __align__(16) double4 tile[FM_TILE];
    const int b = blockIdx.z;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    if ((int64_t)blockIdx.y * RB_FUND_SLICE >= n) return;
    const int k = blockIdx.x * FM_THREADS + threadIdx.x;
    const int hl = k / FM_MODELS, m = k - hl * FM_MODELS;
    const int64_t slot = (int64_t)b * FM_ROUND + hl;
    const bool act = m < a.nmod[slot];
    if (!__syncthreads_or(act)) return;
    for (int i = threadIdx.x; i <= RB_FUND_TABLE; i += FM_THREADS) tab[i] = a.table[i];     // visible after ransac_scan's barrier
    double f[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) f[i] = act ? a.F[(slot * FM_MODELS + m) * 9 + i] : 0.0;
    const FundThresh th = fund_thresh(a.thresh);
    const double2* X0 = reinterpret_cast<const double2*>(a.x0) + off;
    const double2* X1 = reinterpret_cast<const double2*>(a.x1) + off;
    auto load = [&](int64_t j) {
        const double2 p = X0[j], q = X1[j];
        return make_double4(p.x, p.y, q.x, q.y);
    };
    double loss = 0.0;
    int cnt = 0;
    ransac_scan<FM_THREADS>(tile, n, RB_FUND_SLICE, act, load, [&](const double4& p) {
        const double r2 = sampson2(f, p.x, p.y, p.z, p.w);
        cnt += r2 < th.t2;
        loss = __dadd_rn(loss, r2 < th.l2 ? table_at(tab, __dmul_rn(r2, th.sc)) : 1.0);
    });
    if (act) {
        const int64_t o = ((int64_t)b * splits + blockIdx.y) * FM_SLOTS + k;
        a.counts[o] = cnt;
        a.losses[o] = loss;
    }
}

// ---------------------------------------------------------------------------------------------------------------- select
// One warp per pair.  Within a step of 32 hypotheses the best loss before hypothesis i is min(best, losses of the earlier
// hypotheses of the step), so the records are where a hypothesis' smallest model loss is below min(best, exclusive prefix minimum);
// niters after a record depends only on that record's counts and the niters before it, so walking the records in order (each
// one's models in slot order) reproduces the sequential loop exactly.
__global__ void __launch_bounds__(128) fund_select_kernel(rb_fund_args a, int splits) {
    rb::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= a.batch) return;
    int* st = a.state + (int64_t)b * RB_FUND_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const int nsl = (int)((n + RB_FUND_SLICE - 1) / RB_FUND_SLICE);
    const int64_t slot0 = (int64_t)b * FM_ROUND;
    int iter, niters, hyp, hm, run;
    double best;
    if (a.round == 0) {
        iter = 0; niters = n == 7 ? 1 : a.max_iters; hyp = -1; hm = 0; run = n >= 7; best = INFINITY;
    } else {
        iter = st[FS_ITER]; niters = st[FS_NITERS]; hyp = st[FS_HYP]; hm = st[FS_SLOT]; run = st[FS_RUN]; best = a.best_loss[b];
    }
    const int hyp_in = hyp;
    if (run) {
        bool stop = false;
        for (int base = 0; base < FM_ROUND && !stop; base += 32) {
            const int g = a.round * FM_ROUND + base;          // iteration of lane 0; g == iter here
            if (g >= niters) { stop = true; break; }
            const int hl = base + lane;
            const int nm = a.nmod[slot0 + hl];
            double L[FM_MODELS];
            int C[FM_MODELS];
            double hmin = INFINITY;
#pragma unroll
            for (int m = 0; m < FM_MODELS; ++m) {
                L[m] = INFINITY; C[m] = 0;
                if (m < nm) {
                    const int64_t o = (int64_t)b * splits * FM_SLOTS + hl * FM_MODELS + m;
                    double s = 0.0;
                    int c = 0;
                    for (int y = 0; y < nsl; ++y) { s = __dadd_rn(s, a.losses[o + (int64_t)y * FM_SLOTS]); c += a.counts[o + (int64_t)y * FM_SLOTS]; }
                    L[m] = s; C[m] = c;
                    if (s < hmin) hmin = s;
                }
            }
            double incl = hmin;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const double v = __shfl_up_sync(FM_FULL, incl, d);
                if (lane >= d) incl = fmin(incl, v);
            }
            double excl = __shfl_up_sync(FM_FULL, incl, 1);
            if (lane == 0) excl = INFINITY;
            unsigned rec = __ballot_sync(FM_FULL, nm > 0 && hmin < fmin(best, excl));
            while (rec) {
                const int l = __ffs(rec) - 1;
                rec &= rec - 1;
                const int gi = g + l;
                if (gi >= niters) { iter = niters; stop = true; break; }
                const int nml = __shfl_sync(FM_FULL, nm, l);
#pragma unroll
                for (int m = 0; m < FM_MODELS; ++m) {
                    const double lm = __shfl_sync(FM_FULL, L[m], l);
                    const int cm = __shfl_sync(FM_FULL, C[m], l);
                    if (m < nml && lm < best) {
                        best = lm; hyp = gi; hm = m;
                        niters = ransac_update_num_iters<7>(a.conf, __ddiv_rn((double)(n - cm), (double)n), niters);
                    }
                }
                if (gi + 1 >= niters) { iter = gi + 1; stop = true; break; }
            }
            if (!stop) {
                if (g + 32 >= niters) { iter = niters; stop = true; }
                else iter = g + 32;
            }
        }
        run = !stop;
        if (hyp != hyp_in && lane < 9) a.best_F[(int64_t)b * 9 + lane] = a.F[((slot0 + (hyp - a.round * FM_ROUND)) * FM_MODELS + hm) * 9 + lane];
        if (run && lane == 0) a.running[0] = 1;
    }
    if (lane == 0) {
        st[FS_ITER] = iter; st[FS_NITERS] = niters; st[FS_HYP] = hyp; st[FS_SLOT] = hm; st[FS_RUN] = run; st[FS_N] = (int)n;
        a.best_loss[b] = best;
    }
}

// ---------------------------------------------------------------------------------------------------------------- refine
struct FundRefineSmem {
    double red[FM_REFINE_THREADS / 32][FM_NSUMS];
    double tot[FM_NSUMS];
    double tab[2][RB_FUND_TABLE + 1];
    double L[9][9], V[9][9];
    double F[9], Fr[9], nr[6];
    int flag;
};

// the MAGSAC++ loss of F over the pair, summed over the CTA in a fixed order (every thread receives it)
__device__ __forceinline__ double fund_loss(const double* F, const double2* X0, const double2* X1, int64_t n, const FundThresh& th,
                                            FundRefineSmem& sm) {
    double f[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) f[i] = F[i];
    double s[1] = {0.0};
    for (int64_t i = threadIdx.x; i < n; i += FM_REFINE_THREADS) {
        const double2 p = X0[i], q = X1[i];
        const double r2 = sampson2(f, p.x, p.y, q.x, q.y);
        s[0] += r2 < th.l2 ? table_at(sm.tab[0], __dmul_rn(r2, th.sc)) : 1.0;
    }
    cta_sum<1, FM_REFINE_THREADS>(s, sm.red, sm.tot);
    return sm.tot[0];
}

__global__ void __launch_bounds__(FM_REFINE_THREADS, 1) fund_refine_kernel(rb_fund_args a) {
    rb::pdl_wait();
    __shared__ FundRefineSmem sm;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int* st = a.state + (int64_t)b * RB_FUND_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const double2* X0 = reinterpret_cast<const double2*>(a.x0) + off;
    const double2* X1 = reinterpret_cast<const double2*>(a.x1) + off;
    const double4* xn = reinterpret_cast<const double4*>(a.xn) + off;
    uint8_t* mask = a.mask + off;
    double* outF = a.out_F + (int64_t)b * 9;
    if (!(n >= 7 && st[FS_HYP] >= 0)) {
        for (int64_t i = tid; i < n; i += FM_REFINE_THREADS) mask[i] = 0;
        if (tid < 9) outF[tid] = 0.0;
        if (tid == 0) a.ok[b] = 0;
        return;
    }
    for (int i = tid; i < 2 * (RB_FUND_TABLE + 1); i += FM_REFINE_THREADS) (&sm.tab[0][0])[i] = a.table[i];
    if (tid < 9) sm.F[tid] = a.best_F[(int64_t)b * 9 + tid];
    if (tid < 6) sm.nr[tid] = a.norm[(int64_t)b * 6 + tid];
    __syncthreads();
    const FundThresh th = fund_thresh(a.thresh);
    double cur = fund_loss(sm.F, X0, X1, n, th, sm);
    for (int it = 0; it < RB_FUND_REFINE_ITERS && n >= 8; ++it) {
        // sum of w a a^T over the points, a = (x'x, x'y, x', y'x, y'y, y', x, y, 1) of the normalised points, upper triangle by rows
        double acc[FM_NSUMS];
#pragma unroll
        for (int k = 0; k < FM_NSUMS; ++k) acc[k] = 0.0;
        double f[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) f[i] = sm.F[i];
        for (int64_t i = tid; i < n; i += FM_REFINE_THREADS) {
            const double2 p = X0[i], q = X1[i];
            const double r2 = sampson2(f, p.x, p.y, q.x, q.y);
            if (!(r2 < th.l2)) continue;
            const double w = table_at(sm.tab[1], __dmul_rn(r2, th.sc));
            if (!(w > 0.0)) continue;
            const double4 z = xn[i];
            const double r[9] = {z.z * z.x, z.z * z.y, z.z, z.w * z.x, z.w * z.y, z.w, z.x, z.y, 1.0};
            int k = 0;
#pragma unroll
            for (int u = 0; u < 9; ++u) {
                const double wu = w * r[u];
#pragma unroll
                for (int v = u; v < 9; ++v) acc[k++] += wu * r[v];
            }
        }
        cta_sum<FM_NSUMS, FM_REFINE_THREADS>(acc, sm.red, sm.tot);
        if (tid == 0) {
            int k = 0;
            for (int u = 0; u < 9; ++u)
                for (int v = u; v < 9; ++v, ++k) sm.L[u][v] = sm.L[v][u] = sm.tot[k];
        }
        __syncthreads();
        if (tid < 32) jacobi_eig_warp<9>(sm.L, sm.V, 15);
        __syncthreads();
        if (tid == 0) {
            int kmin = 0;
            for (int i = 1; i < 9; ++i)
                if (sm.L[i][i] < sm.L[kmin][kmin]) kmin = i;
            double Fn[9], u[3][3], v[3][3], s[2];
#pragma unroll
            for (int i = 0; i < 9; ++i) Fn[i] = sm.V[i][kmin];
            svd3(Fn, u, v, s);                       // rank 2: s0 u0 v0^T + s1 u1 v1^T
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) Fn[3 * i + j] = s[0] * u[0][i] * v[0][j] + s[1] * u[1][i] * v[1][j];
            double F[9];
            sm.flag = fund_denormalise(Fn, sm.nr, F);
#pragma unroll
            for (int i = 0; i < 9; ++i) sm.Fr[i] = F[i];
        }
        __syncthreads();
        if (!sm.flag) break;
        const double nl = fund_loss(sm.Fr, X0, X1, n, th, sm);
        if (!(nl < cur)) break;
        cur = nl;
        if (tid < 9) sm.F[tid] = sm.Fr[tid];
        __syncthreads();
    }
    double f[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) f[i] = sm.F[i];
    double fm = f[0];                                // the first entry of largest magnitude
#pragma unroll
    for (int i = 1; i < 9; ++i)
        if (fabs(f[i]) > fabs(fm)) fm = f[i];
    const double sg = fm < 0.0 ? -1.0 : 1.0;
    if (tid < 9) outF[tid] = sg * sm.F[tid];
    if (tid == 0) a.ok[b] = 1;
    for (int64_t i = tid; i < n; i += FM_REFINE_THREADS) {
        const double2 p = X0[i], q = X1[i];
        mask[i] = sampson2(f, p.x, p.y, q.x, q.y) < th.t2;
    }
}

static int fund_check(const rb_fund_args* a, const char* what) {
    if (ransac_check(a, what, 65535, FM_ROUND)) return 1;
    RB_REQUIRE(a->x0 && a->x1 && a->norm && a->xn && a->table, "%s: null argument", what);
    RB_REQUIRE(a->thresh > 0.0 && a->thresh < INFINITY, "%s: thresh %g is not positive and finite", what, a->thresh);
    return 0;
}

static int fund_splits(int64_t max_n) { return (int)((max_n + RB_FUND_SLICE - 1) / RB_FUND_SLICE) + (max_n == 0); }

}  // namespace rb

using namespace rb;

// cv2.findFundamentalMat(..., cv2.USAC_MAGSAC, ...) of README.md:62-78: normalisation (round 0) and the seven-point hypotheses
extern "C" int romab200_fund_hypotheses(const rb_fund_args* a, void* stream) {
    if (fund_check(a, "fund_hypotheses")) return 1;
    RB_REQUIRE(a->sample && a->nmod && a->F && a->running, "fund_hypotheses: null output");
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(cudaMemsetAsync(a->running, 0, sizeof(int32_t), st) == cudaSuccess, "fund_hypotheses: memset failed");
    if (a->round == 0) {
        rb::launch_pdl(fund_norm_kernel, dim3(a->batch), dim3(FM_NORM_THREADS), 0, st, *a);
        if (check_launch("fund_hypotheses(normalise)")) return 1;
    }
    rb::launch_pdl(fund_hypotheses_kernel, dim3(FM_ROUND / FM_THREADS, a->batch), dim3(FM_THREADS), 0, st, *a);
    return check_launch("fund_hypotheses");
}

// README.md:62-78: the MAGSAC++ loss and inlier count of every model of the round
extern "C" int romab200_fund_score(const rb_fund_args* a, void* stream) {
    if (fund_check(a, "fund_score")) return 1;
    RB_REQUIRE(a->nmod && a->F && a->counts && a->losses, "fund_score: null argument");
    const int splits = fund_splits(a->max_n);
    RB_REQUIRE(splits <= 65535, "fund_score: max_n %lld needs more than 65535 slices", (long long)a->max_n);
    rb::launch_pdl(fund_score_kernel, dim3(FM_SLOTS / FM_THREADS, splits, a->batch), dim3(FM_THREADS), 0, (cudaStream_t)stream, *a, splits);
    return check_launch("fund_score");
}

// README.md:62-78: the sequential best-model loop over the round
extern "C" int romab200_fund_select(const rb_fund_args* a, void* stream) {
    if (fund_check(a, "fund_select")) return 1;
    RB_REQUIRE(a->nmod && a->F && a->counts && a->losses && a->best_F && a->best_loss && a->running, "fund_select: null argument");
    rb::launch_pdl(fund_select_kernel, dim3((a->batch + 3) / 4), dim3(128), 0, (cudaStream_t)stream, *a, fund_splits(a->max_n));
    return check_launch("fund_select");
}

// README.md:62-78: sigma-consensus++ on the best model and the returned mask
extern "C" int romab200_fund_refine(const rb_fund_args* a, void* stream) {
    RB_REQUIRE(a && a->x0 && a->x1 && a->offsets && a->table && a->norm && a->xn && a->state && a->best_F && a->out_F && a->ok && a->mask,
               "fund_refine: null argument");
    RB_REQUIRE(a->batch > 0 && a->batch <= 65535, "fund_refine: batch %d outside [1, 65535]", a->batch);
    RB_REQUIRE(a->thresh > 0.0 && a->thresh < INFINITY, "fund_refine: thresh %g is not positive and finite", a->thresh);
    rb::launch_pdl(fund_refine_kernel, dim3(a->batch), dim3(FM_REFINE_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("fund_refine");
}
