// Homography on the device: cv2.findHomography(src, dst, cv2.RANSAC, ...) as the HPatches harness calls it
// (romatch/benchmarks/hpatches_sequences_homog_benchmark.py:80-86), for a batch of pairs.  The estimator is OpenCV 4.13's (classic
// RANSACPointSetRegistrator, HomographyEstimatorCallback, least-squares refinement); only the stream of minimal samples differs
// (Philox4x32-10, documented in include/romab200.h).
//   hypotheses  one thread per hypothesis: draw 4 indices, OpenCV's checkSubset (redraw on failure, at most 10 000 attempts),
//               normalised 8x9 system solved by Gauss-Jordan in registers (every operation rounded separately, so the numpy
//               restatement in oracle/homography_ransac.py reproduces it);
//   score       one thread per hypothesis, H rounded to float in registers, the pair's points streamed through shared memory;
//               grid.y cuts the points into slices whose integer partial counts `select` adds in a fixed order;
//   select      one warp per pair replays OpenCV's sequential loop 32 hypotheses at a time: an exclusive prefix maximum of the
//               counts marks the records (count > max(best, 3)), and only the records and "not found" hypotheses are walked in order;
//   refine      one CTA per pair: inlier mask, normalised DLT over the inliers (cyclic Jacobi on the 9x9 L^T L, one warp), then at most 10
//               Levenberg-Marquardt steps; every sum over the points is a per-thread partial followed by a fixed-order tree.  The
//               returned mask is the inlier set of the refined model, as OpenCV 4.13 returns it.
// Everything is deterministic: no atomics, no order-dependent sums.
#include "geometry.cuh"

namespace rb {

constexpr int HG_ROUND = RB_HOMOG_ROUND;
constexpr int HG_THREADS = 128;                   // hypotheses per CTA of the solver and of the score
constexpr int HG_TILE = 512;                      // score: points per shared-memory tile (8 KB)
constexpr int HG_REFINE_THREADS = 256;
constexpr int HG_NRED = 31;                       // refine: partial sums per thread (30 + a maximum)
enum { HS_ITER = 0, HS_NITERS, HS_BEST, HS_HYP, HS_RUN, HS_N, HS_NOT_FOUND };
constexpr double HG_DBL_EPS = 2.220446049250313080847e-16;
constexpr double HG_FLT_EPS = 1.1920928955078125e-07;
constexpr unsigned HG_FULL = 0xffffffffu;

// ---------------------------------------------------------------------------------------------------------------- checks
// OpenCV's haveCollinearPoints(ms, 4): the last point against every pair of earlier ones.  The differences are float
// subtractions (Point2f members), the test is in double.
__device__ __forceinline__ bool collinear_last(const float (&x)[4], const float (&y)[4]) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        const double dx1 = (double)__fsub_rn(x[j], x[3]), dy1 = (double)__fsub_rn(y[j], y[3]);
#pragma unroll
        for (int k = 0; k < j; ++k) {
            const double dx2 = (double)__fsub_rn(x[k], x[3]), dy2 = (double)__fsub_rn(y[k], y[3]);
            const double lhs = fabs(__dsub_rn(__dmul_rn(dx2, dy1), __dmul_rn(dy2, dx1)));
            const double rhs = __dmul_rn(HG_FLT_EPS, __dadd_rn(__dadd_rn(__dadd_rn(fabs(dx1), fabs(dy1)), fabs(dx2)), fabs(dy2)));
            if (lhs <= rhs) return true;
        }
    }
    return false;
}

// determinant of [[x0 y0 1] [x1 y1 1] [x2 y2 1]] in cv::Matx33d's cofactor order
__device__ __forceinline__ double det3(double x0, double y0, double x1, double y1, double x2, double y2) {
    const double c0 = __dsub_rn(__dmul_rn(y1, 1.0), __dmul_rn(y2, 1.0));
    const double c1 = __dsub_rn(__dmul_rn(x1, 1.0), __dmul_rn(x2, 1.0));
    const double c2 = __dsub_rn(__dmul_rn(x1, y2), __dmul_rn(x2, y1));
    return __dadd_rn(__dsub_rn(__dmul_rn(x0, c0), __dmul_rn(y0, c1)), __dmul_rn(1.0, c2));
}

// OpenCV's HomographyEstimatorCallback::checkSubset for 4 correspondences
__device__ __forceinline__ bool check_subset(const float (&sx)[4], const float (&sy)[4], const float (&dx)[4], const float (&dy)[4]) {
    if (collinear_last(sx, sy) || collinear_last(dx, dy)) return false;
    constexpr int tt[4][3] = {{0, 1, 2}, {1, 2, 3}, {0, 2, 3}, {1, 3, 0}};
    int negative = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int p = tt[i][0], q = tt[i][1], r = tt[i][2];
        const double dA = det3(sx[p], sy[p], sx[q], sy[q], sx[r], sy[r]);
        const double dB = det3(dx[p], dy[p], dx[q], dy[q], dx[r], dy[r]);
        negative += __dmul_rn(dA, dB) < 0.0;
    }
    return negative == 0 || negative == 4;
}

// ---------------------------------------------------------------------------------------------------------------- solver
// H = inv(Tm) H0 TM with OpenCV's normalisations, then multiplied by 1 / H[2][2]
__device__ __forceinline__ void denormalise(const double (&h0)[9], double cmx, double cmy, double smx, double smy, double cMx, double cMy,
                                            double sMx, double sMy, double (&H)[9]) {
    const double inv[9] = {__ddiv_rn(1.0, smx), 0.0, cmx, 0.0, __ddiv_rn(1.0, smy), cmy, 0.0, 0.0, 1.0};
    const double nrm[9] = {sMx, 0.0, -__dmul_rn(cMx, sMx), 0.0, sMy, -__dmul_rn(cMy, sMy), 0.0, 0.0, 1.0};
    double t[9];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            t[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(inv[3 * i], h0[j]), __dmul_rn(inv[3 * i + 1], h0[3 + j])), __dmul_rn(inv[3 * i + 2], h0[6 + j]));
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j)
            H[3 * i + j] = __dadd_rn(__dadd_rn(__dmul_rn(t[3 * i], nrm[j]), __dmul_rn(t[3 * i + 1], nrm[3 + j])), __dmul_rn(t[3 * i + 2], nrm[6 + j]));
    const double s = __ddiv_rn(1.0, H[8]);
#pragma unroll
    for (int i = 0; i < 9; ++i) H[i] = __dmul_rn(H[i], s);
}

// the minimal solver: 4 correspondences (src -> dst), OpenCV's normalisation, null vector of the 8x9 system by Gauss-Jordan with
// partial pivoting (first largest |pivot|).  Returns false when a normalisation sum is below DBL_EPSILON or a pivot is not finite or
// below 1e-12 of the first.
__device__ __forceinline__ bool solve_four(const float (&sx)[4], const float (&sy)[4], const float (&dx)[4], const float (&dy)[4], double (&H)[9]) {
    double cmx = 0.0, cmy = 0.0, cMx = 0.0, cMy = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        cmx = __dadd_rn(cmx, (double)dx[i]); cmy = __dadd_rn(cmy, (double)dy[i]);
        cMx = __dadd_rn(cMx, (double)sx[i]); cMy = __dadd_rn(cMy, (double)sy[i]);
    }
    cmx = __ddiv_rn(cmx, 4.0); cmy = __ddiv_rn(cmy, 4.0); cMx = __ddiv_rn(cMx, 4.0); cMy = __ddiv_rn(cMy, 4.0);
    double smx = 0.0, smy = 0.0, sMx = 0.0, sMy = 0.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        smx = __dadd_rn(smx, fabs(__dsub_rn((double)dx[i], cmx))); smy = __dadd_rn(smy, fabs(__dsub_rn((double)dy[i], cmy)));
        sMx = __dadd_rn(sMx, fabs(__dsub_rn((double)sx[i], cMx))); sMy = __dadd_rn(sMy, fabs(__dsub_rn((double)sy[i], cMy)));
    }
    if (!(fabs(smx) >= HG_DBL_EPS && fabs(smy) >= HG_DBL_EPS && fabs(sMx) >= HG_DBL_EPS && fabs(sMy) >= HG_DBL_EPS)) return false;
    smx = __ddiv_rn(4.0, smx); smy = __ddiv_rn(4.0, smy); sMx = __ddiv_rn(4.0, sMx); sMy = __ddiv_rn(4.0, sMy);
    // rows 2i, 2i + 1: Lx = (X, Y, 1, 0, 0, 0, -x X, -x Y, -x), Ly = (0, 0, 0, X, Y, 1, -y X, -y Y, -y)
    double a[8][9];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const double x = __dmul_rn(__dsub_rn((double)dx[i], cmx), smx), y = __dmul_rn(__dsub_rn((double)dy[i], cmy), smy);
        const double X = __dmul_rn(__dsub_rn((double)sx[i], cMx), sMx), Y = __dmul_rn(__dsub_rn((double)sy[i], cMy), sMy);
        const double lx[9] = {X, Y, 1.0, 0.0, 0.0, 0.0, -__dmul_rn(x, X), -__dmul_rn(x, Y), -x};
        const double ly[9] = {0.0, 0.0, 0.0, X, Y, 1.0, -__dmul_rn(y, X), -__dmul_rn(y, Y), -y};
#pragma unroll
        for (int c = 0; c < 9; ++c) { a[2 * i][c] = lx[c]; a[2 * i + 1][c] = ly[c]; }
    }
    double p0 = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int piv = k;
        double best = -1.0;
#pragma unroll
        for (int r = k; r < 8; ++r) {
            const double v = fabs(a[r][k]);
            if (v > best) { best = v; piv = r; }
        }
#pragma unroll
        for (int r = k + 1; r < 8; ++r)
            if (r == piv) {
#pragma unroll
                for (int c = k; c < 9; ++c) { const double t = a[k][c]; a[k][c] = a[r][c]; a[r][c] = t; }
            }
        const double p = a[k][k];
        if (k == 0) p0 = fabs(p);
        if (!(fabs(p) > 1e-12 * p0) || !isfinite(p)) return false;
#pragma unroll
        for (int c = k; c < 9; ++c) a[k][c] = __ddiv_rn(a[k][c], p);
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            if (r == k) continue;
            const double f = a[r][k];
#pragma unroll
            for (int c = k; c < 9; ++c) a[r][c] = __dsub_rn(a[r][c], __dmul_rn(f, a[k][c]));
        }
    }
    double h0[9];
#pragma unroll
    for (int r = 0; r < 8; ++r) h0[r] = -a[r][8];
    h0[8] = 1.0;
    denormalise(h0, cmx, cmy, smx, smy, cMx, cMy, sMx, sMy, H);
    bool fin = true;
#pragma unroll
    for (int i = 0; i < 9; ++i) fin &= isfinite(H[i]);
    return fin;
}

__global__ void __launch_bounds__(HG_THREADS) homog_hypotheses_kernel(rb_homography_args a) {
    rb::pdl_wait();
    const int b = blockIdx.y, hl = blockIdx.x * HG_THREADS + threadIdx.x;
    const int64_t h = (int64_t)a.round * HG_ROUND + hl;
    const int64_t slot = (int64_t)b * HG_ROUND + hl;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    if (!(ransac_drawn<4>(n, h, a.max_iters) && (a.round == 0 || a.state[b * RB_HOMOG_STATE + HS_RUN] != 0))) {
        a.status[slot] = 0;
        return;
    }
    const float* S = a.src + 2 * off;
    const float* D = a.dst + 2 * off;
    int id[4] = {0, 1, 2, 3};
    float sx[4], sy[4], dx[4], dy[4];
    int att = 0;
    bool found = n == 4;
    if (n == 4) {
#pragma unroll
        for (int k = 0; k < 4; ++k) { sx[k] = S[2 * k]; sy[k] = S[2 * k + 1]; dx[k] = D[2 * k]; dy[k] = D[2 * k + 1]; }
    } else {
        for (; att < RB_HOMOG_MAX_ATTEMPTS; ++att) {
            ransac_draw(id, n, a.seed, [&](uint32_t sub) { return make_uint4((uint32_t)h, (uint32_t)b, (uint32_t)att, sub); });
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 s = reinterpret_cast<const float2*>(S)[id[k]], d = reinterpret_cast<const float2*>(D)[id[k]];
                sx[k] = s.x; sy[k] = s.y; dx[k] = d.x; dy[k] = d.y;
            }
            if (check_subset(sx, sy, dx, dy)) { found = true; break; }
        }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) a.sample[slot * 4 + k] = id[k];
    a.attempts[slot] = att;
    if (!found) {
        a.status[slot] = -1;
        return;
    }
    double H[9];
    const bool ok = solve_four(sx, sy, dx, dy, H);
#pragma unroll
    for (int i = 0; i < 9; ++i) a.H[slot * 9 + i] = ok ? H[i] : 0.0;
    a.status[slot] = ok ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------------- score
// OpenCV's HomographyEstimatorCallback::computeError in float32, every operation rounded separately (no contraction).  A NaN
// error (NaN point, 0/0) is never an inlier.
__device__ __forceinline__ bool homog_inlier(const float (&f)[8], float x, float y, float u, float v, float t) {
    const float ww = __fdiv_rn(1.0f, __fadd_rn(__fadd_rn(__fmul_rn(f[6], x), __fmul_rn(f[7], y)), 1.0f));
    const float ex = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(f[0], x), __fmul_rn(f[1], y)), f[2]), ww), u);
    const float ey = __fsub_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(f[3], x), __fmul_rn(f[4], y)), f[5]), ww), v);
    return __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)) <= t;
}

__device__ __forceinline__ float homog_thresh(double th) { return __double2float_rn(__dmul_rn(th, th)); }

// grid (RB_HOMOG_ROUND / 128, splits, batch): thread = hypothesis
__global__ void __launch_bounds__(HG_THREADS) homog_score_kernel(rb_homography_args a, int per_split) {
    rb::pdl_wait();
    __shared__ __align__(16) float4 tile[HG_TILE];
    const int b = blockIdx.z;
    const int hl = blockIdx.x * HG_THREADS + threadIdx.x;
    const int64_t slot = (int64_t)b * HG_ROUND + hl;
    const bool act = a.status[slot] == 1;
    if (!__syncthreads_or(act)) return;
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = act ? __double2float_rn(a.H[slot * 9 + i]) : 0.0f;
    const float t = homog_thresh(a.thresh);
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const float2* S = reinterpret_cast<const float2*>(a.src) + off;
    const float2* D = reinterpret_cast<const float2*>(a.dst) + off;
    auto load = [&](int64_t j) {
        const float2 s = S[j], d = D[j];
        return make_float4(s.x, s.y, d.x, d.y);
    };
    const int cnt = ransac_count<HG_THREADS>(tile, n, per_split, act, load, [&](const float4& p) { return homog_inlier(f, p.x, p.y, p.z, p.w, t); });
    if (act) a.counts[((int64_t)b * RB_HOMOG_MAX_SPLITS + blockIdx.y) * HG_ROUND + hl] = cnt;
}

// ---------------------------------------------------------------------------------------------------------------- select
// One warp per pair.  Within a step of 32 hypotheses the best count before hypothesis i is max(best, counts of the earlier
// hypotheses of the step), so the records are where count > max(best, 3, exclusive prefix maximum); niters after a record depends
// only on that record's count and the niters before it, so walking the records (and "not found" hypotheses) in order reproduces
// the sequential loop exactly.
__global__ void __launch_bounds__(128) homog_select_kernel(rb_homography_args a, int splits) {
    rb::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (b >= a.batch) return;
    int* st = a.state + (int64_t)b * RB_HOMOG_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const int64_t slot0 = (int64_t)b * HG_ROUND;
    double* bestH = a.best_H + (int64_t)b * 9;
    int iter, niters, best, hyp, run, nf = 0;
    if (a.round == 0) {
        iter = 0; niters = a.max_iters; best = 0; hyp = -1; run = n > 4;
        if (n == 4 && a.status[slot0] == 1) {        // OpenCV's count == modelPoints case: the 4 points, all inliers
            best = 4; hyp = 0;
            if (lane < 9) bestH[lane] = a.H[slot0 * 9 + lane];
        }
    } else {
        iter = st[HS_ITER]; niters = st[HS_NITERS]; best = st[HS_BEST]; hyp = st[HS_HYP]; run = st[HS_RUN]; nf = st[HS_NOT_FOUND];
    }
    __syncwarp();
    const int hyp_in = hyp;
    if (run) {
        bool stop = false;
        for (int base = 0; base < HG_ROUND && !stop; base += 32) {
            const int g = a.round * HG_ROUND + base;          // iteration of lane 0; g == iter here
            if (g >= niters) { stop = true; break; }
            const int hl = base + lane;
            const int s = a.status[slot0 + hl];
            int c = -1;
            if (s == 1) {
                c = 0;
                const int32_t* cp = a.counts + (int64_t)b * RB_HOMOG_MAX_SPLITS * HG_ROUND + hl;
                for (int y = 0; y < splits; ++y) c += cp[(int64_t)y * HG_ROUND];
            }
            int incl = c;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int v = __shfl_up_sync(HG_FULL, incl, d);
                if (lane >= d) incl = max(incl, v);
            }
            int excl = __shfl_up_sync(HG_FULL, incl, 1);
            if (lane == 0) excl = -1;
            const unsigned rec = __ballot_sync(HG_FULL, s == 1 && c > max(max(best, 3), excl));
            const unsigned notf = __ballot_sync(HG_FULL, s == -1);
            unsigned ev = rec | notf;
            while (ev) {
                const int l = __ffs(ev) - 1;
                ev &= ev - 1;
                const int gi = g + l;
                if (gi >= niters) { iter = niters; stop = true; break; }
                if ((notf >> l) & 1u) { iter = gi; nf = 1; stop = true; break; }       // getSubset failed: the loop ends here
                const int cl = __shfl_sync(HG_FULL, c, l);
                best = cl; hyp = gi;
                niters = ransac_update_num_iters<4>(a.conf, (double)(n - cl) / (double)n, niters);
                if (gi + 1 >= niters) { iter = gi + 1; stop = true; break; }
            }
            if (!stop) {
                if (g + 32 >= niters) { iter = niters; stop = true; }
                else iter = g + 32;
            }
        }
        run = !stop;
        if (hyp != hyp_in && lane < 9) bestH[lane] = a.H[(slot0 + (hyp - a.round * HG_ROUND)) * 9 + lane];
        if (run && lane == 0) a.running[0] = 1;
    }
    if (lane == 0) {
        st[HS_ITER] = iter; st[HS_NITERS] = niters; st[HS_BEST] = best; st[HS_HYP] = hyp; st[HS_RUN] = run; st[HS_N] = (int)n;
        st[HS_NOT_FOUND] = nf;
    }
}

// ---------------------------------------------------------------------------------------------------------------- refine
// maximum of v over the CTA into *out (visible to every thread on return)
__device__ __forceinline__ void cta_max(double v, double (*red)[HG_NRED], double* out) {
#pragma unroll
    for (int d = 16; d; d >>= 1) v = fmax(v, __shfl_xor_sync(HG_FULL, v, d));
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][0] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        double m = 0.0;
        for (int q = 0; q < HG_REFINE_THREADS / 32; ++q) m = fmax(m, red[q][0]);
        *out = m;
    }
    __syncthreads();
}

// OpenCV's HomographyRefineCallback in double: with g = (Mx, My, 1) ww, ww = 1 / (h6 Mx + h7 My + 1) (0 when |.| <= DBL_EPSILON),
// (xi, yi) = (h0 Mx + h1 My + h2, h3 Mx + h4 My + h5) ww, the residual is r = (xi - x', yi - y') and the Jacobian rows are
// Jx = (g, 0, 0, 0, -g0 xi, -g1 xi), Jy = (0, 0, 0, g, -g0 yi, -g1 yi).  J^T J, J^T r and |r|^2 are assembled from the distinct
// sums (the two 3x3 blocks of J^T J coincide, the off-diagonal 3x3 block is zero), which keeps the per-thread partials in registers:
//   [0, 6) g_i g_j (i <= j < 3)   [6, 12) g_i g_j xi (i < 3, j < 2)   [12, 18) g_i g_j yi   [18, 21) g_i g_j (xi^2 + yi^2) (i <= j < 2)
//   [21, 24) g_i rx   [24, 27) g_i ry   [27, 29) g_j (xi rx + yi ry)   [29] |r|^2   [30] max |r| (a maximum, reduced apart)
constexpr int LM_SUMS = 30;
__device__ __forceinline__ void lm_partials(const double* h, const float2* S, const float2* Dp, const uint8_t* sel, int64_t n,
                                            double (&acc)[HG_NRED]) {
#pragma unroll
    for (int k = 0; k <= LM_SUMS; ++k) acc[k] = 0.0;
    for (int64_t i = threadIdx.x; i < n; i += HG_REFINE_THREADS) {
        if (!sel[i]) continue;
        const float2 s = S[i], d = Dp[i];
        const double Mx = s.x, My = s.y;
        double ww = h[6] * Mx + h[7] * My + 1.0;
        ww = fabs(ww) > HG_DBL_EPS ? 1.0 / ww : 0.0;
        const double xi = (h[0] * Mx + h[1] * My + h[2]) * ww;
        const double yi = (h[3] * Mx + h[4] * My + h[5]) * ww;
        const double rx = xi - (double)d.x, ry = yi - (double)d.y;
        const double g[3] = {Mx * ww, My * ww, ww};
        const double q2 = xi * xi + yi * yi, qr = xi * rx + yi * ry;
        acc[0] += g[0] * g[0]; acc[1] += g[0] * g[1]; acc[2] += g[0] * g[2];
        acc[3] += g[1] * g[1]; acc[4] += g[1] * g[2]; acc[5] += g[2] * g[2];
#pragma unroll
        for (int u = 0; u < 3; ++u)
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                const double gg = g[u] * g[v];
                acc[6 + 2 * u + v] += gg * xi;
                acc[12 + 2 * u + v] += gg * yi;
            }
        acc[18] += g[0] * g[0] * q2; acc[19] += g[0] * g[1] * q2; acc[20] += g[1] * g[1] * q2;
#pragma unroll
        for (int u = 0; u < 3; ++u) { acc[21 + u] += g[u] * rx; acc[24 + u] += g[u] * ry; }
        acc[27] += g[0] * qr; acc[28] += g[1] * qr;
        acc[29] += rx * rx + ry * ry;
        acc[30] = fmax(acc[30], fmax(fabs(rx), fabs(ry)));
    }
}

// J^T J (8x8), J^T r (8) and |r|^2 from the totals of lm_partials
__device__ __forceinline__ void lm_assemble(const double* t, double (*A)[8], double* v, double& S) {
    for (int r = 0; r < 8; ++r)
        for (int c = 0; c < 8; ++c) A[r][c] = 0.0;
    const int gi[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
    for (int u = 0; u < 3; ++u)
        for (int w = 0; w < 3; ++w) { A[u][w] = t[gi[u][w]]; A[3 + u][3 + w] = t[gi[u][w]]; }
    for (int u = 0; u < 3; ++u)
        for (int w = 0; w < 2; ++w) {
            A[u][6 + w] = A[6 + w][u] = -t[6 + 2 * u + w];
            A[3 + u][6 + w] = A[6 + w][3 + u] = -t[12 + 2 * u + w];
        }
    A[6][6] = t[18]; A[6][7] = A[7][6] = t[19]; A[7][7] = t[20];
    for (int u = 0; u < 3; ++u) { v[u] = t[21 + u]; v[3 + u] = t[24 + u]; }
    v[6] = -t[27]; v[7] = -t[28];
    S = t[29];
}

// solves the 8x8 system M d = r by Gauss-Jordan with partial pivoting (one thread, shared memory); false when singular
__device__ bool solve8(double (*M)[17], int ncols) {
#pragma unroll 1
    for (int k = 0; k < 8; ++k) {
        int piv = k;
        for (int r = k + 1; r < 8; ++r)
            if (fabs(M[r][k]) > fabs(M[piv][k])) piv = r;
        if (piv != k)
            for (int c = 0; c < ncols; ++c) { const double t = M[k][c]; M[k][c] = M[piv][c]; M[piv][c] = t; }
        const double p = M[k][k];
        if (!(fabs(p) > 0.0) || !isfinite(p)) return false;
        for (int c = 0; c < ncols; ++c) M[k][c] /= p;
        for (int r = 0; r < 8; ++r) {
            if (r == k) continue;
            const double f = M[r][k];
            for (int c = 0; c < ncols; ++c) M[r][c] -= f * M[k][c];
        }
    }
    return true;
}

struct RefineSmem {
    double red[HG_REFINE_THREADS / 32][HG_NRED];
    double tot[HG_NRED];
    double L[9][9], V[9][9];
    double H[9];
    double x[8], xd[8], d[8], v[8], D[8];
    double A[8][8];
    double M[8][17];
    double S, rinf, rinf_d, lambda, lc;
    int flag;
};

__global__ void __launch_bounds__(HG_REFINE_THREADS, 1) homog_refine_kernel(rb_homography_args a) {
    rb::pdl_wait();
    __shared__ RefineSmem sm;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int* st = a.state + (int64_t)b * RB_HOMOG_STATE;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const float2* S = reinterpret_cast<const float2*>(a.src) + off;
    const float2* Dp = reinterpret_cast<const float2*>(a.dst) + off;
    uint8_t* mask = a.mask + off;
    double* outH = a.out_H + (int64_t)b * 9;
    const bool ransac = a.method != 0;
    const bool have = n >= 4 && (!ransac || st[HS_BEST] > 0);
    auto fail = [&]() {
        for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) mask[i] = 0;
        if (tid < 9) outH[tid] = 0.0;
        if (tid == 0) a.ok[b] = 0;
    };
    if (!have) { fail(); return; }
    // ---- the inlier mask of the best model (RANSAC), or every point (method 0)
    if (ransac && n > 4) {
        float f[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) f[i] = __double2float_rn(a.best_H[(int64_t)b * 9 + i]);
        const float t = homog_thresh(a.thresh);
        for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) {
            const float2 s = S[i], d = Dp[i];
            mask[i] = homog_inlier(f, s.x, s.y, d.x, d.y, t);
        }
    } else {
        for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) mask[i] = 1;
    }
    if (tid < 9) sm.H[tid] = ransac ? a.best_H[(int64_t)b * 9 + tid] : 0.0;
    __syncthreads();
    if (ransac && n == 4) {                          // the minimal case: no refinement
        if (tid < 9) outH[tid] = sm.H[tid];
        if (tid == 0) a.ok[b] = 1;
        return;
    }
    // ---- normalised DLT over the selected points (HomographyEstimatorCallback::runKernel)
    double acc[HG_NRED];
    {
        double s4[4] = {0.0, 0.0, 0.0, 0.0};
        double cnt[1] = {0.0};
        for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) {
            if (!mask[i]) continue;
            const float2 s = S[i], d = Dp[i];
            s4[0] += d.x; s4[1] += d.y; s4[2] += s.x; s4[3] += s.y;
            cnt[0] += 1.0;
        }
        cta_sum<1, HG_REFINE_THREADS>(cnt, sm.red, sm.tot);
        const double count = sm.tot[0];
        cta_sum<4, HG_REFINE_THREADS>(s4, sm.red, sm.tot);
        const double cmx = sm.tot[0] / count, cmy = sm.tot[1] / count, cMx = sm.tot[2] / count, cMy = sm.tot[3] / count;
        double a4[4] = {0.0, 0.0, 0.0, 0.0};
        for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) {
            if (!mask[i]) continue;
            const float2 s = S[i], d = Dp[i];
            a4[0] += fabs(d.x - cmx); a4[1] += fabs(d.y - cmy); a4[2] += fabs(s.x - cMx); a4[3] += fabs(s.y - cMy);
        }
        cta_sum<4, HG_REFINE_THREADS>(a4, sm.red, sm.tot);
        const bool degenerate = !(fabs(sm.tot[0]) >= HG_DBL_EPS && fabs(sm.tot[1]) >= HG_DBL_EPS && fabs(sm.tot[2]) >= HG_DBL_EPS &&
                                  fabs(sm.tot[3]) >= HG_DBL_EPS);
        if (degenerate) {
            // OpenCV keeps the RANSAC model and refines it; least squares on all points has no model
            if (!ransac) { fail(); return; }
        } else {
            const double smx = count / sm.tot[0], smy = count / sm.tot[1], sMx = count / sm.tot[2], sMy = count / sm.tot[3];
            // L^T L from its distinct sums, p = (X, Y, 1): the two 3x3 blocks p p^T coincide, the off-diagonal block is zero,
            // [0, 6) p_i p_j (i <= j < 3, p_2 p_2 = count)   [6, 15) -p_i p_j x   [15, 24) -p_i p_j y   [24, 30) p_i p_j (x^2 + y^2)
#pragma unroll
            for (int k = 0; k < LM_SUMS; ++k) acc[k] = 0.0;
            for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) {
                if (!mask[i]) continue;
                const float2 s = S[i], d = Dp[i];
                const double x = (d.x - cmx) * smx, y = (d.y - cmy) * smy;
                const double p[3] = {(s.x - cMx) * sMx, (s.y - cMy) * sMy, 1.0};
                const double q2 = x * x + y * y;
                int k = 0;
#pragma unroll
                for (int u = 0; u < 3; ++u)
#pragma unroll
                    for (int w = u; w < 3; ++w) {
                        const double pp = p[u] * p[w];
                        acc[k] += pp; acc[24 + k] += pp * q2;
                        ++k;
                    }
#pragma unroll
                for (int u = 0; u < 3; ++u)
#pragma unroll
                    for (int w = 0; w < 3; ++w) {
                        const double pp = p[u] * p[w];
                        acc[6 + 3 * u + w] -= pp * x;
                        acc[15 + 3 * u + w] -= pp * y;
                    }
            }
            cta_sum<LM_SUMS, HG_REFINE_THREADS>(acc, sm.red, sm.tot);
            if (tid == 0) {
                const int pi[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
                for (int r = 0; r < 9; ++r)
                    for (int c = 0; c < 9; ++c) sm.L[r][c] = 0.0;
                for (int u = 0; u < 3; ++u)
                    for (int w = 0; w < 3; ++w) {
                        sm.L[u][w] = sm.L[3 + u][3 + w] = sm.tot[pi[u][w]];
                        sm.L[u][6 + w] = sm.L[6 + w][u] = sm.tot[6 + 3 * u + w];
                        sm.L[3 + u][6 + w] = sm.L[6 + w][3 + u] = sm.tot[15 + 3 * u + w];
                        sm.L[6 + u][6 + w] = sm.tot[24 + pi[u][w]];
                    }
            }
            __syncthreads();
            if (tid < 32) jacobi_eig_warp<9>(sm.L, sm.V, 15);
            __syncthreads();
            if (tid == 0) {
                int kmin = 0;
                for (int i = 1; i < 9; ++i)
                    if (sm.L[i][i] < sm.L[kmin][kmin]) kmin = i;
                double h0[9], H[9];
                for (int i = 0; i < 9; ++i) h0[i] = sm.V[i][kmin];
                denormalise(h0, cmx, cmy, smx, smy, cMx, cMy, sMx, sMy, H);
                bool fin = true;
                for (int i = 0; i < 9; ++i) fin &= isfinite(H[i]);
                sm.flag = fin;
                if (fin)
                    for (int i = 0; i < 9; ++i) sm.H[i] = H[i];
            }
            __syncthreads();
            if (!sm.flag && !ransac) { fail(); return; }
        }
    }
    if (n == 4) {                                    // least squares on exactly 4 points: no refinement
        if (tid < 9) outH[tid] = sm.H[tid];
        if (tid == 0) a.ok[b] = 1;
        return;
    }
    // ---- Levenberg-Marquardt on the 8 parameters (H[2][2] fixed), restated in oracle/homography_ransac.py:lm_refine
    if (tid < 8) sm.x[tid] = sm.H[tid];
    __syncthreads();
    lm_partials(sm.x, S, Dp, mask, n, acc);
    cta_max(acc[LM_SUMS], sm.red, &sm.rinf_d);
    cta_sum<LM_SUMS, HG_REFINE_THREADS>(acc, sm.red, sm.tot);
    if (tid == 0) {
        lm_assemble(sm.tot, sm.A, sm.v, sm.S);
        for (int r = 0; r < 8; ++r) sm.D[r] = sm.A[r][r];
        sm.rinf = sm.rinf_d;
        sm.lambda = 1.0; sm.lc = 0.75;
    }
    __syncthreads();
    for (int it = 0; it < 10; ++it) {
        if (tid == 0) {                              // d = (A + lambda diag(D))^-1 v, xd = x - d
            for (int r = 0; r < 8; ++r) {
                for (int c = 0; c < 8; ++c) sm.M[r][c] = sm.A[r][c];
                sm.M[r][r] += sm.lambda * sm.D[r];
                sm.M[r][8] = sm.v[r];
            }
            sm.flag = solve8(sm.M, 9);
            for (int r = 0; r < 8; ++r) { sm.d[r] = sm.flag ? sm.M[r][8] : 0.0; sm.xd[r] = sm.x[r] - sm.d[r]; }
        }
        __syncthreads();
        if (!sm.flag) break;
        // the residual at xd, and (used only if the step is taken) J^T J and J^T r there
        lm_partials(sm.xd, S, Dp, mask, n, acc);
        cta_max(acc[LM_SUMS], sm.red, &sm.rinf_d);
        cta_sum<LM_SUMS, HG_REFINE_THREADS>(acc, sm.red, sm.tot);
        if (tid == 0) {
            const double Sd = sm.tot[29];
            double dS = 0.0, dv = 0.0, dinf = 0.0;
            for (int r = 0; r < 8; ++r) {
                double Ad = 0.0;
                for (int c = 0; c < 8; ++c) Ad += sm.A[r][c] * sm.d[c];
                dS += sm.d[r] * (2.0 * sm.v[r] - Ad);
                dv += sm.d[r] * sm.v[r];
                dinf = fmax(dinf, fabs(sm.d[r]));
            }
            const double R = (sm.S - Sd) / (fabs(dS) > HG_DBL_EPS ? dS : 1.0);
            if (R > 0.75) {
                sm.lambda *= 0.5;
                if (sm.lambda < sm.lc) sm.lambda = 0.0;
            } else if (R < 0.25) {
                double nu = (Sd - sm.S) / (fabs(dv) > HG_DBL_EPS ? dv : 1.0) + 2.0;
                nu = fmin(fmax(nu, 2.0), 10.0);
                if (sm.lambda == 0.0) {              // lambda = lc = 1 / max |diag(inv(A))|
                    for (int r = 0; r < 8; ++r)
                        for (int c = 0; c < 16; ++c) sm.M[r][c] = c < 8 ? sm.A[r][c] : (c - 8 == r ? 1.0 : 0.0);
                    double maxval = HG_DBL_EPS;
                    if (solve8(sm.M, 16))
                        for (int r = 0; r < 8; ++r) maxval = fmax(maxval, fabs(sm.M[r][8 + r]));
                    sm.lambda = sm.lc = 1.0 / maxval;
                    nu *= 0.5;
                }
                sm.lambda *= nu;
            }
            if (Sd < sm.S) {                         // take the step
                lm_assemble(sm.tot, sm.A, sm.v, sm.S);
                for (int r = 0; r < 8; ++r) sm.x[r] = sm.xd[r];
                sm.rinf = sm.rinf_d;
            }
            sm.flag = dinf >= HG_FLT_EPS && sm.rinf >= HG_FLT_EPS;
        }
        __syncthreads();
        if (!sm.flag) break;
    }
    if (tid < 8) outH[tid] = sm.x[tid];
    if (tid == 8) outH[8] = sm.H[8];
    if (tid == 0) a.ok[b] = 1;
    // OpenCV 4.13 returns the inliers of the refined model, by the same float32 test
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = __double2float_rn(sm.x[i]);
    const float t = homog_thresh(a.thresh);
    for (int64_t i = tid; i < n; i += HG_REFINE_THREADS) {
        const float2 s = S[i], d = Dp[i];
        mask[i] = homog_inlier(f, s.x, s.y, d.x, d.y, t);
    }
}

static int homog_check(const rb_homography_args* a, const char* what) {
    if (ransac_check(a, what, 65535, HG_ROUND)) return 1;
    RB_REQUIRE(a->src && a->dst, "%s: null argument", what);
    RB_REQUIRE(a->method == 0 || a->method == 8, "%s: method %d is neither 0 nor RANSAC (8)", what, a->method);
    return 0;
}

static int homog_splits(int64_t max_n) { return ransac_splits(max_n, 512, RB_HOMOG_MAX_SPLITS); }

}  // namespace rb

using namespace rb;

extern "C" int romab200_homography_hypotheses(const rb_homography_args* a, void* stream) {
    if (homog_check(a, "homography_hypotheses")) return 1;
    RB_REQUIRE(a->sample && a->attempts && a->status && a->H && a->running, "homography_hypotheses: null output");
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(cudaMemsetAsync(a->running, 0, sizeof(int32_t), st) == cudaSuccess, "homography_hypotheses: memset failed");
    rb::launch_pdl(homog_hypotheses_kernel, dim3(HG_ROUND / HG_THREADS, a->batch), dim3(HG_THREADS), 0, st, *a);
    return check_launch("homography_hypotheses");
}

extern "C" int romab200_homography_score(const rb_homography_args* a, void* stream) {
    if (homog_check(a, "homography_score")) return 1;
    RB_REQUIRE(a->status && a->H && a->counts, "homography_score: null argument");
    const int splits = homog_splits(a->max_n);
    const int per_split = (int)((a->max_n + splits - 1) / splits);
    rb::launch_pdl(homog_score_kernel, dim3(HG_ROUND / HG_THREADS, splits, a->batch), dim3(HG_THREADS), 0, (cudaStream_t)stream, *a,
                   max(per_split, 1));
    return check_launch("homography_score");
}

extern "C" int romab200_homography_select(const rb_homography_args* a, void* stream) {
    if (homog_check(a, "homography_select")) return 1;
    RB_REQUIRE(a->status && a->H && a->counts && a->best_H && a->running, "homography_select: null argument");
    rb::launch_pdl(homog_select_kernel, dim3((a->batch + 3) / 4), dim3(128), 0, (cudaStream_t)stream, *a, homog_splits(a->max_n));
    return check_launch("homography_select");
}

extern "C" int romab200_homography_refine(const rb_homography_args* a, void* stream) {
    RB_REQUIRE(a && a->src && a->dst && a->offsets && a->state && a->best_H && a->out_H && a->ok && a->mask, "homography_refine: null argument");
    RB_REQUIRE(a->batch > 0 && a->batch <= 65535, "homography_refine: batch %d outside [1, 65535]", a->batch);
    RB_REQUIRE(a->method == 0 || a->method == 8, "homography_refine: method %d is neither 0 nor RANSAC (8)", a->method);
    rb::launch_pdl(homog_refine_kernel, dim3(a->batch), dim3(HG_REFINE_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("homography_refine");
}
