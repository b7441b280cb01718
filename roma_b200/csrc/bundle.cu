// Bundle adjustment of cameras and track points (include/romab200.h): Levenberg-Marquardt with a Schur-reduced camera system.
//   setup      a warp per track checks its used elements and keys them by image; radix_sort_hi32 (common.cuh) makes the list
//              camera-major, ascending element order within an image; per-image offsets by binary search.
//   linearize  a warp per track: residuals, IRLS weights and Jacobians of its used observations; V_k, g_k and the cost summed by a
//              xor butterfly; the damped V_k^-1 and every observation's W_e = w J_c^T J_X.
//   cameras    a CTA per free camera walks its observations in list order: U_i, g_i, and row i of S = U - W V^-1 W^T (every entry
//              written by one thread per observation, in list order; the observations of a track lie in distinct images).
//   cholesky   right-looking, RB_BA_NB-wide panels (panel, triangular solve, trailing update), then both substitutions.
//   step       the trial cameras (Rodrigues), then a warp per track: d_X, the trial cost and the depth check; fixed-order tree sums.
// No float atomics and a fixed order in every reduction, so the result is bit-identical from run to run.
// The kernels that touch a camera are templated on the camera model M: 0 = PINHOLE (6 parameters per camera), 1 = SIMPLE_RADIAL
// (8: the pose, then f and k).
#include "common.cuh"

namespace rb {

constexpr int BA_THREADS = 128;
constexpr int BA_WARPS = BA_THREADS / 32;
constexpr int BA_CAM_THREADS = 256;
constexpr int BA_SUM_THREADS = 1024;
constexpr unsigned BA_FULL = 0xffffffffu;
constexpr int NB = RB_BA_NB;
static_assert(NB == 32, "the substitutions give a panel column to each lane of a warp");

// per model: camera parameters NC, the length of a cams row, and the thread that starts the W V^-1 products of the camera kernel
template <int M> struct BaModel;
template <> struct BaModel<0> { static constexpr int NC = 6, CAM = RB_BA_CAM, A0 = 32; };
template <> struct BaModel<1> { static constexpr int NC = 8, CAM = RB_BA_CAM1, A0 = 64; };

template <int N>
__device__ __forceinline__ void ba_warp_sum(double (&v)[N]) {
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int d = 16; d; d >>= 1) v[k] += __shfl_xor_sync(BA_FULL, v[k], d);
}

__device__ __forceinline__ bool ba_used(const rb_ba_args& a, int64_t e) { return a.inlier[e] != 0; }

// rule 2: rho(s) and w = rho'(s)
__device__ __forceinline__ double ba_rho(double s, double c2, double* w) {
    if (c2 == 0.0) {
        *w = 1.0;
        return s;
    }
    *w = 1.0 / (1.0 + s / c2);
    return c2 * log1p(s / c2);
}

// observation of element e (ids checked) under camera c at X: residual (ru, rv), depth and, with JAC, the Jacobians Jc [2][NC]
// and JX [2][3].  Model 0: c = R (9), t (3), K (9) and Jc = (d_omega, d_t).  Model 1: c = R (9), t (3), f, cx, cy, k and
// Jc = (d_omega, d_t, d_f, d_k).
template <bool JAC, int M>
__device__ __forceinline__ void ba_project(const double* c, const double (&X)[3], double ox, double oy, double* ru, double* rv,
                                           double* depth, double (*Jc)[BaModel<M>::NC], double (*JX)[3]) {
    double A[3], p[3];
#pragma unroll
    for (int j = 0; j < 3; ++j) A[j] = c[3 * j] * X[0] + c[3 * j + 1] * X[1] + c[3 * j + 2] * X[2];
#pragma unroll
    for (int j = 0; j < 3; ++j) p[j] = A[j] + c[9 + j];
    double Jp[2][3];
    if constexpr (M == 0) {
        double q[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) q[j] = c[12 + 3 * j] * p[0] + c[13 + 3 * j] * p[1] + c[14 + 3 * j] * p[2];
        const double u = q[0] / q[2], v = q[1] / q[2];
        *ru = u - ox;
        *rv = v - oy;
        *depth = p[2];
        if (!JAC) return;
        const double iz = 1.0 / q[2];
        double Jq[2][3] = {{iz, 0.0, -u * iz}, {0.0, iz, -v * iz}};
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int m = 0; m < 3; ++m) Jp[r][m] = Jq[r][0] * c[12 + m] + Jq[r][1] * c[15 + m] + Jq[r][2] * c[18 + m];
    } else {
        const double f = c[12], k = c[15];
        const double x = p[0] / p[2], y = p[1] / p[2], r2 = x * x + y * y, d = 1.0 + k * r2;
        *ru = f * d * x + c[13] - ox;
        *rv = f * d * y + c[14] - oy;
        *depth = p[2];
        if (!JAC) return;
        // d(u, v)/d(x, y), then through (x, y) = (p0, p1) / p2
        const double iz = 1.0 / p[2];
        const double uxx = f * (d + 2.0 * k * x * x), uxy = 2.0 * f * k * x * y, uyy = f * (d + 2.0 * k * y * y);
        Jp[0][0] = uxx * iz; Jp[0][1] = uxy * iz; Jp[0][2] = -(uxx * x + uxy * y) * iz;
        Jp[1][0] = uxy * iz; Jp[1][1] = uyy * iz; Jp[1][2] = -(uxy * x + uyy * y) * iz;
        Jc[0][6] = d * x; Jc[1][6] = d * y;
        Jc[0][7] = f * r2 * x; Jc[1][7] = f * r2 * y;
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        // d/d_omega of Exp(d_omega) R X is -[R X]x, so row r is (R X) x Jp
        Jc[r][0] = A[1] * Jp[r][2] - A[2] * Jp[r][1];
        Jc[r][1] = A[2] * Jp[r][0] - A[0] * Jp[r][2];
        Jc[r][2] = A[0] * Jp[r][1] - A[1] * Jp[r][0];
#pragma unroll
        for (int m = 0; m < 3; ++m) Jc[r][3 + m] = Jp[r][m];
#pragma unroll
        for (int m = 0; m < 3; ++m) JX[r][m] = Jp[r][0] * c[m] + Jp[r][1] * c[3 + m] + Jp[r][2] * c[6 + m];
    }
}

__device__ __forceinline__ void ba_keypoint(const rb_ba_args& a, int64_t e, int* img, double* ox, double* oy) {
    const int i = a.elements[2 * e];
    const int64_t r = a.kp_offsets[i] + a.elements[2 * e + 1];
    *img = i;
    *ox = (double)a.keypoints[2 * r];
    *oy = (double)a.keypoints[2 * r + 1];
}

__device__ __forceinline__ double ba_clamp_diag(double h) { return fmin(fmax(h, 1e-6), 1e32); }

// ---- setup ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(BA_THREADS) ba_setup_kernel(rb_ba_args a) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * BA_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * BA_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) {
        const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
        const bool ok = a.track_ok[k] != 0;
        int bad = 0;
        for (int64_t e = lane; e < L; e += 32) {
            const int64_t g = base + e;
            a.elem_track[g] = (int32_t)k;
            int img = a.num_images;
            if (ok && ba_used(a, g)) {
                const int i = a.elements[2 * g], id = a.elements[2 * g + 1];
                if (i < 0 || i >= a.num_images || id < 0 || id >= a.kp_offsets[i + 1] - a.kp_offsets[i]) {
                    bad |= RB_BA_BAD_ID;
                } else {
                    img = i;
                    for (int64_t f = e + 1; f < L; ++f)
                        if (ba_used(a, base + f) && a.elements[2 * (base + f)] == i) bad |= RB_BA_REPEATED;
                }
            }
            a.keys[g] = ((unsigned long long)(uint32_t)img << 32) | (uint32_t)g;
        }
        bad = __reduce_or_sync(BA_FULL, bad);
        if (lane == 0 && bad) atomicOr((unsigned long long*)a.info, (unsigned long long)bad);
    }
}

// obs_offsets[i] = the first sorted key of image >= i; obs = the element ids in sorted order; info[1] = the used observations
__global__ void __launch_bounds__(256) ba_offsets_kernel(rb_ba_args a, const uint64_t* __restrict__ sorted) {
    pdl_wait();
    const int64_t t0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, step = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = t0; i <= a.num_images; i += step) {
        int64_t lo = 0, hi = a.num_elements;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if ((int64_t)(sorted[mid] >> 32) < i) lo = mid + 1;
            else hi = mid;
        }
        a.obs_offsets[i] = lo;
        if (i == a.num_images) a.info[1] = lo;
    }
    for (int64_t q = t0; q < a.num_elements; q += step) a.obs[q] = (int32_t)(uint32_t)sorted[q];
}

// ---- linearize --------------------------------------------------------------------------------------------------------------
template <int M>
__global__ void __launch_bounds__(BA_THREADS) ba_linearize_kernel(rb_ba_args a) {
    constexpr int NC = BaModel<M>::NC;
    pdl_wait();
    const int lane = threadIdx.x & 31;
    if (blockIdx.x == 0 && threadIdx.x < RB_BA_RESULT) a.result[threadIdx.x] = 0.0;
    const int64_t stride = (int64_t)gridDim.x * BA_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * BA_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) {
        double* out = a.track_sys + k * RB_BA_TRACK;
        if (!a.track_ok[k]) {
            if (lane < RB_BA_TRACK) out[lane] = 0.0;
            continue;
        }
        const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
        const double X[3] = {a.X[3 * k], a.X[3 * k + 1], a.X[3 * k + 2]};
        double s[10];                                     // V (00, 01, 02, 11, 12, 22), g_X (3), cost
#pragma unroll
        for (int j = 0; j < 10; ++j) s[j] = 0.0;
        for (int64_t e = base + lane; e < base + L; e += 32) {
            if (!ba_used(a, e)) continue;
            int img;
            double ox, oy, ru, rv, depth, Jc[2][NC], JX[2][3], w;
            ba_keypoint(a, e, &img, &ox, &oy);
            ba_project<true, M>(a.cams + (int64_t)img * BaModel<M>::CAM, X, ox, oy, &ru, &rv, &depth, Jc, JX);
            s[9] += 0.5 * ba_rho(ru * ru + rv * rv, a.loss_scale2, &w);
            s[0] += w * (JX[0][0] * JX[0][0] + JX[1][0] * JX[1][0]);
            s[1] += w * (JX[0][0] * JX[0][1] + JX[1][0] * JX[1][1]);
            s[2] += w * (JX[0][0] * JX[0][2] + JX[1][0] * JX[1][2]);
            s[3] += w * (JX[0][1] * JX[0][1] + JX[1][1] * JX[1][1]);
            s[4] += w * (JX[0][1] * JX[0][2] + JX[1][1] * JX[1][2]);
            s[5] += w * (JX[0][2] * JX[0][2] + JX[1][2] * JX[1][2]);
#pragma unroll
            for (int m = 0; m < 3; ++m) s[6 + m] += w * (JX[0][m] * ru + JX[1][m] * rv);
            double* W = a.W + e * (3 * NC);
#pragma unroll
            for (int r = 0; r < NC; ++r)
#pragma unroll
                for (int m = 0; m < 3; ++m) W[3 * r + m] = w * (Jc[0][r] * JX[0][m] + Jc[1][r] * JX[1][m]);
        }
        ba_warp_sum(s);
        const double D0 = ba_clamp_diag(s[0]), D1 = ba_clamp_diag(s[3]), D2 = ba_clamp_diag(s[5]);
        const double a00 = s[0] + a.lambda * D0, a01 = s[1], a02 = s[2], a11 = s[3] + a.lambda * D1, a12 = s[4], a22 = s[5] + a.lambda * D2;
        const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
        const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
        const double idet = 1.0 / (a00 * c00 + a01 * c01 + a02 * c02);
        const double v[RB_BA_TRACK] = {c00 * idet, c01 * idet, c02 * idet, c11 * idet, c12 * idet, c22 * idet, s[6], s[7], s[8], D0, D1, D2, s[9]};
#pragma unroll
        for (int j = 0; j < RB_BA_TRACK; ++j)
            if (lane == j) out[j] = v[j];
    }
}

// ---- camera blocks ------------------------------------------------------------------------------------------------------------
template <int M>
__global__ void __launch_bounds__(BA_CAM_THREADS) ba_cameras_kernel(rb_ba_args a) {
    constexpr int NC = BaModel<M>::NC, NU = NC * (NC + 1) / 2, A0 = BaModel<M>::A0;
    pdl_wait();
    __shared__ double sJ[2 * NC + 3];  // Jc (2 NC), r (2), w of the current observation
    __shared__ double sA[3 * NC];      // W_e V_k^-1 (NC x 3)
    __shared__ double sW[3 * NC], sV[9], sg[3];
    const int fi = blockIdx.x, tid = threadIdx.x;
    const int img = a.free_cams[fi];
    const int64_t n = NC * (int64_t)a.num_free;
    double* Srow = a.S + NC * (int64_t)fi * n;
    for (int64_t q = tid; q < NC * n; q += BA_CAM_THREADS) Srow[q] = 0.0;
    // thread t < NU accumulates U entry (p, q), p <= q, in row-major order of the upper triangle; NU <= t < NU + NC g_c;
    // NU + NC <= t < NU + 2 NC the reduced right-hand side's W V^-1 g_X term
    int up = 0, uq = 0;
    if (tid < NU) {
        int t = tid;
        while (t >= NC - up) { t -= NC - up; ++up; }
        uq = up + t;
    }
    double acc = 0.0;
    const double* cam = a.cams + (int64_t)img * BaModel<M>::CAM;
    for (int64_t o = a.obs_offsets[img]; o < a.obs_offsets[img + 1]; ++o) {
        const int64_t e = a.obs[o];
        const int64_t k = a.elem_track[e];
        __syncthreads();                                  // the previous observation is done with the shared operands
        if (tid == 0) {
            int im;
            double ox, oy, ru, rv, depth, Jc[2][NC], JX[2][3], w;
            ba_keypoint(a, e, &im, &ox, &oy);
            const double X[3] = {a.X[3 * k], a.X[3 * k + 1], a.X[3 * k + 2]};
            ba_project<true, M>(cam, X, ox, oy, &ru, &rv, &depth, Jc, JX);
            ba_rho(ru * ru + rv * rv, a.loss_scale2, &w);
#pragma unroll
            for (int r = 0; r < NC; ++r) { sJ[r] = Jc[0][r]; sJ[NC + r] = Jc[1][r]; }
            sJ[2 * NC] = ru; sJ[2 * NC + 1] = rv; sJ[2 * NC + 2] = w;
        } else if (tid >= 32 && tid < 32 + 3 * NC) {
            sW[tid - 32] = a.W[e * (3 * NC) + tid - 32];
        } else if (tid >= 64 && tid < 73) {
            const int r = (tid - 64) / 3, c = (tid - 64) % 3;
            const int lo = min(r, c), hi = max(r, c);
            sV[tid - 64] = a.track_sys[k * RB_BA_TRACK + (lo == 0 ? hi : (lo == 1 ? 2 + hi : 5))];
        } else if (tid >= 96 && tid < 99) {
            sg[tid - 96] = a.track_sys[k * RB_BA_TRACK + 6 + tid - 96];
        }
        __syncthreads();
        if (tid < NU) {
            acc += sJ[2 * NC + 2] * (sJ[up] * sJ[uq] + sJ[NC + up] * sJ[NC + uq]);
        } else if (tid < NU + NC) {
            const int p = tid - NU;
            acc += sJ[2 * NC + 2] * (sJ[p] * sJ[2 * NC] + sJ[NC + p] * sJ[2 * NC + 1]);
        } else if (tid >= A0 && tid < A0 + 3 * NC) {
            const int r = (tid - A0) / 3, c = (tid - A0) % 3;
            sA[tid - A0] = sW[3 * r] * sV[c] + sW[3 * r + 1] * sV[3 + c] + sW[3 * r + 2] * sV[6 + c];
        }
        __syncthreads();
        if (tid >= NU + NC && tid < NU + 2 * NC) {
            const int p = tid - NU - NC;
            acc += sA[3 * p] * sg[0] + sA[3 * p + 1] * sg[1] + sA[3 * p + 2] * sg[2];
        }
        // block (fi, fj) -= A W_e'^T over the track's used observations in free cameras fj <= fi
        const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
        for (int64_t q = tid; q < NC * NC * L; q += BA_CAM_THREADS) {
            const int64_t f = base + q / (NC * NC);
            if (!ba_used(a, f)) continue;
            const int fj = a.free_index[a.elements[2 * f]];
            if (fj < 0 || fj > fi) continue;
            const int r = (int)(q % (NC * NC)) / NC, c = (int)(q % (NC * NC)) % NC;
            const double* Wf = a.W + f * (3 * NC) + 3 * c;
            Srow[r * n + NC * (int64_t)fj + c] -= sA[3 * r] * Wf[0] + sA[3 * r + 1] * Wf[1] + sA[3 * r + 2] * Wf[2];
        }
    }
    __syncthreads();
    // U and its damping on the diagonal block, the right-hand side, g_c and D_c
    double* diag = Srow + NC * (int64_t)fi;
    if (tid < NU) {
        double u = acc;
        if (up == uq) {
            const double D = ba_clamp_diag(acc);
            a.cam_sys[2 * NC * (int64_t)fi + NC + up] = D;
            u += a.lambda * D;
        }
        diag[up * n + uq] += u;
        if (up != uq) diag[uq * n + up] += acc;
    }
    __syncthreads();
    __shared__ double sb[NC];
    if (tid >= NU && tid < NU + NC) sb[tid - NU] = -acc;
    __syncthreads();
    if (tid >= NU && tid < NU + NC) a.cam_sys[2 * NC * (int64_t)fi + tid - NU] = acc;
    if (tid >= NU + NC && tid < NU + 2 * NC) a.rhs[NC * (int64_t)fi + tid - NU - NC] = sb[tid - NU - NC] + acc;
    __syncthreads();
    // rule 4: a pinned row becomes e_r with a zero right-hand side, and so does its column.  Model 0 pins the t_x row of a camera
    // in fixed_tx; model 1 the rows set in pin.
    for (int64_t q = tid; q < NC * n; q += BA_CAM_THREADS) {
        const int r = (int)(q / n);
        const int64_t col = q % n, row = NC * (int64_t)fi + r;
        if (col > row) continue;
        bool row_pin, col_pin;
        if constexpr (M == 0) {
            row_pin = r == 3 && a.fixed_tx[fi];
            col_pin = col % 6 == 3 && a.fixed_tx[col / 6];
        } else {
            row_pin = a.pin[row] != 0;
            col_pin = a.pin[col] != 0;
        }
        if (row_pin || col_pin) Srow[q] = col == row ? 1.0 : 0.0;
        if (row_pin && col == row) a.rhs[row] = 0.0;
    }
}

// ---- shared intrinsics: fold and unfold -------------------------------------------------------------------------------------
// S' = P^T S P and b' = P^T b of order n' = 6F + 2G: free camera fi's pose rows at 6 fi, group g's (f, k) rows at 6F + 2g.  P maps
// camera fi's parameter p < 6 to pose row 6 fi + p and its f, k to its group's rows.  S holds its lower triangle (rows of 8F); so
// does S'.
__device__ __forceinline__ double ba_lower(const double* S, int64_t n, int64_t r, int64_t c) { return r >= c ? S[r * n + c] : S[c * n + r]; }

// a thread per entry (R, C) of S' with a pose column C <= R: pose-pose entries are copies, group-pose entries sum over the group's
// members in list order; then b'.  A pinned group row becomes 0 here (its diagonal is in the group-group block).
__global__ void __launch_bounds__(256) ba_fold_kernel(rb_ba_groups_args a) {
    pdl_wait();
    const int64_t F = a.num_free, n = 8 * F, np = 6 * F + 2 * (int64_t)a.num_groups, t0 = blockIdx.x * (int64_t)256 + threadIdx.x;
    const int64_t step = (int64_t)gridDim.x * 256;
    for (int64_t q = t0; q < np * 6 * F; q += step) {
        const int64_t R = q / (6 * F), C = q % (6 * F);
        if (C > R) continue;
        const int64_t c8 = 8 * (C / 6) + C % 6;
        double v;
        if (R < 6 * F) {
            v = a.S[(8 * (R / 6) + R % 6) * n + c8];
        } else {
            const int g = (int)((R - 6 * F) >> 1), j = (int)((R - 6 * F) & 1);
            v = 0.0;
            if (!a.group_pin[2 * g + j])
                for (int m = a.group_offsets[g]; m < a.group_offsets[g + 1]; ++m) v += ba_lower(a.S, n, 8 * (int64_t)a.group_members[m] + 6 + j, c8);
        }
        a.S_groups[R * np + C] = v;
    }
    for (int64_t R = t0; R < np; R += step) {
        double v;
        if (R < 6 * F) {
            v = a.rhs[8 * (R / 6) + R % 6];
        } else {
            const int g = (int)((R - 6 * F) >> 1), j = (int)((R - 6 * F) & 1);
            v = 0.0;
            if (!a.group_pin[2 * g + j])
                for (int m = a.group_offsets[g]; m < a.group_offsets[g + 1]; ++m) v += a.rhs[8 * (int64_t)a.group_members[m] + 6 + j];
        }
        a.rhs_groups[R] = v;
    }
}

// a CTA per group pair (g, h), h <= g: the 2 x 2 block of S' at rows 6F + 2g, columns 6F + 2h, each entry the sum over the
// |g| |h| member pairs (member pair q = (q / |h|, q % |h|)): every thread a strided slice in order, then a fixed tree.  A pinned
// row or column becomes that of the identity.
__global__ void __launch_bounds__(256) ba_fold_groups_kernel(rb_ba_groups_args a) {
    pdl_wait();
    const int g = blockIdx.y, h = blockIdx.x, tid = threadIdx.x;
    if (h > g) return;
    __shared__ double red[4][256];
    const int64_t F = a.num_free, n = 8 * F, np = 6 * F + 2 * (int64_t)a.num_groups;
    const int og = a.group_offsets[g], oh = a.group_offsets[h], nh = a.group_offsets[h + 1] - oh;
    const int64_t terms = (int64_t)(a.group_offsets[g + 1] - og) * nh;
    double s[4] = {0.0, 0.0, 0.0, 0.0};             // (j, l) = (0, 0), (0, 1), (1, 0), (1, 1)
    for (int64_t q = tid; q < terms; q += 256) {
        const int64_t r = 8 * (int64_t)a.group_members[og + q / nh] + 6, c = 8 * (int64_t)a.group_members[oh + q % nh] + 6;
#pragma unroll
        for (int k = 0; k < 4; ++k) s[k] += ba_lower(a.S, n, r + (k >> 1), c + (k & 1));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) red[k][tid] = s[k];
    __syncthreads();
    for (int w = 128; w; w >>= 1) {
        if (tid < w)
#pragma unroll
            for (int k = 0; k < 4; ++k) red[k][tid] += red[k][tid + w];
        __syncthreads();
    }
    if (tid < 4) {
        const int j = tid >> 1, l = tid & 1;
        const int64_t R = 6 * F + 2 * g + j, C = 6 * F + 2 * h + l;
        if (C <= R) {
            const bool pinned = a.group_pin[2 * g + j] || a.group_pin[2 * h + l];
            a.S_groups[R * np + C] = pinned ? (R == C ? 1.0 : 0.0) : red[tid][0];
        }
    }
}

// d = P d': a CTA per group, a thread per member writes its camera's 8 rows of rhs
__global__ void __launch_bounds__(128) ba_unfold_kernel(rb_ba_groups_args a) {
    pdl_wait();
    const int g = blockIdx.x;
    const int64_t F = a.num_free;
    const double* d = a.rhs_groups;
    for (int m = a.group_offsets[g] + threadIdx.x; m < a.group_offsets[g + 1]; m += 128) {
        const int64_t fi = a.group_members[m];
#pragma unroll
        for (int p = 0; p < 6; ++p) a.rhs[8 * fi + p] = d[6 * fi + p];
        a.rhs[8 * fi + 6] = d[6 * F + 2 * g];
        a.rhs[8 * fi + 7] = d[6 * F + 2 * g + 1];
    }
}

// ---- Cholesky -----------------------------------------------------------------------------------------------------------------
// the nb x nb diagonal block at k0 (nb <= NB), unblocked in shared memory; a pivot that is not > 0 and finite sets result[3]
__global__ void __launch_bounds__(256) ba_potrf_panel_kernel(double* S, int64_t n, int64_t k0, int nb, double* result) {
    pdl_wait();
    __shared__ double P[NB][NB + 1];
    const int tid = threadIdx.x;
    for (int q = tid; q < nb * nb; q += 256) P[q / nb][q % nb] = S[(k0 + q / nb) * n + k0 + q % nb];
    __syncthreads();
    for (int j = 0; j < nb; ++j) {
        if (tid == 0) {
            const double d = P[j][j];
            if (!(d > 0.0) || !isfinite(d)) result[3] = 1.0;
            P[j][j] = sqrt(d);
        }
        __syncthreads();
        if (tid > j && tid < nb) P[tid][j] /= P[j][j];
        __syncthreads();
        for (int q = tid; q < nb * nb; q += 256) {
            const int r = q / nb, c = q % nb;
            if (c > j && r >= c) P[r][c] -= P[r][j] * P[c][j];
        }
        __syncthreads();
    }
    for (int q = tid; q < nb * nb; q += 256)
        if (q % nb <= q / nb) S[(k0 + q / nb) * n + k0 + q % nb] = P[q / nb][q % nb];
}

// rows below the panel: L21 = A21 L11^-T, a thread per row
__global__ void __launch_bounds__(128) ba_trsm_kernel(double* S, int64_t n, int64_t k0) {
    pdl_wait();
    __shared__ double P[NB][NB + 1];
    for (int q = threadIdx.x; q < NB * NB; q += 128) P[q / NB][q % NB] = S[(k0 + q / NB) * n + k0 + q % NB];
    __syncthreads();
    const int64_t r = k0 + NB + blockIdx.x * (int64_t)128 + threadIdx.x;
    if (r >= n) return;
    double* row = S + r * n + k0;
    double x[NB];
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        double v = row[j];
#pragma unroll
        for (int m = 0; m < j; ++m) v -= x[m] * P[j][m];
        x[j] = v / P[j][j];
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) row[j] = x[j];
}

// trailing update of the lower triangle: A22 -= L21 L21^T, a 32 x 32 tile per CTA
__global__ void __launch_bounds__(256) ba_syrk_kernel(double* S, int64_t n, int64_t k0) {
    pdl_wait();
    const int bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    __shared__ double Ai[NB][NB + 1], Aj[NB][NB + 1];
    const int64_t k1 = k0 + NB, ri = k1 + (int64_t)bi * NB, rj = k1 + (int64_t)bj * NB;
    for (int q = threadIdx.x; q < NB * NB; q += 256) {
        const int r = q / NB, c = q % NB;
        Ai[r][c] = ri + r < n ? S[(ri + r) * n + k0 + c] : 0.0;
        Aj[r][c] = rj + r < n ? S[(rj + r) * n + k0 + c] : 0.0;
    }
    __syncthreads();
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int s = 0; s < NB / 8; ++s) {
        const int r = ty + 8 * s;
        const int64_t row = ri + r, col = rj + tx;
        if (row >= n || col > row) continue;
        double v = 0.0;
#pragma unroll
        for (int m = 0; m < NB; ++m) v += Ai[r][m] * Aj[tx][m];
        S[row * n + col] -= v;
    }
}

// rhs <- L^-T L^-1 rhs, one CTA: per panel, a warp solves the diagonal block and all threads update the rest
__global__ void __launch_bounds__(1024) ba_potrs_kernel(const double* __restrict__ S, int64_t n, double* rhs) {
    pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31;
    for (int64_t k0 = 0; k0 < n; k0 += NB) {
        const int nb = (int)min((int64_t)NB, n - k0);
        if (tid < 32) {
            double y = lane < nb ? rhs[k0 + lane] : 0.0;
            for (int j = 0; j < nb; ++j) {
                const double yj = __shfl_sync(BA_FULL, y, j) / S[(k0 + j) * n + k0 + j];
                if (lane == j) y = yj;
                if (lane > j && lane < nb) y -= S[(k0 + lane) * n + k0 + j] * yj;
            }
            if (lane < nb) rhs[k0 + lane] = y;
        }
        __syncthreads();
        for (int64_t r = k0 + nb + tid; r < n; r += 1024) {
            double v = rhs[r];
            for (int m = 0; m < nb; ++m) v -= S[r * n + k0 + m] * rhs[k0 + m];
            rhs[r] = v;
        }
        __syncthreads();
    }
    for (int64_t k0 = (n - 1) / NB * NB; k0 >= 0; k0 -= NB) {
        const int nb = (int)min((int64_t)NB, n - k0);
        if (tid < 32) {
            double x = lane < nb ? rhs[k0 + lane] : 0.0;
            for (int j = nb - 1; j >= 0; --j) {
                const double xj = __shfl_sync(BA_FULL, x, j) / S[(k0 + j) * n + k0 + j];
                if (lane == j) x = xj;
                if (lane < j) x -= S[(k0 + j) * n + k0 + lane] * xj;
            }
            if (lane < nb) rhs[k0 + lane] = x;
        }
        __syncthreads();
        for (int64_t c = tid; c < k0; c += 1024) {
            double v = rhs[c];
            for (int m = 0; m < nb; ++m) v -= S[(k0 + m) * n + c] * rhs[k0 + m];
            rhs[c] = v;
        }
        __syncthreads();
    }
}

// ---- step ---------------------------------------------------------------------------------------------------------------------
template <int M>
__global__ void __launch_bounds__(128) ba_step_cameras_kernel(rb_ba_args a) {
    constexpr int NC = BaModel<M>::NC, CAM = BaModel<M>::CAM;
    pdl_wait();
    const int i = blockIdx.x * 128 + threadIdx.x;
    if (i >= a.num_images) return;
    const double* c = a.cams + (int64_t)i * CAM;
    double* o = a.cams_trial + (int64_t)i * CAM;
    const int fi = a.num_free > 0 ? a.free_index[i] : -1;
    if (fi < 0) {
        for (int j = 0; j < CAM; ++j) o[j] = c[j];
        a.cam_pred[i] = 0.0;
        return;
    }
    double d[NC], pred = 0.0;
#pragma unroll
    for (int j = 0; j < NC; ++j) d[j] = a.rhs[NC * (int64_t)fi + j];
#pragma unroll
    for (int j = 0; j < NC; ++j) pred += d[j] * (a.lambda * a.cam_sys[2 * NC * (int64_t)fi + NC + j] * d[j] - a.cam_sys[2 * NC * (int64_t)fi + j]);
    if constexpr (M == 0) {
        const double w[3] = {d[0], d[1], d[2]};
        double E[3][3];
        so3_exp(w, E);
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int m = 0; m < 3; ++m) o[3 * r + m] = E[r][0] * c[m] + E[r][1] * c[3 + m] + E[r][2] * c[6 + m];
#pragma unroll
        for (int j = 0; j < 3; ++j) o[9 + j] = c[9 + j] + d[3 + j];
        for (int j = 12; j < CAM; ++j) o[j] = c[j];
    } else {
        // a pinned parameter is copied, so it comes back bit-identical whatever its sign of zero
        const uint8_t* pin = a.pin + NC * (int64_t)fi;
        if (pin[0] && pin[1] && pin[2]) {
            for (int j = 0; j < 9; ++j) o[j] = c[j];
        } else {
            const double w[3] = {d[0], d[1], d[2]};
            double E[3][3];
            so3_exp(w, E);
#pragma unroll
            for (int r = 0; r < 3; ++r)
#pragma unroll
                for (int m = 0; m < 3; ++m) o[3 * r + m] = E[r][0] * c[m] + E[r][1] * c[3 + m] + E[r][2] * c[6 + m];
        }
#pragma unroll
        for (int j = 0; j < 3; ++j) o[9 + j] = pin[3 + j] ? c[9 + j] : c[9 + j] + d[3 + j];
        o[12] = pin[6] ? c[12] : c[12] + d[6];
        o[13] = c[13];
        o[14] = c[14];
        o[15] = pin[7] ? c[15] : c[15] + d[7];
    }
    a.cam_pred[i] = 0.5 * pred;
}

template <int M>
__global__ void __launch_bounds__(BA_THREADS) ba_step_points_kernel(rb_ba_args a) {
    constexpr int NC = BaModel<M>::NC;
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * BA_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * BA_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) {
        double* part = a.track_part + 3 * k;
        if (!a.track_ok[k]) {
            if (lane < 3) {
                a.X_trial[3 * k + lane] = a.X[3 * k + lane];
                part[lane] = 0.0;
            }
            continue;
        }
        const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
        const double* ts = a.track_sys + k * RB_BA_TRACK;
        double b[3] = {0.0, 0.0, 0.0};                    // sum_e W_e^T d_c
        if (a.num_free > 0) {
            for (int64_t e = base + lane; e < base + L; e += 32) {
                if (!ba_used(a, e)) continue;
                const int fj = a.free_index[a.elements[2 * e]];
                if (fj < 0) continue;
                const double* W = a.W + e * (3 * NC);
                const double* d = a.rhs + NC * (int64_t)fj;
#pragma unroll
                for (int m = 0; m < 3; ++m) {
                    if constexpr (M == 0) {
                        b[m] += W[m] * d[0] + W[3 + m] * d[1] + W[6 + m] * d[2] + W[9 + m] * d[3] + W[12 + m] * d[4] + W[15 + m] * d[5];
                    } else {
                        b[m] += W[m] * d[0] + W[3 + m] * d[1] + W[6 + m] * d[2] + W[9 + m] * d[3] + W[12 + m] * d[4] + W[15 + m] * d[5] +
                                W[18 + m] * d[6] + W[21 + m] * d[7];
                    }
                }
            }
            ba_warp_sum(b);
        }
        const double r0 = -ts[6] - b[0], r1 = -ts[7] - b[1], r2 = -ts[8] - b[2];
        const double dX[3] = {ts[0] * r0 + ts[1] * r1 + ts[2] * r2, ts[1] * r0 + ts[3] * r1 + ts[4] * r2, ts[2] * r0 + ts[4] * r1 + ts[5] * r2};
        double pred = 0.0;
#pragma unroll
        for (int m = 0; m < 3; ++m) pred += dX[m] * (a.lambda * ts[9 + m] * dX[m] - ts[6 + m]);
        const double X1[3] = {a.X[3 * k] + dX[0], a.X[3 * k + 1] + dX[1], a.X[3 * k + 2] + dX[2]};
        double s[2] = {0.0, 0.0};                         // trial cost, depths <= 0
        for (int64_t e = base + lane; e < base + L; e += 32) {
            if (!ba_used(a, e)) continue;
            int img;
            double ox, oy, ru, rv, depth, w;
            ba_keypoint(a, e, &img, &ox, &oy);
            const double* cam = a.cams_trial + (int64_t)img * BaModel<M>::CAM;
            ba_project<false, M>(cam, X1, ox, oy, &ru, &rv, &depth, nullptr, nullptr);
            s[0] += 0.5 * ba_rho(ru * ru + rv * rv, a.loss_scale2, &w);
            if constexpr (M == 0) s[1] += !(depth > 0.0);
            else s[1] += !(depth > 0.0) || !(cam[12] > 0.0);        // a trial focal length that is not > 0 rejects the step
        }
        ba_warp_sum(s);
        if (lane < 3) a.X_trial[3 * k + lane] = lane == 0 ? X1[0] : (lane == 1 ? X1[1] : X1[2]);
        if (lane == 0) {
            part[0] = s[0];
            part[1] = 0.5 * pred;
            part[2] = s[1];
        }
    }
}

// one CTA: the sum of v[j * stride] over j < n, each thread a contiguous chunk in order, then a fixed tree
__device__ double ba_block_sum(const double* __restrict__ v, int64_t n, int stride) {
    __shared__ double part[BA_SUM_THREADS];
    const int64_t per = (n + BA_SUM_THREADS - 1) / BA_SUM_THREADS;
    const int64_t b = min(n, (int64_t)threadIdx.x * per), e = min(n, b + per);
    double s = 0.0;
    for (int64_t j = b; j < e; ++j) s += v[j * stride];
    __syncthreads();
    part[threadIdx.x] = s;
    __syncthreads();
    for (int h = BA_SUM_THREADS / 2; h; h >>= 1) {
        if (threadIdx.x < h) part[threadIdx.x] += part[threadIdx.x + h];
        __syncthreads();
    }
    return part[0];
}

// STEP: result[0..2] = trial cost, pred, depths <= 0.  Otherwise result[0] = the cost of the linearization point.
template <bool STEP>
__global__ void __launch_bounds__(BA_SUM_THREADS) ba_sum_kernel(rb_ba_args a) {
    pdl_wait();
    if (!STEP) {
        const double F = ba_block_sum(a.track_sys + RB_BA_TRACK - 1, a.num_tracks, RB_BA_TRACK);
        if (threadIdx.x == 0) { a.result[0] = F; a.result[1] = 0.0; }
        return;
    }
    const double F = ba_block_sum(a.track_part, a.num_tracks, 3);
    const double pt = ba_block_sum(a.track_part + 1, a.num_tracks, 3);
    const double pc = ba_block_sum(a.cam_pred, a.num_images, 1);
    const double bad = ba_block_sum(a.track_part + 2, a.num_tracks, 3);
    if (threadIdx.x == 0) {
        a.result[0] = F;
        a.result[1] = pt + pc;
        a.result[2] = bad;
    }
}

template <int M>
__global__ void __launch_bounds__(BA_THREADS) ba_error_kernel(rb_ba_args a) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * BA_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * BA_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) {
        double s[2] = {0.0, 0.0};
        if (a.track_ok[k]) {
            const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
            const double X[3] = {a.X[3 * k], a.X[3 * k + 1], a.X[3 * k + 2]};
            for (int64_t e = base + lane; e < base + L; e += 32) {
                if (!ba_used(a, e)) continue;
                int img;
                double ox, oy, ru, rv, depth;
                ba_keypoint(a, e, &img, &ox, &oy);
                ba_project<false, M>(a.cams + (int64_t)img * BaModel<M>::CAM, X, ox, oy, &ru, &rv, &depth, nullptr, nullptr);
                s[0] += sqrt(ru * ru + rv * rv);
                s[1] += 1.0;
            }
            ba_warp_sum(s);
        }
        if (lane == 0) a.error[k] = s[1] > 0.0 ? s[0] / s[1] : 0.0;
    }
}

static int ba_check(const rb_ba_args* a, const char* what) {
    RB_REQUIRE(a && a->track_offsets && a->elements && a->kp_offsets && a->keypoints && a->track_ok && a->inlier && a->info && a->cams &&
               a->X, "%s: null argument", what);
    RB_REQUIRE(a->num_tracks > 0 && a->num_images > 0 && a->num_elements > 0 && a->num_elements < (1ll << 31) && a->num_rows > 0 &&
               a->num_free >= 0 && a->num_free <= a->num_images, "%s: bad sizes num_tracks=%d num_images=%d num_free=%d num_elements=%lld "
               "num_rows=%lld", what, a->num_tracks, a->num_images, a->num_free, (long long)a->num_elements, (long long)a->num_rows);
    RB_REQUIRE(a->loss_scale2 >= 0.0 && isfinite(a->loss_scale2) && a->lambda > 0.0 && isfinite(a->lambda), "%s: bad loss_scale2=%g or "
               "lambda=%g", what, a->loss_scale2, a->lambda);
    RB_REQUIRE(a->camera_model == 0 || a->camera_model == 1, "%s: bad camera_model=%d", what, a->camera_model);
    return 0;
}

// the folded system's arguments: 1 <= num_groups <= num_free and every buffer
static int ba_check_groups(const rb_ba_groups_args* a, const char* what) {
    RB_REQUIRE(a && a->num_free > 0 && a->num_groups > 0 && a->num_groups <= a->num_free && a->num_groups <= 65535, "%s: null argument "
               "or bad num_groups=%d (num_free=%d)", what, a ? a->num_groups : 0, a ? a->num_free : 0);
    RB_REQUIRE(a->group_offsets && a->group_members && a->group_pin && a->S && a->rhs && a->S_groups && a->rhs_groups && a->result,
               "%s: null argument", what);
    return 0;
}

// S = L L^T in place (lower triangle, order n), then rhs <- S^-1 rhs; a pivot that is not > 0 and finite sets result[3]
static int ba_cholesky_solve(double* S, int64_t n, double* rhs, double* result, cudaStream_t st) {
    for (int64_t k0 = 0; k0 < n; k0 += NB) {
        const int nb = (int)(n - k0 < NB ? n - k0 : NB);
        launch_pdl(ba_potrf_panel_kernel, dim3(1), dim3(256), 0, st, S, n, k0, nb, result);
        if (check_launch("ba_cholesky(panel)")) return 1;
        const int64_t rest = n - k0 - NB;
        if (rest <= 0) break;
        launch_pdl(ba_trsm_kernel, dim3((unsigned)((rest + 127) / 128)), dim3(128), 0, st, S, n, k0);
        if (check_launch("ba_cholesky(trsm)")) return 1;
        const unsigned tiles = (unsigned)((rest + NB - 1) / NB);
        launch_pdl(ba_syrk_kernel, dim3(tiles, tiles), dim3(256), 0, st, S, n, k0);
        if (check_launch("ba_cholesky(update)")) return 1;
    }
    launch_pdl(ba_potrs_kernel, dim3(1), dim3(1024), 0, st, (const double*)S, n, rhs);
    return check_launch("ba_cholesky(solve)");
}

static unsigned ba_track_grid(const rb_ba_args* a) { return grid1d(a->num_tracks, BA_WARPS, 64 * 1024); }

}  // namespace rb

using namespace rb;

extern "C" int romab200_ba_setup(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_setup")) return 1;
    RB_REQUIRE(a->elem_track && a->keys && a->keys_alt && a->hist && a->obs_offsets && a->obs, "ba_setup: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(a->info, 0, 2 * sizeof(int64_t), st) != cudaSuccess) return check_launch("ba_setup(info)");
    launch_pdl(ba_setup_kernel, dim3(ba_track_grid(a)), dim3(BA_THREADS), 0, st, *a);
    if (check_launch("ba_setup(check)")) return 1;
    const int bits = 32 - __builtin_clz((unsigned)a->num_images);              // images lie in [0, num_images]
    uint64_t* sorted = nullptr;
    if (radix_sort_hi32<RB_TRACKS_TILE>(a->keys, a->keys_alt, a->hist, a->num_elements, bits, st, "ba_setup(radix)", &sorted)) return 1;
    launch_pdl(ba_offsets_kernel, dim3(grid1d(a->num_elements, 256, 16 * 1024)), dim3(256), 0, st, *a, (const uint64_t*)sorted);
    return check_launch("ba_setup(offsets)");
}

extern "C" int romab200_ba_linearize(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_linearize")) return 1;
    RB_REQUIRE(a->W && a->track_sys && a->result, "ba_linearize: null argument");
    launch_pdl(a->camera_model ? ba_linearize_kernel<1> : ba_linearize_kernel<0>, dim3(ba_track_grid(a)), dim3(BA_THREADS), 0,
               (cudaStream_t)stream, *a);
    return check_launch("ba_linearize");
}

extern "C" int romab200_ba_cost(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_cost")) return 1;
    RB_REQUIRE(a->track_sys && a->result, "ba_cost: null argument");
    launch_pdl(ba_sum_kernel<false>, dim3(1), dim3(BA_SUM_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("ba_cost");
}

extern "C" int romab200_ba_cameras(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_cameras")) return 1;
    RB_REQUIRE(a->num_free > 0 && a->free_index && a->free_cams && (a->camera_model ? a->pin != nullptr : a->fixed_tx != nullptr) &&
               a->elem_track && a->obs_offsets && a->obs && a->W && a->track_sys && a->cam_sys && a->S && a->rhs,
               "ba_cameras: null argument or no free camera");
    launch_pdl(a->camera_model ? ba_cameras_kernel<1> : ba_cameras_kernel<0>, dim3(a->num_free), dim3(BA_CAM_THREADS), 0,
               (cudaStream_t)stream, *a);
    return check_launch("ba_cameras");
}

extern "C" int romab200_ba_cholesky(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_cholesky")) return 1;
    RB_REQUIRE(a->num_free > 0 && a->S && a->rhs && a->result, "ba_cholesky: null argument or no free camera");
    return ba_cholesky_solve(a->S, (a->camera_model ? 8 : 6) * (int64_t)a->num_free, a->rhs, a->result, (cudaStream_t)stream);
}

extern "C" int romab200_ba_fold(const rb_ba_groups_args* a, void* stream) {
    if (ba_check_groups(a, "ba_fold")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t F = a->num_free, np = 6 * F + 2 * (int64_t)a->num_groups;
    launch_pdl(ba_fold_kernel, dim3(grid1d(np * 6 * F, 256, 64 * 1024)), dim3(256), 0, st, *a);
    if (check_launch("ba_fold(poses)")) return 1;
    launch_pdl(ba_fold_groups_kernel, dim3(a->num_groups, a->num_groups), dim3(256), 0, st, *a);
    return check_launch("ba_fold(groups)");
}

extern "C" int romab200_ba_groups_cholesky(const rb_ba_groups_args* a, void* stream) {
    if (ba_check_groups(a, "ba_groups_cholesky")) return 1;
    return ba_cholesky_solve(a->S_groups, 6 * (int64_t)a->num_free + 2 * (int64_t)a->num_groups, a->rhs_groups, a->result,
                             (cudaStream_t)stream);
}

extern "C" int romab200_ba_unfold(const rb_ba_groups_args* a, void* stream) {
    if (ba_check_groups(a, "ba_unfold")) return 1;
    launch_pdl(ba_unfold_kernel, dim3(a->num_groups), dim3(128), 0, (cudaStream_t)stream, *a);
    return check_launch("ba_unfold");
}

extern "C" int romab200_ba_step(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_step")) return 1;
    RB_REQUIRE(a->cams_trial && a->X_trial && a->track_sys && a->cam_pred && a->track_part && a->result &&
               (a->num_free == 0 || (a->free_index && a->rhs && a->cam_sys && a->W && (!a->camera_model || a->pin))),
               "ba_step: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    launch_pdl(a->camera_model ? ba_step_cameras_kernel<1> : ba_step_cameras_kernel<0>, dim3((a->num_images + 127) / 128), dim3(128), 0,
               st, *a);
    if (check_launch("ba_step(cameras)")) return 1;
    launch_pdl(a->camera_model ? ba_step_points_kernel<1> : ba_step_points_kernel<0>, dim3(ba_track_grid(a)), dim3(BA_THREADS), 0, st,
               *a);
    if (check_launch("ba_step(points)")) return 1;
    launch_pdl(ba_sum_kernel<true>, dim3(1), dim3(BA_SUM_THREADS), 0, st, *a);
    return check_launch("ba_step(sum)");
}

extern "C" int romab200_ba_error(const rb_ba_args* a, void* stream) {
    if (ba_check(a, "ba_error")) return 1;
    RB_REQUIRE(a->error, "ba_error: null argument");
    launch_pdl(a->camera_model ? ba_error_kernel<1> : ba_error_kernel<0>, dim3(ba_track_grid(a)), dim3(BA_THREADS), 0,
               (cudaStream_t)stream, *a);
    return check_launch("ba_error");
}
