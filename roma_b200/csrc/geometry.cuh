// Helpers shared by the two-view geometry estimators (pose.cu, homography.cu, fundamental.cu).
#pragma once
#include "common.cuh"

namespace rb {

// q^M as M - 1 products from the left: q * q * ... * q
template <int M>
__device__ __forceinline__ double pow_left(double q) {
    if constexpr (M == 1) return q;
    else return pow_left<M - 1>(q) * q;
}

// Whether OpenCV's loop draws hypothesis h for a pair of n points: it needs M points, draws once when there are exactly M,
// and stops at max_iters.  After the first round a caller also skips the pairs whose state row no longer says running.
template <int M>
__device__ __forceinline__ bool ransac_drawn(int64_t n, int64_t h, int max_iters) {
    return n >= M && h < max_iters && (n > M || h == 0);
}

// M distinct indices in [0, n): the four words of philox4x32_10(ctr(sub), seed) for sub = 0, 1, ... in order, index
// (w * n) >> 32, repeats skipped.  Only the counter differs between the estimators' streams (include/romab200.h).
template <int M, typename CtrOf>
__device__ __forceinline__ void ransac_draw(int (&id)[M], int64_t n, uint64_t seed, CtrOf ctr) {
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    int got = 0;
    for (uint32_t sub = 0; got < M; ++sub) {
        const uint4 r = philox4x32_10(ctr(sub), k0, k1);
        const uint32_t words[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int v = (int)(((uint64_t)words[q] * (uint64_t)n) >> 32);
            bool dup = false;
#pragma unroll
            for (int k = 0; k < M; ++k) dup |= (k < got && id[k] == v);
            if (!dup && got < M) {
#pragma unroll
                for (int k = 0; k < M; ++k)
                    if (k == got) id[k] = v;
                ++got;
            }
        }
    }
}

// Visits the points of score slice blockIdx.y (per_split points each, n in all) in index order: the CTA of THREADS threads
// stages them through `tile`, load(j) giving point j, and every thread with act set calls visit(p) on each.  Every thread must
// call it.
template <int THREADS, typename T, int TILE, typename Load, typename Visit>
__device__ __forceinline__ void ransac_scan(T (&tile)[TILE], int64_t n, int per_split, bool act, Load load, Visit visit) {
    const int64_t j0 = (int64_t)blockIdx.y * per_split, j1 = min(n, j0 + per_split);
    for (int64_t t0 = j0; t0 < j1; t0 += TILE) {
        const int m = (int)min((int64_t)TILE, j1 - t0);
        __syncthreads();
        for (int j = threadIdx.x; j < m; j += THREADS) tile[j] = load(t0 + j);
        __syncthreads();
        if (act) {
#pragma unroll 4
            for (int j = 0; j < m; ++j) visit(tile[j]);
        }
    }
}

// Inliers of this thread's model among the points of score slice blockIdx.y; inlier(p) tests one.  The count is meaningful
// for the threads with act set.  Integer counts: the slices add up in any order.
template <int THREADS, typename T, int TILE, typename Load, typename Inlier>
__device__ __forceinline__ int ransac_count(T (&tile)[TILE], int64_t n, int per_split, bool act, Load load, Inlier inlier) {
    int cnt = 0;
    ransac_scan<THREADS>(tile, n, per_split, act, load, [&](const T& p) { cnt += inlier(p); });
    return cnt;
}

// Score slices of one pair: one per points_per_split points, at least 1 and at most max_splits
static inline int ransac_splits(int64_t max_n, int points_per_split, int max_splits) {
    const int64_t s = (max_n + points_per_split - 1) / points_per_split;
    return s < 1 ? 1 : (s > max_splits ? max_splits : (int)s);
}

// The checks every RANSAC stage shares: pair layout, state rows, batch size and the round within max_iters
template <typename Args>
static int ransac_check(const Args* a, const char* what, int max_batch, int round_size) {
    RB_REQUIRE(a && a->offsets && a->state, "%s: null argument", what);
    RB_REQUIRE(a->batch > 0 && a->batch <= max_batch, "%s: batch %d outside [1, %d]", what, a->batch, max_batch);
    RB_REQUIRE(a->max_n >= 0 && a->max_n < (1ll << 31), "%s: bad max_n %lld", what, (long long)a->max_n);
    RB_REQUIRE(a->max_iters > 0 && a->round >= 0 && (int64_t)a->round * round_size < a->max_iters, "%s: round %d outside max_iters %d",
               what, a->round, a->max_iters);
    return 0;
}

// cv::RANSACUpdateNumIters(p, ep, model_points, maxIters), with (1 - ep)^model_points as products from the left
template <int MODEL_POINTS>
__device__ __forceinline__ int ransac_update_num_iters(double p, double ep, int max_iters) {
    p = fmin(fmax(p, 0.0), 1.0);
    ep = fmin(fmax(ep, 0.0), 1.0);
    double num = fmax(1.0 - p, 2.2250738585072014e-308);
    const double q = 1.0 - ep;
    double denom = 1.0 - pow_left<MODEL_POINTS>(q);
    if (denom < 2.2250738585072014e-308) return 0;
    num = log(num);
    denom = log(denom);
    return denom >= 0.0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
}

// cyclic Jacobi on a symmetric N x N matrix: on return the columns of V are eigenvectors, diag(A) the eigenvalues
template <int N, typename MatA, typename MatV>
__device__ __forceinline__ void jacobi_eig(MatA& A, MatV& V, int sweeps) {
#pragma unroll
    for (int i = 0; i < N; ++i)
#pragma unroll
        for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
#pragma unroll 1
    for (int sw = 0; sw < sweeps; ++sw) {
#pragma unroll
        for (int p = 0; p < N - 1; ++p)
#pragma unroll
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq;
                }
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
                }
#pragma unroll
                for (int k = 0; k < N; ++k) {
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
                }
            }
    }
}

// jacobi_eig on a matrix in shared memory, run by one warp: lane k updates entry k of the two columns, then of the two rows of each
// rotation (and of V's two columns), the same operations on every element in the same order as jacobi_eig, without N^3 unrolled code
template <int N>
__device__ __forceinline__ void jacobi_eig_warp(double (*A)[N], double (*V)[N], int sweeps) {
    static_assert(N <= 32, "jacobi_eig_warp: one lane per index");
    const int k = threadIdx.x & 31;
    if (k < N)
        for (int j = 0; j < N; ++j) V[k][j] = k == j ? 1.0 : 0.0;
    __syncwarp();
#pragma unroll 1
    for (int sw = 0; sw < sweeps; ++sw) {
#pragma unroll 1
        for (int p = 0; p < N - 1; ++p)
#pragma unroll 1
            for (int q = p + 1; q < N; ++q) {
                const double apq = A[p][q];
                if (apq == 0.0) continue;
                const double theta = (A[q][q] - A[p][p]) / (2.0 * apq);
                const double tt = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
                __syncwarp();
                if (k < N) {
                    const double akp = A[k][p], akq = A[k][q];
                    A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq;
                }
                __syncwarp();
                if (k < N) {
                    const double apk = A[p][k], aqk = A[q][k];
                    A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
                    const double vkp = V[k][p], vkq = V[k][q];
                    V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
                }
                __syncwarp();
            }
    }
}

// Linear (DLT) triangulation of normalised (x0, y0) <-> (x1, y1) with P0 = [I | 0], P1 = [R | t] (R row-major): the eigenvector of
// the smallest eigenvalue of the 4x4 A^T A (10 Jacobi sweeps), i.e. the right singular vector of the smallest singular value of A,
// as homogeneous Q.  recoverPose's chirality test (pose.cu) and the two-view statistics (twoview.cu) share it.
__device__ __forceinline__ void dlt_two_view(const double* R, const double* t, double x0, double y0, double x1, double y1,
                                             double (&Q)[4]) {
    const double rows[4][4] = {{-1.0, 0.0, x0, 0.0},
                               {0.0, -1.0, y0, 0.0},
                               {x1 * R[6] - R[0], x1 * R[7] - R[1], x1 * R[8] - R[2], x1 * t[2] - t[0]},
                               {y1 * R[6] - R[3], y1 * R[7] - R[4], y1 * R[8] - R[5], y1 * t[2] - t[1]}};
    double M[4][4], V[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) M[i][j] = rows[0][i] * rows[0][j] + rows[1][i] * rows[1][j] + rows[2][i] * rows[2][j] + rows[3][i] * rows[3][j];
    jacobi_eig<4>(M, V, 10);
    int k = 0;
    double mn = M[0][0];
#pragma unroll
    for (int i = 1; i < 4; ++i)
        if (M[i][i] < mn) { mn = M[i][i]; k = i; }
#pragma unroll
    for (int i = 0; i < 4; ++i) Q[i] = k == 0 ? V[i][0] : (k == 1 ? V[i][1] : (k == 2 ? V[i][2] : V[i][3]));
}

// SIMPLE_RADIAL undistortion of a radius (include/romab200.h, keypoint undistortion rules 2 and 4): rho with rho (1 + k rho^2) =
// rd by Newton from rho = rd, or the turning radius 1 / sqrt(-3 k) with clamped set when k < 0 and rd is at or beyond its image.
// The caller handles k = 0 and rd = 0.  camera.cu (keypoints) and dense.cu (dense warps) share it.
__device__ __forceinline__ double radial_undistort_rho(double rd, double k, bool& clamped) {
    if (k < 0.0 && rd >= 2.0 / (3.0 * sqrt(-3.0 * k))) {
        clamped = true;
        return 1.0 / sqrt(-3.0 * k);
    }
    clamped = false;
    double rho = rd;
#pragma unroll 1
    for (int it = 0; it < RB_UNDISTORT_ITERS; ++it) {
        const double step = (rho * (1.0 + k * rho * rho) - rd) / (1.0 + 3.0 * k * rho * rho);
        if (step == 0.0) break;
        rho -= step;
    }
    return rho;
}

// 3x3 SVD M = sum_k s_k u_k v_k^T from cyclic Jacobi on M^T M: v[k] is the k-th right singular vector by descending singular
// value with det [v0 v1 v2] = +1, u[k] = M v_k / s_k and s[k] = |M v_k| for k < 2, u[2] = u[0] x u[1] (M row-major)
__device__ __forceinline__ void svd3(const double* M, double (&u)[3][3], double (&v)[3][3], double (&s)[2]) {
    double A[3][3], V[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) A[i][j] = M[i] * M[j] + M[3 + i] * M[3 + j] + M[6 + i] * M[6 + j];   // M^T M
    jacobi_eig<3>(A, V, 12);
    // order the eigenvalues descending: columns i0 (largest), i1, i2 (smallest)
    double e0 = A[0][0], e1 = A[1][1], e2 = A[2][2];
    int i0 = 0, i1 = 1, i2 = 2;
    if (e1 > e0) { const double t = e0; e0 = e1; e1 = t; const int k = i0; i0 = i1; i1 = k; }
    if (e2 > e1) { const double t = e1; e1 = e2; e2 = t; const int k = i1; i1 = i2; i2 = k; }
    if (e1 > e0) { const double t = e0; e0 = e1; e1 = t; const int k = i0; i0 = i1; i1 = k; }
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        v[0][i] = i0 == 0 ? V[i][0] : (i0 == 1 ? V[i][1] : V[i][2]);
        v[1][i] = i1 == 0 ? V[i][0] : (i1 == 1 ? V[i][1] : V[i][2]);
        v[2][i] = i2 == 0 ? V[i][0] : (i2 == 1 ? V[i][1] : V[i][2]);
    }
    const double dv = v[0][0] * (v[1][1] * v[2][2] - v[1][2] * v[2][1]) - v[0][1] * (v[1][0] * v[2][2] - v[1][2] * v[2][0]) +
                      v[0][2] * (v[1][0] * v[2][1] - v[1][1] * v[2][0]);
    if (dv < 0.0) { v[2][0] = -v[2][0]; v[2][1] = -v[2][1]; v[2][2] = -v[2][2]; }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        double nn = 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) { u[k][i] = M[3 * i] * v[k][0] + M[3 * i + 1] * v[k][1] + M[3 * i + 2] * v[k][2]; nn += u[k][i] * u[k][i]; }
        nn = sqrt(nn);
        s[k] = nn;
#pragma unroll
        for (int i = 0; i < 3; ++i) u[k][i] /= nn;
    }
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
}

// Sums of v[0..N) over a CTA of THREADS threads: per-warp butterfly, then the warp partials added in warp order.  Fixed order,
// so the result does not depend on the batch.  Leaves the totals in tot[0..N) (visible to every thread on return).
template <int N, int THREADS, int M, int W>
__device__ __forceinline__ void cta_sum(double (&v)[M], double (*red)[W], double* tot) {
    static_assert(N <= M && N <= W && N <= THREADS, "cta_sum: too many sums");
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < N; ++k) {
#pragma unroll
        for (int d = 16; d; d >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], d);
    }
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) red[w][k] = v[k];
    }
    __syncthreads();
    if (threadIdx.x < N) {
        double s = 0.0;
        for (int q = 0; q < THREADS / 32; ++q) s += red[q][threadIdx.x];
        tot[threadIdx.x] = s;
    }
    __syncthreads();
}

}  // namespace rb
