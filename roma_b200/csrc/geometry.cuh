// Helpers shared by the two-view geometry estimators (pose.cu, homography.cu).
#pragma once
#include "common.cuh"

namespace rb {

// q^M as M - 1 products from the left: q * q * ... * q
template <int M>
__device__ __forceinline__ double pow_left(double q) {
    if constexpr (M == 1) return q;
    else return pow_left<M - 1>(q) * q;
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

}  // namespace rb
