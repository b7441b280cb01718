// Two-view initialisation (include/romab200.h): the statistics of each candidate pair's relative pose that decide whether it can
// start a reconstruction.  One CTA per candidate:
//   pass 1   a thread per masked match: the DLT point of the chirality test (dlt_two_view), the good-point tests, and its
//            triangulation angle into the per-point scratch (-1 when not good); the good count by an integer block sum;
//   select   the middle one or two good angles by a radix select on their bits: 8 passes of 8-bit digits, each a shared-memory
//            histogram (integer atomics, so the counts do not depend on their order) of the points whose higher digits match,
//            then thread 0 walks the 256 bins.
// No float atomics and fixed-order reductions only, so the result is bit-identical from run to run.
#include "geometry.cuh"

namespace rb {

constexpr int TV_THREADS = 256;
constexpr int TV_WARPS = TV_THREADS / 32;
constexpr double TV_DEG = 57.295779513082320876798154814105;   // 180 / pi

// the k-th smallest (0-based) non-negative value of angle[0, n), by bits; every thread must call it and gets the value
__device__ double tv_select(const double* angle, int64_t n, long long k, int* hist, unsigned long long* prefix_s, long long* k_s) {
    unsigned long long prefix = 0;
#pragma unroll 1
    for (int pass = 0; pass < 8; ++pass) {
        const int shift = 56 - 8 * pass;
        for (int d = threadIdx.x; d < 256; d += TV_THREADS) hist[d] = 0;
        __syncthreads();
        for (int64_t i = threadIdx.x; i < n; i += TV_THREADS) {
            const unsigned long long bits = (unsigned long long)__double_as_longlong(angle[i]);
            if ((bits >> 63) == 0 && (pass == 0 || (bits >> (shift + 8)) == prefix)) atomicAdd(&hist[(bits >> shift) & 255u], 1);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long below = 0;
            int d = 0;
            for (; d < 255 && k >= below + hist[d]; ++d) below += hist[d];
            *k_s = k - below;
            *prefix_s = (prefix << 8) | (unsigned long long)d;
        }
        __syncthreads();
        k = *k_s;
        prefix = *prefix_s;
        __syncthreads();
    }
    return __longlong_as_double((long long)prefix);
}

__global__ void __launch_bounds__(TV_THREADS) twoview_score_kernel(rb_twoview_args a) {
    pdl_wait();
    __shared__ int hist[256];
    __shared__ long long warp_cnt[TV_WARPS];
    __shared__ unsigned long long prefix_s;
    __shared__ long long k_s;
    const int b = blockIdx.x;
    const int64_t off = a.offsets[b], n = a.offsets[b + 1] - off;
    const double* R = a.R + (int64_t)b * 9;
    const double* t = a.t + (int64_t)b * 3;
    const double* K0 = a.K + (int64_t)b * 18;
    const double* K1 = K0 + 9;
    double* angle = a.angle + off;
    const bool ok = a.ok[b] != 0;
    long long cnt = 0;
    for (int64_t i = threadIdx.x; i < n; i += TV_THREADS) {
        double ang = -1.0;
        if (ok && a.mask[off + i]) {
            const double* p = a.xn + 4 * (off + i);
            double Q[4];
            dlt_two_view(R, t, p[0], p[1], p[2], p[3], Q);
            const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
            const double X1 = R[0] * X + R[1] * Y + R[2] * Z + t[0];
            const double Y1 = R[3] * X + R[4] * Y + R[5] * Z + t[1];
            const double Z1 = R[6] * X + R[7] * Y + R[8] * Z + t[2];
            bool good = Q[3] != 0.0 && isfinite(X) && isfinite(Y) && isfinite(Z) && Z > 0.0 && Z1 > 0.0;
            if (good) {
                const double* x0 = a.x0 + 2 * (off + i);
                const double* x1 = a.x1 + 2 * (off + i);
                const double w0 = K0[6] * X + K0[7] * Y + K0[8] * Z;
                const double u0 = (K0[0] * X + K0[1] * Y + K0[2] * Z) / w0 - x0[0];
                const double v0 = (K0[3] * X + K0[4] * Y + K0[5] * Z) / w0 - x0[1];
                const double w1 = K1[6] * X1 + K1[7] * Y1 + K1[8] * Z1;
                const double u1 = (K1[0] * X1 + K1[1] * Y1 + K1[2] * Z1) / w1 - x1[0];
                const double v1 = (K1[3] * X1 + K1[4] * Y1 + K1[5] * Z1) / w1 - x1[1];
                good = u0 * u0 + v0 * v0 <= a.max_error2 && u1 * u1 + v1 * v1 <= a.max_error2;
            }
            if (good) {
                // b = X - C1 with C1 = -R^T t
                const double bx = X + (R[0] * t[0] + R[3] * t[1] + R[6] * t[2]);
                const double by = Y + (R[1] * t[0] + R[4] * t[1] + R[7] * t[2]);
                const double bz = Z + (R[2] * t[0] + R[5] * t[1] + R[8] * t[2]);
                const double cx = Y * bz - Z * by, cy = Z * bx - X * bz, cz = X * by - Y * bx;
                ang = atan2(sqrt(cx * cx + cy * cy + cz * cz), X * bx + Y * by + Z * bz) * TV_DEG;
                ++cnt;
            }
        }
        angle[i] = ang;
    }
#pragma unroll
    for (int d = 16; d; d >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, d);
    if ((threadIdx.x & 31) == 0) warp_cnt[threadIdx.x >> 5] = cnt;
    __syncthreads();                                     // also makes the scratch angles visible to the whole CTA
    long long good = 0;
#pragma unroll
    for (int w = 0; w < TV_WARPS; ++w) good += warp_cnt[w];
    double median = 0.0;
    if (good > 0) {
        const double lo = tv_select(angle, n, (good - 1) / 2, hist, &prefix_s, &k_s);
        median = lo;
        if (good % 2 == 0) median = (lo + tv_select(angle, n, good / 2, hist, &prefix_s, &k_s)) / 2.0;
    }
    if (threadIdx.x == 0) {
        a.num_good[b] = good;
        a.median_angle[b] = median;
        a.forward[b] = fabs(t[2]);
    }
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_twoview_score(const rb_twoview_args* a, void* stream) {
    RB_REQUIRE(a && a->offsets && a->x0 && a->x1 && a->xn && a->mask && a->K && a->R && a->t && a->ok && a->angle && a->num_good &&
                   a->median_angle && a->forward, "twoview_score: null argument");
    RB_REQUIRE(a->batch > 0, "twoview_score: batch %d < 1", a->batch);
    RB_REQUIRE(a->max_error2 > 0.0, "twoview_score: max_error2 %g <= 0", a->max_error2);
    launch_pdl(twoview_score_kernel, dim3(a->batch), dim3(TV_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("twoview_score");
}
