// Keypoint undistortion under SIMPLE_RADIAL cameras (include/romab200.h): a thread per keypoint, all in float64.  The image of a
// keypoint is found by binary search on kp_offsets.  The clamped count is an integer atomic, so it does not depend on the order.
#include "common.cuh"

namespace rb {

constexpr int UD_THREADS = 256;

__global__ void __launch_bounds__(UD_THREADS) undistort_kernel(rb_undistort_args a) {
    pdl_wait();
    const int64_t stride = (int64_t)gridDim.x * UD_THREADS;
    long long clamped = 0;
    for (int64_t r = blockIdx.x * (int64_t)UD_THREADS + threadIdx.x; r < a.num_rows; r += stride) {
        int lo = 0, hi = a.num_images;                        // the image i with kp_offsets[i] <= r < kp_offsets[i + 1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (a.kp_offsets[mid] <= r) lo = mid;
            else hi = mid;
        }
        const double* c = a.intrinsics + 4 * (int64_t)lo;
        const double f = c[0], cx = c[1], cy = c[2], k = c[3];
        const float u = a.keypoints[2 * r], v = a.keypoints[2 * r + 1];
        const double dx = (double)u - cx, dy = (double)v - cy;
        const double rd = sqrt(dx * dx + dy * dy) / f;
        if (k == 0.0 || rd == 0.0) {
            a.out[2 * r] = u;
            a.out[2 * r + 1] = v;
            continue;
        }
        double rho;
        if (k < 0.0 && rd >= 2.0 / (3.0 * sqrt(-3.0 * k))) {
            rho = 1.0 / sqrt(-3.0 * k);                        // the turning radius: no inverse at or beyond it
            ++clamped;
        } else {
            rho = rd;
#pragma unroll 1
            for (int it = 0; it < RB_UNDISTORT_ITERS; ++it) {
                const double step = (rho * (1.0 + k * rho * rho) - rd) / (1.0 + 3.0 * k * rho * rho);
                if (step == 0.0) break;
                rho -= step;
            }
        }
        const double s = rho / rd;
        a.out[2 * r] = (float)(cx + dx * s);
        a.out[2 * r + 1] = (float)(cy + dy * s);
    }
    for (int d = 16; d; d >>= 1) clamped += __shfl_xor_sync(0xffffffffu, clamped, d);
    if ((threadIdx.x & 31) == 0 && clamped) atomicAdd((unsigned long long*)a.clamped, (unsigned long long)clamped);
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_undistort_keypoints(const rb_undistort_args* a, void* stream) {
    RB_REQUIRE(a && a->kp_offsets && a->keypoints && a->intrinsics && a->out && a->clamped, "undistort_keypoints: null argument");
    RB_REQUIRE(a->num_images > 0 && a->num_rows >= 0, "undistort_keypoints: bad sizes num_images=%d num_rows=%lld", a->num_images,
               (long long)a->num_rows);
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(a->clamped, 0, sizeof(int64_t), st) != cudaSuccess) return check_launch("undistort_keypoints(clamped)");
    if (a->num_rows == 0) return 0;
    launch_pdl(undistort_kernel, dim3(grid1d(a->num_rows, UD_THREADS, 16 * 1024)), dim3(UD_THREADS), 0, st, *a);
    return check_launch("undistort_keypoints");
}
