// Triangulation of feature tracks with known cameras (include/romab200.h): one warp per track.
//   check      the lanes check the track's element ids; a bad one sets RB_TRI_BAD_ID and leaves the track not ok.
//   hypotheses lane l takes the pairs h = l, l + 32, ...: a two-view DLT (cyclic Jacobi on the 4x4 A^T A), then its inliers among all
//              the track's observations; the best is the warp maximum of (count << 32) | ~h, so ties go to the smallest h.
//   refine     the multi-view DLT over the best hypothesis's inliers, then Gauss-Newton; the 4x4 DLT matrix and the 3x3 normal
//              equations are summed by every lane over its elements in order, then by a xor butterfly, so every lane holds the same
//              bits and every branch on them is uniform.
//   accept     the final inliers, and the lanes split the angle test over the inlier pairs.
// No float atomics and a fixed reduction order, so the result is bit-identical from run to run.
#include "geometry.cuh"

namespace rb {

constexpr int TRI_THREADS = 128;
constexpr int TRI_WARPS = TRI_THREADS / 32;
constexpr unsigned TRI_FULL = 0xffffffffu;

struct TriObs {
    double x, y;
    const double* cam;      // the image's row of the camera table (RB_TRI_CAM doubles)
    int img;
};

// element e (absolute index) whose ids have been checked
__device__ __forceinline__ TriObs tri_obs(const rb_tri_args& a, int64_t e) {
    const int i = a.elements[2 * e], id = a.elements[2 * e + 1];
    const int64_t r = a.kp_offsets[i] + id;
    return {(double)a.keypoints[2 * r], (double)a.keypoints[2 * r + 1], a.cameras + (int64_t)i * RB_TRI_CAM, i};
}

__device__ __forceinline__ double tri_depth(const double* c, const double (&X)[3]) {
    return c[12] * X[0] + c[13] * X[1] + c[14] * X[2] + c[15];
}

// the observation's image is not among the registered images: it is not an observation (its other camera entries are not read)
__device__ __forceinline__ bool tri_excluded(const TriObs& o) { return o.cam[19] != 0.0; }

// rule 4: depth > 0 and squared reprojection error <= max_error2; *err2 receives the squared error.  An observation of an excluded
// image is never an inlier.
__device__ __forceinline__ bool tri_inlier(const TriObs& o, const double (&X)[3], double max_error2, double* err2) {
    const double* c = o.cam;
    if (tri_excluded(o)) {
        *err2 = 0.0;
        return false;
    }
    const double p0 = c[0] * X[0] + c[1] * X[1] + c[2] * X[2] + c[3];
    const double p1 = c[4] * X[0] + c[5] * X[1] + c[6] * X[2] + c[7];
    const double p2 = c[8] * X[0] + c[9] * X[1] + c[10] * X[2] + c[11];
    const double du = p0 / p2 - o.x, dv = p1 / p2 - o.y;
    *err2 = du * du + dv * dv;
    return tri_depth(c, X) > 0.0 && *err2 <= max_error2;
}

// adds the two DLT rows x P^3 - P^1 and y P^3 - P^2 of an observation to the upper triangle of M
__device__ __forceinline__ void tri_dlt_add(const TriObs& o, double (&M)[4][4]) {
    const double* c = o.cam;
    double r0[4], r1[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        r0[j] = o.x * c[8 + j] - c[j];
        r1[j] = o.y * c[8 + j] - c[4 + j];
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = i; j < 4; ++j) M[i][j] += r0[i] * r0[j] + r1[i] * r1[j];
}

// the eigenvector of the smallest eigenvalue of the symmetric M (upper triangle given), dehomogenised; false if not finite
__device__ __forceinline__ bool tri_dlt_solve(double (&M)[4][4], double (&X)[3]) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < i; ++j) M[i][j] = M[j][i];
    double V[4][4];
    jacobi_eig<4>(M, V, 10);
    int k = 0;
    double mn = M[0][0];
#pragma unroll
    for (int i = 1; i < 4; ++i)
        if (M[i][i] < mn) { mn = M[i][i]; k = i; }
    double Q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) Q[i] = k == 0 ? V[i][0] : (k == 1 ? V[i][1] : (k == 2 ? V[i][2] : V[i][3]));
#pragma unroll
    for (int i = 0; i < 3; ++i) X[i] = Q[i] / Q[3];
    return isfinite(X[0]) && isfinite(X[1]) && isfinite(X[2]);
}

// pair h of the L (L - 1) / 2 pairs p < q in lexicographic order
__device__ __forceinline__ void tri_pair_of(int64_t h, int64_t L, int64_t* p, int64_t* q) {
    int64_t i = 0;
    while (h >= L - 1 - i) { h -= L - 1 - i; ++i; }
    *p = i;
    *q = i + 1 + h;
}

template <int N>
__device__ __forceinline__ void tri_warp_sum(double (&v)[N]) {
#pragma unroll
    for (int k = 0; k < N; ++k)
#pragma unroll
        for (int d = 16; d; d >>= 1) v[k] += __shfl_xor_sync(TRI_FULL, v[k], d);
}

// Gauss-Newton sums at X over the inliers of Xh (the best hypothesis's point): J^T J (00, 01, 02, 11, 12, 22), J^T r, the cost
__device__ __forceinline__ void tri_gn_sums(const rb_tri_args& a, int64_t base, int64_t L, int lane, const double (&Xh)[3],
                                            const double (&X)[3], double (&s)[10]) {
#pragma unroll
    for (int k = 0; k < 10; ++k) s[k] = 0.0;
    for (int64_t e = lane; e < L; e += 32) {
        const TriObs o = tri_obs(a, base + e);
        double err2;
        if (!tri_inlier(o, Xh, a.max_error2, &err2)) continue;
        const double* c = o.cam;
        const double p0 = c[0] * X[0] + c[1] * X[1] + c[2] * X[2] + c[3];
        const double p1 = c[4] * X[0] + c[5] * X[1] + c[6] * X[2] + c[7];
        const double p2 = c[8] * X[0] + c[9] * X[1] + c[10] * X[2] + c[11];
        const double u = p0 / p2, v = p1 / p2, ru = u - o.x, rv = v - o.y;
        double ju[3], jv[3];
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            ju[j] = (c[j] - u * c[8 + j]) / p2;
            jv[j] = (c[4 + j] - v * c[8 + j]) / p2;
        }
        s[0] += ju[0] * ju[0] + jv[0] * jv[0];
        s[1] += ju[0] * ju[1] + jv[0] * jv[1];
        s[2] += ju[0] * ju[2] + jv[0] * jv[2];
        s[3] += ju[1] * ju[1] + jv[1] * jv[1];
        s[4] += ju[1] * ju[2] + jv[1] * jv[2];
        s[5] += ju[2] * ju[2] + jv[2] * jv[2];
#pragma unroll
        for (int j = 0; j < 3; ++j) s[6 + j] += ju[j] * ru + jv[j] * rv;
        s[9] += ru * ru + rv * rv;
    }
    tri_warp_sum(s);
}

// the Gauss-Newton step: (J^T J) d = -J^T r by Cramer's rule; false if not finite
__device__ __forceinline__ bool tri_gn_step(const double (&s)[10], double (&d)[3]) {
    const double a00 = s[0], a01 = s[1], a02 = s[2], a11 = s[3], a12 = s[4], a22 = s[5];
    const double b0 = -s[6], b1 = -s[7], b2 = -s[8];
    const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
    const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
    const double det = a00 * c00 + a01 * c01 + a02 * c02;
    d[0] = (c00 * b0 + c01 * b1 + c02 * b2) / det;
    d[1] = (c01 * b0 + c11 * b1 + c12 * b2) / det;
    d[2] = (c02 * b0 + c12 * b1 + c22 * b2) / det;
    return isfinite(d[0]) && isfinite(d[1]) && isfinite(d[2]);
}

// largest-angle test of rule 6: is there an inlier pair in distinct images whose rays from X subtend >= min_angle?  Reads the
// inlier flags the warp has just written.
__device__ __forceinline__ bool tri_angle_ok(const rb_tri_args& a, int64_t base, int64_t L, int lane, const double (&X)[3]) {
    for (int64_t e = 0; e + 1 < L; ++e) {
        if (!a.inlier[base + e]) continue;
        const TriObs oe = tri_obs(a, base + e);
        const double ex = X[0] - oe.cam[16], ey = X[1] - oe.cam[17], ez = X[2] - oe.cam[18];
        bool found = false;
        for (int64_t f = e + 1 + lane; f < L; f += 32) {
            if (!a.inlier[base + f]) continue;
            const TriObs of = tri_obs(a, base + f);
            if (of.img == oe.img) continue;
            const double fx = X[0] - of.cam[16], fy = X[1] - of.cam[17], fz = X[2] - of.cam[18];
            const double cx = ey * fz - ez * fy, cy = ez * fx - ex * fz, cz = ex * fy - ey * fx;
            found |= atan2(sqrt(cx * cx + cy * cy + cz * cz), ex * fx + ey * fy + ez * fz) >= a.min_angle;
        }
        if (__any_sync(TRI_FULL, found)) return true;
    }
    return false;
}

__device__ void tri_track(const rb_tri_args& a, int k, int lane) {
    const int64_t base = a.track_offsets[k], L = a.track_offsets[k + 1] - base;
    bool bad = false;
    for (int64_t e = lane; e < L; e += 32) {
        const int i = a.elements[2 * (base + e)], id = a.elements[2 * (base + e) + 1];
        bad |= i < 0 || i >= a.num_images || id < 0 || id >= a.kp_offsets[i + 1] - a.kp_offsets[i];
    }
    bool ok = false;
    int count = 0;
    double X[3] = {0.0, 0.0, 0.0}, err_sum = 0.0;
    if (__any_sync(TRI_FULL, bad)) {
        if (lane == 0) atomicOr((unsigned long long*)a.info, (unsigned long long)RB_TRI_BAD_ID);
    } else {
        // rule 2-4: the hypotheses, lane l taking h = l, l + 32, ...
        const int64_t all = L * (L - 1) / 2;
        const bool every = all <= a.max_hypotheses;
        const int64_t H = every ? all : a.max_hypotheses;
        unsigned long long best = 0;
        double Xb[3] = {0.0, 0.0, 0.0};
        for (int64_t h = lane; h < H; h += 32) {
            int64_t p, q;
            if (every) {
                tri_pair_of(h, L, &p, &q);
            } else {
                int id[2];
                ransac_draw<2>(id, L, a.seed, [&](uint32_t s) { return make_uint4((uint32_t)h, s, (uint32_t)k, RB_TRI_CTR); });
                p = id[0];
                q = id[1];
            }
            const TriObs op = tri_obs(a, base + p), oq = tri_obs(a, base + q);
            if (op.img == oq.img || tri_excluded(op) || tri_excluded(oq)) continue;
            double M[4][4] = {}, Xh[3];
            tri_dlt_add(op, M);
            tri_dlt_add(oq, M);
            if (!tri_dlt_solve(M, Xh) || !(tri_depth(op.cam, Xh) > 0.0) || !(tri_depth(oq.cam, Xh) > 0.0)) continue;
            unsigned cnt = 0;
            for (int64_t e = 0; e < L; ++e) {
                double err2;
                cnt += tri_inlier(tri_obs(a, base + e), Xh, a.max_error2, &err2);
            }
            const unsigned long long key = (unsigned long long)cnt << 32 | (uint32_t)~(uint32_t)h;
            if (key > best) {
                best = key;
                Xb[0] = Xh[0]; Xb[1] = Xh[1]; Xb[2] = Xh[2];
            }
        }
#pragma unroll
        for (int d = 16; d; d >>= 1) best = max(best, (unsigned long long)__shfl_xor_sync(TRI_FULL, best, d));
        if ((best >> 32) >= 2) {
            const int owner = (int)(~(uint32_t)best & 31u);
#pragma unroll
            for (int i = 0; i < 3; ++i) Xb[i] = __shfl_sync(TRI_FULL, Xb[i], owner);
            // rule 5: the multi-view DLT over the hypothesis's inliers, then Gauss-Newton
            double M[4][4] = {};
            for (int64_t e = lane; e < L; e += 32) {
                const TriObs o = tri_obs(a, base + e);
                double err2;
                if (tri_inlier(o, Xb, a.max_error2, &err2)) tri_dlt_add(o, M);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = i; j < 4; ++j)
#pragma unroll
                    for (int d = 16; d; d >>= 1) M[i][j] += __shfl_xor_sync(TRI_FULL, M[i][j], d);
            if (!tri_dlt_solve(M, X)) { X[0] = Xb[0]; X[1] = Xb[1]; X[2] = Xb[2]; }
            double s[10];
            tri_gn_sums(a, base, L, lane, Xb, X, s);
#pragma unroll 1
            for (int it = 0; it < RB_TRI_GN_ITERS; ++it) {
                double d[3], s1[10];
                if (!tri_gn_step(s, d)) break;
                const double X1[3] = {X[0] + d[0], X[1] + d[1], X[2] + d[2]};
                tri_gn_sums(a, base, L, lane, Xb, X1, s1);
                if (!(s1[9] < s[9])) break;
                X[0] = X1[0]; X[1] = X1[1]; X[2] = X1[2];
#pragma unroll
                for (int j = 0; j < 10; ++j) s[j] = s1[j];
            }
            // rule 4 once more against the refined X: the flags are written now and read back by the angle test
            for (int64_t e0 = 0; e0 < L; e0 += 32) {
                const int64_t e = e0 + lane;
                bool in = false;
                if (e < L) {
                    double err2;
                    in = tri_inlier(tri_obs(a, base + e), X, a.max_error2, &err2);
                    if (in) err_sum += sqrt(err2);
                    a.inlier[base + e] = in;
                }
                count += __popc(__ballot_sync(TRI_FULL, in));
            }
            __syncwarp();
            ok = count >= 2 && tri_angle_ok(a, base, L, lane, X);
        }
    }
    double es[1] = {err_sum};
    tri_warp_sum(es);
    if (!ok)
        for (int64_t e = lane; e < L; e += 32) a.inlier[base + e] = 0;
    if (lane == 0) {
        a.ok[k] = ok;
        a.num_inliers[k] = ok ? count : 0;
        a.error[k] = ok ? es[0] / count : 0.0;
#pragma unroll
        for (int i = 0; i < 3; ++i) a.X[3 * (int64_t)k + i] = ok ? X[i] : 0.0;
    }
}

__global__ void __launch_bounds__(TRI_THREADS) tri_kernel(rb_tri_args a) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * TRI_WARPS;
    for (int64_t k = (int64_t)blockIdx.x * TRI_WARPS + (threadIdx.x >> 5); k < a.num_tracks; k += stride) tri_track(a, (int)k, lane);
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_triangulate(const rb_tri_args* a, void* stream) {
    RB_REQUIRE(a && a->track_offsets && a->elements && a->kp_offsets && a->keypoints && a->cameras && a->info && a->X && a->ok &&
               a->num_inliers && a->error && a->inlier, "triangulate: null argument");
    RB_REQUIRE(a->num_tracks > 0 && a->num_images > 0 && a->num_elements > 0 && a->num_elements < (1ll << 31) && a->num_rows > 0,
               "triangulate: bad sizes num_tracks=%d num_images=%d num_elements=%lld num_rows=%lld", a->num_tracks, a->num_images,
               (long long)a->num_elements, (long long)a->num_rows);
    RB_REQUIRE(a->max_hypotheses >= 1 && a->max_error2 > 0.0 && a->min_angle >= 0.0, "triangulate: bad max_hypotheses=%d, max_error2=%g "
               "or min_angle=%g", a->max_hypotheses, a->max_error2, a->min_angle);
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(a->info, 0, sizeof(int64_t), st) != cudaSuccess) return check_launch("triangulate(info)");
    launch_pdl(tri_kernel, dim3(grid1d(a->num_tracks, TRI_WARPS, 64 * 1024)), dim3(TRI_THREADS), 0, st, *a);
    return check_launch("triangulate");
}
