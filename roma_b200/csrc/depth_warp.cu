// Depth-based ground-truth warps and the MegaDepth dense metric on the device: `warp_kpts` / `get_gt_warp`
// (romatch/utils/utils.py:325-454) and `MegadepthDenseBenchmark.geometric_dist` (romatch/benchmarks/megadepth_dense_benchmark.py:17-42).
// The reference casts both depth maps, the points, the pose and the intrinsics to float64 and runs about 25 eager kernels over
// [B, L, 3] float64 temporaries; the arithmetic is one pass: two 4-tap depth gathers, ~150 float64 operations and a compare per point.
// Here one thread owns a point (grid-stride over the points of a pair, grid.y = pair):
//   dw_warp_point   the one statement of the geometry (include/romab200.h), float64 with every operation rounded separately
//                   (__dadd_rn / __dmul_rn / __ddiv_rn are never contracted), so the three kernels agree bit for bit on a point;
//   camera          inv(K0) by the adjugate, [R | t] and K1 of the pair, set up by thread 0 of every CTA in shared memory;
//   warp_kpts / gt_warp / dense_dist   differ only in where a point comes from and what is written;
//   dense_dist      also leaves one partial per CTA (float64 sum of gd and four counts over its valid pixels: shuffles inside a
//                   warp, then warp 0 over the warps, a fixed tree), and dw_finish_kernel adds the partials of a pair and then
//                   the pairs in index order.  No atomics: the sums do not depend on timing.
// Depth maps (float32 as MegaDepth stores them, or float64) and points are converted in registers; nothing is copied.
#include "common.cuh"

namespace rb {

constexpr int DW_THREADS = 256;

__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double dot3(const double* r, double x, double y, double z) {
    return dadd(dadd(dmul(r[0], x), dmul(r[1], y)), dmul(r[2], z));
}

struct DwCamera { double Kinv[9], R[9], t[3], K1[9]; };

// the arguments the three entry points share, with the depth type resolved
template <typename TD>
struct DwViews {
    const TD* depth0; const TD* depth1; int h0, w0, h1, w1;
    const double* T; int T_rows; const double* K0; const double* K1;
    int mode; double thr;
};
template <typename TD, typename A>
inline DwViews<TD> dw_views(const A* a, int mode) {
    return {(const TD*)a->depth0, (const TD*)a->depth1, a->h0, a->w0, a->h1, a->w1, a->T, a->T_rows, a->K0, a->K1, mode, a->rel_threshold};
}

__device__ __forceinline__ void dw_camera(DwCamera& c, const double* __restrict__ K0, const double* __restrict__ T, int T_rows,
                                          const double* __restrict__ K1, int b) {
    const double* k = K0 + 9 * (int64_t)b;
    const double c00 = dsub(dmul(k[4], k[8]), dmul(k[5], k[7])), c01 = dsub(dmul(k[5], k[6]), dmul(k[3], k[8])),
                 c02 = dsub(dmul(k[3], k[7]), dmul(k[4], k[6]));
    const double det = dadd(dadd(dmul(k[0], c00), dmul(k[1], c01)), dmul(k[2], c02));
    c.Kinv[0] = ddiv(c00, det);
    c.Kinv[1] = ddiv(dsub(dmul(k[2], k[7]), dmul(k[1], k[8])), det);
    c.Kinv[2] = ddiv(dsub(dmul(k[1], k[5]), dmul(k[2], k[4])), det);
    c.Kinv[3] = ddiv(c01, det);
    c.Kinv[4] = ddiv(dsub(dmul(k[0], k[8]), dmul(k[2], k[6])), det);
    c.Kinv[5] = ddiv(dsub(dmul(k[2], k[3]), dmul(k[0], k[5])), det);
    c.Kinv[6] = ddiv(c02, det);
    c.Kinv[7] = ddiv(dsub(dmul(k[1], k[6]), dmul(k[0], k[7])), det);
    c.Kinv[8] = ddiv(dsub(dmul(k[0], k[4]), dmul(k[1], k[3])), det);
    const double* t = T + (int64_t)b * T_rows * 4;
    for (int r = 0; r < 3; ++r) {
        for (int j = 0; j < 3; ++j) c.R[3 * r + j] = t[4 * r + j];
        c.t[r] = t[4 * r + 3];
    }
    for (int j = 0; j < 9; ++j) c.K1[j] = K1[9 * (int64_t)b + j];
}

// F.grid_sample of a one-channel float64 map at the normalised (x, y): zero padding, align_corners=False.  A NaN position gives NaN.
template <typename TD>
__device__ __forceinline__ double dw_sample(const TD* __restrict__ map, int h, int w, double x, double y, int mode) {
    const double ix = dmul(dsub(dmul(dadd(x, 1.0), (double)w), 1.0), 0.5), iy = dmul(dsub(dmul(dadd(y, 1.0), (double)h), 1.0), 0.5);
    if (ix != ix || iy != iy) return __longlong_as_double(0x7ff8000000000000ll);
    if (mode == 1) {
        const double xn = nearbyint(ix), yn = nearbyint(iy);
        return xn >= 0.0 && xn < (double)w && yn >= 0.0 && yn < (double)h ? (double)map[(int64_t)yn * w + (int64_t)xn] : 0.0;
    }
    const double x0 = floor(ix), y0 = floor(iy), x1 = dadd(x0, 1.0), y1 = dadd(y0, 1.0);
    const double wx0 = dsub(x1, ix), wx1 = dsub(ix, x0), wy0 = dsub(y1, iy), wy1 = dsub(iy, y0);
    const bool inx0 = x0 >= 0.0 && x0 < (double)w, inx1 = x1 >= 0.0 && x1 < (double)w;      // in float64: no overflow for far-away points
    const bool iny0 = y0 >= 0.0 && y0 < (double)h, iny1 = y1 >= 0.0 && y1 < (double)h;
    double out = 0.0;
    if (iny0 && inx0) out = dadd(out, dmul((double)map[(int64_t)y0 * w + (int64_t)x0], dmul(wx0, wy0)));
    if (iny0 && inx1) out = dadd(out, dmul((double)map[(int64_t)y0 * w + (int64_t)x1], dmul(wx1, wy0)));
    if (iny1 && inx0) out = dadd(out, dmul((double)map[(int64_t)y1 * w + (int64_t)x0], dmul(wx0, wy1)));
    if (iny1 && inx1) out = dadd(out, dmul((double)map[(int64_t)y1 * w + (int64_t)x1], dmul(wx1, wy1)));
    return out;
}

// steps 1-5 of include/romab200.h for the point (x, y) of pair b: the warped normalised point in (ox, oy), returns valid
template <typename TD>
__device__ __forceinline__ bool dw_warp_point(const DwViews<TD>& v, const DwCamera& c, int b, double x, double y, double& ox, double& oy) {
    const double d0 = dw_sample(v.depth0 + (int64_t)b * v.h0 * v.w0, v.h0, v.w0, x, y, v.mode);
    const double px = dmul(dmul((double)v.w0, dadd(x, 1.0)), 0.5), py = dmul(dmul((double)v.h0, dadd(y, 1.0)), 0.5);
    const double hx = dmul(px, d0), hy = dmul(py, d0), hz = d0;
    const double X = dot3(c.Kinv, hx, hy, hz), Y = dot3(c.Kinv + 3, hx, hy, hz), Z = dot3(c.Kinv + 6, hx, hy, hz);
    const double cx = dadd(dot3(c.R, X, Y, Z), c.t[0]), cy = dadd(dot3(c.R + 3, X, Y, Z), c.t[1]), cz = dadd(dot3(c.R + 6, X, Y, Z), c.t[2]);
    const double den = dadd(dot3(c.K1 + 6, cx, cy, cz), 1e-4);
    const double u = ddiv(dot3(c.K1, cx, cy, cz), den), w = ddiv(dot3(c.K1 + 3, cx, cy, cz), den);
    const bool covisible = u > 0.0 && u < (double)(v.w1 - 1) && w > 0.0 && w < (double)(v.h1 - 1);
    ox = dsub(ddiv(dmul(2.0, u), (double)v.w1), 1.0);
    oy = dsub(ddiv(dmul(2.0, w), (double)v.h1), 1.0);
    const double d1 = dw_sample(v.depth1 + (int64_t)b * v.h1 * v.w1, v.h1, v.w1, ox, oy, v.mode);
    const bool consistent = fabs(ddiv(dsub(d1, cz), d1)) < v.thr;
    return d0 != 0.0 && covisible && consistent;
}

#define DW_CAMERA(v)                                                        \
    __shared__ DwCamera cam;                                                \
    const int b = blockIdx.y;                                               \
    if (threadIdx.x == 0) dw_camera(cam, (v).K0, (v).T, (v).T_rows, (v).K1, b); \
    __syncthreads()

template <typename TD, typename TP>
__global__ void __launch_bounds__(DW_THREADS) dw_warp_kpts_kernel(DwViews<TD> v, const TP* __restrict__ kpts, int64_t L, double* __restrict__ warped,
                                                                  uint8_t* __restrict__ valid) {
    pdl_wait();
    DW_CAMERA(v);
    for (int64_t i = (int64_t)blockIdx.x * DW_THREADS + threadIdx.x; i < L; i += (int64_t)gridDim.x * DW_THREADS) {
        const int64_t p = (int64_t)b * L + i;
        double ox, oy;
        const bool ok = dw_warp_point(v, cam, b, (double)kpts[2 * p], (double)kpts[2 * p + 1], ox, oy);
        reinterpret_cast<double2*>(warped)[p] = make_double2(ox, oy);
        valid[p] = ok;
    }
}

template <typename TD>
__global__ void __launch_bounds__(DW_THREADS) dw_gt_warp_kernel(DwViews<TD> v, const float* __restrict__ grid_x, const float* __restrict__ grid_y, int H,
                                                                int W, double* __restrict__ x2, float* __restrict__ prob) {
    pdl_wait();
    DW_CAMERA(v);
    const int64_t n = (int64_t)H * W;
    for (int64_t i = (int64_t)blockIdx.x * DW_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * DW_THREADS) {
        const int64_t p = (int64_t)b * n + i;
        double ox, oy;
        const bool ok = dw_warp_point(v, cam, b, (double)grid_x[i % W], (double)grid_y[i / W], ox, oy);
        reinterpret_cast<double2*>(x2)[p] = make_double2(ox, oy);
        prob[p] = ok ? 1.f : 0.f;
    }
}

// sum and counts over the 32 lanes of a warp, every lane receiving the result; a butterfly, so the order of the additions is fixed
__device__ __forceinline__ void dw_warp_reduce(double& sum, int (&cnt)[4]) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        sum = dadd(sum, __shfl_xor_sync(0xffffffffu, sum, o));
#pragma unroll
        for (int k = 0; k < 4; ++k) cnt[k] += __shfl_xor_sync(0xffffffffu, cnt[k], o);
    }
}

// (W (x + 1)) / 2 in float32, every operation rounded: the harness converts its float32 prediction to pixels in float32
__device__ __forceinline__ double dw_pixel_f32(int size, float x) { return (double)__fmul_rn(__fmul_rn((float)size, __fadd_rn(x, 1.f)), 0.5f); }

template <typename TD>
__global__ void __launch_bounds__(DW_THREADS) dw_dense_dist_kernel(DwViews<TD> v, rb_dense_geometric_dist_args a) {
    pdl_wait();
    DW_CAMERA(v);
    const int64_t n = (int64_t)a.H * a.W;
    double sum = 0.0;
    int cnt[4] = {0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * DW_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * DW_THREADS) {
        const float* m = a.dense_matches + b * a.dm_sb + (i / a.W) * a.dm_sy + (i % a.W) * a.dm_sx;
        double ox, oy;
        const bool ok = dw_warp_point(v, cam, b, (double)m[0], (double)m[a.dm_sc], ox, oy);
        const double gx = dmul(dmul((double)a.W, dadd(ox, 1.0)), 0.5), gy = dmul(dmul((double)a.H, dadd(oy, 1.0)), 0.5);
        const double dx = dsub(dw_pixel_f32(a.W, m[2 * a.dm_sc]), gx), dy = dsub(dw_pixel_f32(a.H, m[3 * a.dm_sc]), gy);
        const double gd = sqrt(dadd(dmul(dx, dx), dmul(dy, dy)));
        const int64_t p = (int64_t)b * n + i;
        a.gd[p] = ok ? gd : __longlong_as_double(0x7ff8000000000000ll);
        a.prob[p] = ok ? 1.f : 0.f;
        if (ok) {
            sum = dadd(sum, gd);
            cnt[0] += 1; cnt[1] += gd < 1.0; cnt[2] += gd < 3.0; cnt[3] += gd < 5.0;
        }
    }
    // CTA partial in a fixed order: butterfly inside each warp, then warp 0 over the warps
    __shared__ double s_sum[DW_THREADS / 32];
    __shared__ int s_cnt[DW_THREADS / 32][4];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    dw_warp_reduce(sum, cnt);
    if (lane == 0) {
        s_sum[wid] = sum;
        for (int k = 0; k < 4; ++k) s_cnt[wid][k] = cnt[k];
    }
    __syncthreads();
    if (wid != 0) return;
    const bool has = lane < DW_THREADS / 32;
    sum = has ? s_sum[lane] : 0.0;
    for (int k = 0; k < 4; ++k) cnt[k] = has ? s_cnt[lane][k] : 0;
    dw_warp_reduce(sum, cnt);
    if (lane == 0) {
        const int64_t q = (int64_t)b * RB_DEPTH_WARP_MAX_CTAS + blockIdx.x;
        a.partial_sum[q] = sum;
        for (int k = 0; k < 4; ++k) a.partial_cnt[4 * q + k] = cnt[k];
    }
}

// one CTA: per pair the `ctas` partials (thread t takes t, t + 256, ..., then a shared-memory tree), then the pairs in index order
__global__ void __launch_bounds__(DW_THREADS) dw_finish_kernel(rb_dense_geometric_dist_args a, int ctas) {
    pdl_wait();
    __shared__ double s_sum[DW_THREADS];
    __shared__ long long s_cnt[DW_THREADS][4];
    double tot = 0.0;
    long long tot_cnt[4] = {0, 0, 0, 0};
    for (int b = 0; b < a.batch; ++b) {
        double sum = 0.0;
        long long cnt[4] = {0, 0, 0, 0};
        for (int j = threadIdx.x; j < ctas; j += DW_THREADS) {
            const int64_t q = (int64_t)b * RB_DEPTH_WARP_MAX_CTAS + j;
            sum = dadd(sum, a.partial_sum[q]);
            for (int k = 0; k < 4; ++k) cnt[k] += a.partial_cnt[4 * q + k];
        }
        s_sum[threadIdx.x] = sum;
        for (int k = 0; k < 4; ++k) s_cnt[threadIdx.x][k] = cnt[k];
        __syncthreads();
        for (int o = DW_THREADS / 2; o > 0; o >>= 1) {
            if (threadIdx.x < o) {
                s_sum[threadIdx.x] = dadd(s_sum[threadIdx.x], s_sum[threadIdx.x + o]);
                for (int k = 0; k < 4; ++k) s_cnt[threadIdx.x][k] += s_cnt[threadIdx.x + o][k];
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            a.pair_sum[b] = s_sum[0];
            tot = dadd(tot, s_sum[0]);
            for (int k = 0; k < 4; ++k) {
                a.pair_cnt[4 * b + k] = s_cnt[0][k];
                tot_cnt[k] += s_cnt[0][k];
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        // torch's mean on the device: the sum times the reciprocal of the count, in the tensor's type (0 * inf = NaN when empty)
        const float inv = __fdiv_rn(1.f, (float)tot_cnt[0]);
        for (int k = 0; k < 3; ++k) a.pck[k] = __fmul_rn((float)tot_cnt[k + 1], inv);
        a.epe[0] = dmul(tot, ddiv(1.0, (double)tot_cnt[0]));
    }
}

template <typename A>
static int dw_check(const A* a, const char* what) {
    RB_REQUIRE(a && a->depth0 && a->depth1 && a->T && a->K0 && a->K1, "%s: null argument", what);
    RB_REQUIRE(a->batch > 0 && a->batch <= 65535, "%s: batch %d outside 1 .. 65535", what, a->batch);
    RB_REQUIRE(a->h0 > 0 && a->w0 > 0 && a->h1 > 0 && a->w1 > 0, "%s: empty depth map (%dx%d, %dx%d)", what, a->h0, a->w0, a->h1, a->w1);
    RB_REQUIRE(a->T_rows == 3 || a->T_rows == 4, "%s: T must be [batch, 3 or 4, 4] (got %d rows)", what, a->T_rows);
    return 0;
}
static int dw_check_mode(int mode, const char* what) {
    RB_REQUIRE(mode == 0 || mode == 1, "%s: interpolation mode %d unsupported (0 bilinear, 1 nearest)", what, mode);
    return 0;
}
static dim3 dw_grid(int64_t points, int batch) { return dim3(grid1d(points, DW_THREADS, RB_DEPTH_WARP_MAX_CTAS), batch); }

}  // namespace rb

using namespace rb;

extern "C" int romab200_warp_kpts(const rb_warp_kpts_args* a, void* stream) {
    if (dw_check(a, "warp_kpts") || dw_check_mode(a->mode, "warp_kpts")) return 1;
    RB_REQUIRE(a->L >= 0 && (a->L == 0 || (a->kpts && a->warped && a->valid)), "warp_kpts: null argument");
    return with_dtype<float, double>(a->depth_dtype, "warp_kpts", [&](auto td) {
        using TD = typename decltype(td)::type;
        return with_dtype<float, double>(a->kpts_dtype, "warp_kpts", [&](auto tp) {
            using TP = typename decltype(tp)::type;
            if (a->L == 0) return 0;
            launch_pdl(dw_warp_kpts_kernel<TD, TP>, dw_grid(a->L, a->batch), dim3(DW_THREADS), 0, (cudaStream_t)stream, dw_views<TD>(a, a->mode),
                       (const TP*)a->kpts, a->L, a->warped, a->valid);
            return check_launch("warp_kpts");
        });
    });
}

extern "C" int romab200_gt_warp(const rb_gt_warp_args* a, void* stream) {
    if (dw_check(a, "gt_warp") || dw_check_mode(a->mode, "gt_warp")) return 1;
    RB_REQUIRE(a->grid_x && a->grid_y && a->x2 && a->prob, "gt_warp: null argument");
    RB_REQUIRE(a->H > 0 && a->W > 0, "gt_warp: empty grid %dx%d", a->H, a->W);
    return with_dtype<float, double>(a->depth_dtype, "gt_warp", [&](auto td) {
        using TD = typename decltype(td)::type;
        launch_pdl(dw_gt_warp_kernel<TD>, dw_grid((int64_t)a->H * a->W, a->batch), dim3(DW_THREADS), 0, (cudaStream_t)stream, dw_views<TD>(a, a->mode),
                   a->grid_x, a->grid_y, a->H, a->W, a->x2, a->prob);
        return check_launch("gt_warp");
    });
}

extern "C" int romab200_dense_geometric_dist(const rb_dense_geometric_dist_args* a, void* stream) {
    if (dw_check(a, "dense_geometric_dist")) return 1;
    RB_REQUIRE(a->dense_matches && a->gd && a->prob && a->partial_sum && a->partial_cnt && a->pair_sum && a->pair_cnt && a->pck && a->epe,
               "dense_geometric_dist: null argument");
    RB_REQUIRE(a->H > 0 && a->W > 0, "dense_geometric_dist: empty map %dx%d", a->H, a->W);
    return with_dtype<float, double>(a->depth_dtype, "dense_geometric_dist", [&](auto td) {
        using TD = typename decltype(td)::type;
        const dim3 grid = dw_grid((int64_t)a->H * a->W, a->batch);
        launch_pdl(dw_dense_dist_kernel<TD>, grid, dim3(DW_THREADS), 0, (cudaStream_t)stream, dw_views<TD>(a, 0), *a);
        if (check_launch("dense_geometric_dist")) return 1;
        launch_pdl(dw_finish_kernel, dim3(1), dim3(DW_THREADS), 0, (cudaStream_t)stream, *a, (int)grid.x);
        return check_launch("dense_geometric_dist(finish)");
    });
}
