// Dense reconstruction (include/romab200.h): per-image depth maps triangulated from symmetric dense warps, and their multi-view
// fusion into a point cloud.
//   triangulate  pack      the listed images' (score, source) -> 64-bit keys in place, so the maps accumulate across calls;
//                elements  a thread per (pair-half, pixel), grid.y = pair-half: the CTA's relative pose and the two cameras are set
//                          up once in shared memory (as depth_warp.cu does); rules 1-5 in float64, dlt_two_view for the point, an
//                          integer atomicMax of (certainty bits << 32 | ~g) per grid pixel, the element's depth to scratch, and the
//                          reason counts by warp reductions into per-CTA partials;
//                counts    one thread per (pair, reason) adds the partials in a fixed order.
//   resolve      winners   each accepted element whose key won writes its depth (one writer per pixel: keys are unique);
//                unpack    keys -> (score, source).
//   fuse         count / emit  one CTA per RB_DENSE_TILE pixels of one image, one pixel per thread: rules F1-F3 over the image's
//                          neighbours, then a block-wide rank of the emitted pixels in pixel order; count writes the tile's total and
//                          scans the tiles (scan_counts_kernel), emit writes at the scanned offsets.
// No float atomics: the maps, the counts and the cloud are bit-identical from run to run and for any chunking of the pairs.
#include "geometry.cuh"

namespace rb {

constexpr int DN_THREADS = 256;
constexpr int DN_WARPS = DN_THREADS / 32;
static_assert(RB_DENSE_TILE == DN_THREADS, "a fusion tile is one pixel per thread");

// camera table columns (include/romab200.h)
constexpr int CK = 0, CKI = 9, CR = 18, CT = 27, CF = 30;

// normalised coordinates of the pixel (x, y) (rule 4); false when the radial undistortion clamps it
__device__ __forceinline__ bool dn_normalise(const double* cam, int radial, double x, double y, double& a, double& b) {
    if (!radial) {
        const double* Ki = cam + CKI;
        const double h0 = Ki[0] * x + Ki[1] * y + Ki[2], h1 = Ki[3] * x + Ki[4] * y + Ki[5], h2 = Ki[6] * x + Ki[7] * y + Ki[8];
        a = h0 / h2;
        b = h1 / h2;
        return true;
    }
    const double f = cam[CF], cx = cam[CF + 1], cy = cam[CF + 2], k = cam[CF + 3];
    const double dx = x - cx, dy = y - cy;
    const double rd = sqrt(dx * dx + dy * dy) / f;
    double s = 1.0;
    if (k != 0.0 && rd != 0.0) {
        bool clamped;
        s = radial_undistort_rho(rd, k, clamped) / rd;
        if (clamped) return false;
    }
    a = dx * s / f;
    b = dy * s / f;
    return true;
}

// pixel of the camera-frame point (X, Y, Z)
__device__ __forceinline__ void dn_project(const double* cam, int radial, double X, double Y, double Z, double& u, double& v) {
    if (!radial) {
        const double* K = cam + CK;
        const double p0 = K[0] * X + K[1] * Y + K[2] * Z, p1 = K[3] * X + K[4] * Y + K[5] * Z, p2 = K[6] * X + K[7] * Y + K[8] * Z;
        u = p0 / p2;
        v = p1 / p2;
        return;
    }
    const double f = cam[CF], cx = cam[CF + 1], cy = cam[CF + 2], k = cam[CF + 3];
    const double x = X / Z, y = Y / Z, d = 1.0 + k * (x * x + y * y);
    u = f * d * x + cx;
    v = f * d * y + cy;
}

// the 64-bit key of an element: larger certainty first, then smaller g
__device__ __forceinline__ unsigned long long dn_key(float cert, int64_t g) {
    return ((unsigned long long)__float_as_uint(cert) << 32) | (unsigned long long)(~(uint32_t)g);
}

struct DnPair {
    double cg[RB_DENSE_CAM], cm[RB_DENSE_CAM];
    double R[9], t[3], C[3];        // relative pose grid -> match camera, and the match camera's centre in the grid frame
    int gi, mi, Hg, Wg, Hm, Wm, reg;
};

// thread 0 of the CTA: the pair-half blockIdx.y's cameras and relative pose
__device__ __forceinline__ void dn_setup(DnPair& s, const rb_dense_tri_args& a) {
    const int row = blockIdx.y >> 1, half = blockIdx.y & 1;
    const int64_t k = (int64_t)a.first_pair + row;
    s.gi = (int)a.pairs[2 * k + half];
    s.mi = (int)a.pairs[2 * k + 1 - half];
    s.Hg = a.image_sizes[2 * s.gi]; s.Wg = a.image_sizes[2 * s.gi + 1];
    s.Hm = a.image_sizes[2 * s.mi]; s.Wm = a.image_sizes[2 * s.mi + 1];
    s.reg = a.registered[s.gi] && a.registered[s.mi];
    for (int q = 0; q < RB_DENSE_CAM; ++q) {
        s.cg[q] = a.cameras[(int64_t)s.gi * RB_DENSE_CAM + q];
        s.cm[q] = a.cameras[(int64_t)s.mi * RB_DENSE_CAM + q];
    }
    const double* Rg = s.cg + CR; const double* Rm = s.cm + CR;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) s.R[3 * i + j] = Rm[3 * i] * Rg[3 * j] + Rm[3 * i + 1] * Rg[3 * j + 1] + Rm[3 * i + 2] * Rg[3 * j + 2];
    for (int i = 0; i < 3; ++i)
        s.t[i] = s.cm[CT + i] - (s.R[3 * i] * s.cg[CT] + s.R[3 * i + 1] * s.cg[CT + 1] + s.R[3 * i + 2] * s.cg[CT + 2]);
    for (int i = 0; i < 3; ++i) s.C[i] = -(s.R[i] * s.t[0] + s.R[3 + i] * s.t[1] + s.R[6 + i] * s.t[2]);
}

// rules 1-5 for the element of pixel i of the CTA's pair-half: its reason, and its depth when accepted
__device__ __forceinline__ int dn_element(const DnPair& s, const rb_dense_tri_args& a, int64_t i, float& cert, float& depth) {
    const int row = blockIdx.y >> 1, half = blockIdx.y & 1;
    const int r = (int)(i / a.W), c = (int)(i % a.W);
    const int64_t e = ((int64_t)row * a.H + r) * (2 * (int64_t)a.W) + (int64_t)half * a.W + c;
    cert = a.certainty[e];
    const float2 uv = reinterpret_cast<const float2*>(a.warp + 4 * e)[1 - half];
    if (!(cert > a.min_certainty) || !isfinite(cert) || !isfinite(uv.x) || !isfinite(uv.y)) return 1;
    if (!(fabsf(uv.x) <= 1.f && fabsf(uv.y) <= 1.f)) return 2;
    if (!s.reg) return 3;
    const double xg = (double)s.Wg * (c + 0.5) / a.W, yg = (double)s.Hg * (r + 0.5) / a.H;
    const double xm = (double)__fmul_rn((float)s.Wm * 0.5f, __fadd_rn(uv.x, 1.f));
    const double ym = (double)__fmul_rn((float)s.Hm * 0.5f, __fadd_rn(uv.y, 1.f));
    double ag, bg, am, bm;
    if (!dn_normalise(s.cg, a.radial, xg, yg, ag, bg) || !dn_normalise(s.cm, a.radial, xm, ym, am, bm)) return 4;
    double Q[4];
    dlt_two_view(s.R, s.t, ag, bg, am, bm, Q);
    const double X = Q[0] / Q[3], Y = Q[1] / Q[3], Z = Q[2] / Q[3];
    const double Xm = s.R[0] * X + s.R[1] * Y + s.R[2] * Z + s.t[0];
    const double Ym = s.R[3] * X + s.R[4] * Y + s.R[5] * Z + s.t[1];
    const double Zm = s.R[6] * X + s.R[7] * Y + s.R[8] * Z + s.t[2];
    if (Q[3] == 0.0 || !(Z > 0.0) || !(Zm > 0.0)) return 5;
    double u, v;
    dn_project(s.cg, a.radial, X, Y, Z, u, v);
    const double eg = (u - xg) * (u - xg) + (v - yg) * (v - yg);
    dn_project(s.cm, a.radial, Xm, Ym, Zm, u, v);
    const double em = (u - xm) * (u - xm) + (v - ym) * (v - ym);
    if (!(eg <= a.max_error2) || !(em <= a.max_error2)) return 6;
    const double bx = X - s.C[0], by = Y - s.C[1], bz = Z - s.C[2];
    const double cx = Y * bz - Z * by, cy = Z * bx - X * bz, cz = X * by - Y * bx;
    const double ang = atan2(sqrt(cx * cx + cy * cy + cz * cz), X * bx + Y * by + Z * bz);
    if (!(ang >= a.min_angle)) return 7;
    depth = __double2float_rn(Z);
    return 0;
}

// score, source -> key (PACK) or back (!PACK) over the listed images, grid.y = list entry
template <bool PACK>
__global__ void __launch_bounds__(DN_THREADS) dn_pack_kernel(rb_dense_tri_args a) {
    pdl_wait();
    const int64_t n = (int64_t)a.H * a.W;
    const int64_t base = (int64_t)a.images[blockIdx.y] * n;
    for (int64_t i = (int64_t)blockIdx.x * DN_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * DN_THREADS) {
        const int64_t p = base + i;
        if (PACK) {
            const int64_t src = a.source[p];
            a.source[p] = src < 0 ? 0 : (int64_t)dn_key(a.score[p], src);
        } else {
            const unsigned long long key = (unsigned long long)a.source[p];
            a.source[p] = key == 0 ? -1 : (int64_t)(uint32_t)~(uint32_t)key;
            a.score[p] = key == 0 ? 0.f : __uint_as_float((uint32_t)(key >> 32));
        }
    }
}

__global__ void __launch_bounds__(DN_THREADS) dn_triangulate_kernel(rb_dense_tri_args a) {
    pdl_wait();
    __shared__ DnPair s;
    __shared__ int red[DN_WARPS][RB_DENSE_REASONS];
    if (threadIdx.x == 0) dn_setup(s, a);
    __syncthreads();
    const int64_t n = (int64_t)a.H * a.W;
    const int64_t g = 2 * ((int64_t)a.first_pair + (blockIdx.y >> 1)) + (blockIdx.y & 1);
    int cnt[RB_DENSE_REASONS] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int64_t i = (int64_t)blockIdx.x * DN_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * DN_THREADS) {
        float cert, depth = 0.f;
        const int reason = dn_element(s, a, i, cert, depth);
#pragma unroll
        for (int q = 0; q < RB_DENSE_REASONS; ++q) cnt[q] += reason == q;
        a.elem_depth[(int64_t)blockIdx.y * n + i] = depth;
        if (reason == 0) atomicMax((unsigned long long*)&a.source[(int64_t)s.gi * n + i], dn_key(cert, g));
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < RB_DENSE_REASONS; ++q) {
        const int v = __reduce_add_sync(0xffffffffu, cnt[q]);
        if (lane == 0) red[wid][q] = v;
    }
    __syncthreads();
    if (threadIdx.x < RB_DENSE_REASONS) {
        int tot = 0;
        for (int w = 0; w < DN_WARPS; ++w) tot += red[w][threadIdx.x];
        a.partial[((int64_t)blockIdx.y * RB_DENSE_MAX_CTAS + blockIdx.x) * RB_DENSE_REASONS + threadIdx.x] = tot;
    }
}

// one thread per (row, reason): both halves' partials in CTA order, added to the pair's row
__global__ void __launch_bounds__(DN_THREADS) dn_counts_kernel(rb_dense_tri_args a, int ctas) {
    pdl_wait();
    const int t = blockIdx.x * DN_THREADS + threadIdx.x;
    if (t >= a.chunk * RB_DENSE_REASONS) return;
    const int row = t / RB_DENSE_REASONS, q = t % RB_DENSE_REASONS;
    int64_t sum = 0;
    for (int h = 0; h < 2; ++h)
        for (int b = 0; b < ctas; ++b) sum += a.partial[((int64_t)(2 * row + h) * RB_DENSE_MAX_CTAS + b) * RB_DENSE_REASONS + q];
    a.pair_counts[((int64_t)a.first_pair + row) * RB_DENSE_REASONS + q] += sum;
}

__global__ void __launch_bounds__(DN_THREADS) dn_resolve_kernel(rb_dense_tri_args a) {
    pdl_wait();
    const int row = blockIdx.y >> 1, half = blockIdx.y & 1;
    const int64_t k = (int64_t)a.first_pair + row, g = 2 * k + half;
    const int gi = (int)a.pairs[2 * k + half];
    const int64_t n = (int64_t)a.H * a.W;
    for (int64_t i = (int64_t)blockIdx.x * DN_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * DN_THREADS) {
        const float d = a.elem_depth[(int64_t)blockIdx.y * n + i];
        if (!(d > 0.f)) continue;
        const int r = (int)(i / a.W), c = (int)(i % a.W);
        const float cert = a.certainty[((int64_t)row * a.H + r) * (2 * (int64_t)a.W) + (int64_t)half * a.W + c];
        const int64_t p = (int64_t)gi * n + i;
        if ((unsigned long long)a.source[p] == dn_key(cert, g)) a.depth[p] = d;
    }
}

// ---- fusion ----------------------------------------------------------------------------------------------------------------------

struct DnFuse {
    bool emit;
    int views;
    double P[3];
};

// F1: the world point of grid pixel (r, c) of image `img` at depth d; false when its position is clamped
__device__ __forceinline__ bool dn_backproject(const rb_dense_fuse_args& a, const double* cam, int img, int r, int c, double d,
                                               double& px, double& py, double (&Xw)[3]) {
    px = (double)a.image_sizes[2 * img + 1] * (c + 0.5) / a.W;
    py = (double)a.image_sizes[2 * img] * (r + 0.5) / a.H;
    double na, nb;
    if (!dn_normalise(cam, a.radial, px, py, na, nb)) return false;
    const double q[3] = {d * na - cam[CT], d * nb - cam[CT + 1], d - cam[CT + 2]};
    const double* R = cam + CR;
#pragma unroll
    for (int i = 0; i < 3; ++i) Xw[i] = R[i] * q[0] + R[3 + i] * q[1] + R[6 + i] * q[2];
    return true;
}

__device__ __forceinline__ void dn_to_cam(const double* cam, const double (&X)[3], double (&Y)[3]) {
    const double* R = cam + CR;
#pragma unroll
    for (int i = 0; i < 3; ++i) Y[i] = R[3 * i] * X[0] + R[3 * i + 1] * X[1] + R[3 * i + 2] * X[2] + cam[CT + i];
}

// F1-F3 for pixel i of image img (cam: its camera row)
__device__ __forceinline__ DnFuse dn_fuse_pixel(const rb_dense_fuse_args& a, const double* cam, int img, int64_t i) {
    DnFuse out{false, 0, {0.0, 0.0, 0.0}};
    const int64_t n = (int64_t)a.H * a.W;
    const float d = a.depth[(int64_t)img * n + i];
    if (!(d > 0.f)) return out;
    const int r = (int)(i / a.W), c = (int)(i % a.W);
    double px, py, X[3];
    if (!dn_backproject(a, cam, img, r, c, (double)d, px, py, X)) return out;
    double S[3] = {X[0], X[1], X[2]};
    int agree = 0;
    bool lower = false;
    for (int64_t e = a.nbr_offsets[img]; e < a.nbr_offsets[img + 1]; ++e) {
        const int j = a.nbrs[e];
        const double* cj = a.cameras + (int64_t)j * RB_DENSE_CAM;
        double Xj[3];
        dn_to_cam(cj, X, Xj);
        if (!(Xj[2] > 0.0)) continue;
        double u, v;
        dn_project(cj, a.radial, Xj[0], Xj[1], Xj[2], u, v);
        const double gc = floor(u * a.W / a.image_sizes[2 * j + 1]), gr = floor(v * a.H / a.image_sizes[2 * j]);
        if (!(gc >= 0.0 && gc < (double)a.W && gr >= 0.0 && gr < (double)a.H)) continue;
        const int qc = (int)gc, qr = (int)gr;
        const float dq = a.depth[(int64_t)j * n + (int64_t)qr * a.W + qc];
        if (!(dq > 0.f) || !(fabs((double)dq - Xj[2]) <= a.max_depth_error * Xj[2])) continue;
        double qx, qy, Y[3], Yi[3];
        if (!dn_backproject(a, cj, j, qr, qc, (double)dq, qx, qy, Y)) continue;
        dn_to_cam(cam, Y, Yi);
        if (!(Yi[2] > 0.0)) continue;
        dn_project(cam, a.radial, Yi[0], Yi[1], Yi[2], u, v);
        if (!((u - px) * (u - px) + (v - py) * (v - py) <= a.max_reproj_error2)) continue;
        ++agree;
        lower |= j < img;
        S[0] += Y[0]; S[1] += Y[1]; S[2] += Y[2];
    }
    out.emit = agree >= a.min_num_views - 1 && !lower;
    out.views = 1 + agree;
#pragma unroll
    for (int q = 0; q < 3; ++q) out.P[q] = S[q] / out.views;
    return out;
}

template <bool EMIT>
__global__ void __launch_bounds__(DN_THREADS) dn_fuse_kernel(rb_dense_fuse_args a, int tiles) {
    pdl_wait();
    __shared__ double cam[RB_DENSE_CAM];
    __shared__ int wsum[DN_WARPS];
    const int img = blockIdx.x / tiles;
    const int64_t i = (int64_t)(blockIdx.x % tiles) * DN_THREADS + threadIdx.x;
    if (threadIdx.x < RB_DENSE_CAM) cam[threadIdx.x] = a.cameras[(int64_t)img * RB_DENSE_CAM + threadIdx.x];
    __syncthreads();
    const int64_t n = (int64_t)a.H * a.W;
    DnFuse f{false, 0, {0.0, 0.0, 0.0}};
    if (i < n && a.registered[img]) f = dn_fuse_pixel(a, cam, img, i);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const unsigned ball = __ballot_sync(0xffffffffu, f.emit);
    if (lane == 0) wsum[wid] = __popc(ball);
    __syncthreads();
    if (!EMIT) {
        if (threadIdx.x == 0) {
            int64_t tot = 0;
            for (int w = 0; w < DN_WARPS; ++w) tot += wsum[w];
            a.tile_scan[blockIdx.x] = tot;
        }
        return;
    }
    if (!f.emit) return;
    int64_t o = a.tile_scan[blockIdx.x] + __popc(ball & ((1u << lane) - 1u));
    for (int w = 0; w < wid; ++w) o += wsum[w];
    for (int q = 0; q < 3; ++q) a.points[3 * o + q] = f.P[q];
    const int r = (int)(i / a.W), c = (int)(i % a.W);
    uint8_t rgb[3] = {128, 128, 128};
    if (a.colors) {
        const int64_t Hc = a.color_sizes[2 * img], Wc = a.color_sizes[2 * img + 1];
        const int64_t cr = (2 * (int64_t)r + 1) * Hc / (2 * (int64_t)a.H), cc = (2 * (int64_t)c + 1) * Wc / (2 * (int64_t)a.W);
        const uint8_t* px = a.colors + a.color_offsets[img] + 3 * (cr * Wc + cc);
        rgb[0] = px[0]; rgb[1] = px[1]; rgb[2] = px[2];
    }
    for (int q = 0; q < 3; ++q) a.rgb[3 * o + q] = rgb[q];
    a.image[o] = img;
    a.pixel[o] = i;
    a.num_views[o] = f.views;
    a.point_score[o] = a.score[(int64_t)img * n + i];
}

static int dn_tri_check(const rb_dense_tri_args* a, const char* what) {
    RB_REQUIRE(a && a->pairs && a->warp && a->certainty && a->image_sizes && a->cameras && a->registered && a->images && a->depth &&
               a->score && a->source && a->elem_depth && a->partial && a->pair_counts, "%s: null argument", what);
    RB_REQUIRE(a->num_pairs > 0 && a->num_images > 0 && a->H > 0 && a->W > 0 && a->num_list > 0 && a->num_list <= 65535,
               "%s: bad sizes num_pairs=%d num_images=%d H=%d W=%d num_list=%d", what, a->num_pairs, a->num_images, a->H, a->W, a->num_list);
    RB_REQUIRE(a->chunk > 0 && 2 * (int64_t)a->chunk <= 65535 && a->first_pair >= 0 && (int64_t)a->first_pair + a->chunk <= a->num_pairs,
               "%s: rows %d .. %d + %d outside the %d pairs", what, a->first_pair, a->first_pair, a->chunk, a->num_pairs);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_dense_triangulate(const rb_dense_tri_args* a, void* stream) {
    if (dn_tri_check(a, "dense_triangulate")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = (int64_t)a->H * a->W;
    launch_pdl(dn_pack_kernel<true>, dim3(grid1d(n, DN_THREADS, 1024), a->num_list), dim3(DN_THREADS), 0, st, *a);
    if (check_launch("dense_triangulate(pack)")) return 1;
    const unsigned ctas = grid1d(n, DN_THREADS, RB_DENSE_MAX_CTAS);
    launch_pdl(dn_triangulate_kernel, dim3(ctas, 2 * a->chunk), dim3(DN_THREADS), 0, st, *a);
    if (check_launch("dense_triangulate")) return 1;
    launch_pdl(dn_counts_kernel, dim3(grid1d((int64_t)a->chunk * RB_DENSE_REASONS, DN_THREADS, 1 << 20)), dim3(DN_THREADS), 0, st, *a,
               (int)ctas);
    return check_launch("dense_triangulate(counts)");
}

extern "C" int romab200_dense_resolve(const rb_dense_tri_args* a, void* stream) {
    if (dn_tri_check(a, "dense_resolve")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t n = (int64_t)a->H * a->W;
    launch_pdl(dn_resolve_kernel, dim3(grid1d(n, DN_THREADS, RB_DENSE_MAX_CTAS), 2 * a->chunk), dim3(DN_THREADS), 0, st, *a);
    if (check_launch("dense_resolve")) return 1;
    launch_pdl(dn_pack_kernel<false>, dim3(grid1d(n, DN_THREADS, 1024), a->num_list), dim3(DN_THREADS), 0, st, *a);
    return check_launch("dense_resolve(unpack)");
}

static int dn_fuse_check(const rb_dense_fuse_args* a, const char* what, int64_t& tiles) {
    RB_REQUIRE(a && a->image_sizes && a->cameras && a->registered && a->nbr_offsets && a->nbrs && a->depth && a->score && a->tile_scan,
               "%s: null argument", what);
    RB_REQUIRE(!a->colors || (a->color_offsets && a->color_sizes), "%s: colors without color_offsets / color_sizes", what);
    RB_REQUIRE(a->num_images > 0 && a->H > 0 && a->W > 0, "%s: bad sizes num_images=%d H=%d W=%d", what, a->num_images, a->H, a->W);
    tiles = ((int64_t)a->H * a->W + RB_DENSE_TILE - 1) / RB_DENSE_TILE;
    RB_REQUIRE(tiles * a->num_images < (1ll << 31) - 1, "%s: %lld tiles, at most 2^31 - 2 are supported", what,
               (long long)(tiles * a->num_images));
    return 0;
}

extern "C" int romab200_dense_fuse_count(const rb_dense_fuse_args* a, void* stream) {
    int64_t tiles;
    if (dn_fuse_check(a, "dense_fuse_count", tiles)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int total = (int)(tiles * a->num_images);
    launch_pdl(dn_fuse_kernel<false>, dim3(total), dim3(DN_THREADS), 0, st, *a, (int)tiles);
    if (check_launch("dense_fuse_count")) return 1;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->tile_scan, total);
    return check_launch("dense_fuse_count(scan)");
}

extern "C" int romab200_dense_fuse_emit(const rb_dense_fuse_args* a, void* stream) {
    int64_t tiles;
    if (dn_fuse_check(a, "dense_fuse_emit", tiles)) return 1;
    RB_REQUIRE(a->num_points >= 0 && (a->num_points == 0 || (a->points && a->rgb && a->image && a->pixel && a->num_views && a->point_score)),
               "dense_fuse_emit: null argument");
    if (a->num_points == 0) return 0;
    launch_pdl(dn_fuse_kernel<true>, dim3((unsigned)(tiles * a->num_images)), dim3(DN_THREADS), 0, (cudaStream_t)stream, *a, (int)tiles);
    return check_launch("dense_fuse_emit");
}
