// `RegressionMatcher.match_keypoints` on the device (romatch/models/matcher.py:743-762): the two grid samples of the warp and
// the certainty at the keypoints of A, and the mutual nearest neighbours of x_A_to_B and x_B under the exact-difference distance
//   D[i, j] = sqrt_rn(dx*dx + dy*dy),  dx = x_A_to_B[i].x - x_B[j].x,  every operation rounded to fp32 (no FMA contraction),
// with (i, j) returned iff D[i,j] is the minimum of its row and of its column, cert_A[i] > cert_th and D[i,j] < max_dist.
// No N_A x N_B buffer exists anywhere:
//   min      row minima and column minima of d^2 = D^2 in two sweeps.  A thread owns KP_ROWS points in registers, the other
//            set streams through shared memory; the other set is cut into `splits` slices (grid.y) whose partial minima a
//            second kernel combines.  min is exact, so the result does not depend on the order: deterministic without atomics.
//            `min.NaN` propagates NaN like torch.min; sqrt_rn is monotone, so sqrt_rn(min d^2) = min D.
//   count    one thread per row: rows failing the certainty or the max_dist test are skipped, the others count the columns j
//            with colmin[j] == rowmin[i] and D[i,j] == rowmin[i] (the two minimum conditions; D[i,j] is only evaluated on the
//            rare column whose minimum equals the row's);
//   scan     exclusive scan of the counts in one CTA (scan_counts_kernel) -> offsets[0..n_a], offsets[n_a] = number of matches;
//   emit     the same sweep writes (i, j) at the row's offset, j ascending: the order of torch.nonzero.
#include "common.cuh"
#include "tma.cuh"

namespace rb {

constexpr int KP_THREADS = 128;
constexpr int KP_ROWS = 4;                      // points owned by one thread in the min sweeps
constexpr int KP_TILE = 1024;                   // points of the other set per shared-memory tile (8 KB)
constexpr int KP_MAX_SPLITS = 16;

// torch.min semantics: NaN if either operand is NaN
__device__ __forceinline__ float min_nan(float a, float b) {
    float r;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// dx*dx + dy*dy with every operation rounded separately.  Round-to-nearest subtraction is sign-symmetric, so the value does not
// depend on which point comes first: both sweeps and the count see the same d^2 for a pair.
__device__ __forceinline__ float dist2(float px, float py, float qx, float qy) {
    const float dx = __fsub_rn(px, qx), dy = __fsub_rn(py, qy);
    return __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
}

// grid_sample (bilinear, zero padding, align_corners=False) of `nch` channels at the normalised position (x, y): ATen's
// unnormalisation ((x + 1) * size - 1) / 2 and corner weights, corners accumulated in the order nw, ne, sw, se.  A NaN position
// gives NaN.
__device__ __forceinline__ void sample_bilinear(const float* __restrict__ map, int h, int w, int64_t ld_row, int64_t ld_px, int64_t ld_ch,
                                                int nch, float x, float y, float* out) {
    const float ix = ((x + 1.f) * (float)w - 1.f) / 2.f, iy = ((y + 1.f) * (float)h - 1.f) / 2.f;
    if (ix != ix || iy != iy) {
        for (int c = 0; c < nch; ++c) out[c] = __int_as_float(0x7fc00000);
        return;
    }
    const float x0 = floorf(ix), y0 = floorf(iy), x1 = x0 + 1.f, y1 = y0 + 1.f;
    const float wts[4] = {(x1 - ix) * (y1 - iy), (ix - x0) * (y1 - iy), (x1 - ix) * (iy - y0), (ix - x0) * (iy - y0)};
    const float cx[4] = {x0, x1, x0, x1}, cy[4] = {y0, y0, y1, y1};
    for (int c = 0; c < nch; ++c) out[c] = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (cx[k] >= 0.f && cx[k] < (float)w && cy[k] >= 0.f && cy[k] < (float)h) {     // in float: no overflow for far-away points
            const float* q = map + (int64_t)cy[k] * ld_row + (int64_t)cx[k] * ld_px;
            for (int c = 0; c < nch; ++c) out[c] += q[c * ld_ch] * wts[k];
        }
    }
}

__global__ void __launch_bounds__(KP_THREADS) kp_sample_kernel(rb_keypoints_sample_args a) {
    rb::pdl_wait();
    const int i = blockIdx.x * KP_THREADS + threadIdx.x;
    if (i >= a.n) return;
    const float x = a.x[2 * (int64_t)i], y = a.x[2 * (int64_t)i + 1];
    float v[2], c;
    sample_bilinear(a.warp, a.warp_h, a.warp_w, a.warp_ld_row, a.warp_ld_px, a.warp_ld_ch, 2, x, y, v);
    sample_bilinear(a.cert, a.cert_h, a.cert_w, a.cert_ld_row, a.cert_ld_px, 1, 1, x, y, &c);
    a.x_to_B[2 * (int64_t)i] = v[0];
    a.x_to_B[2 * (int64_t)i + 1] = v[1];
    a.cert_out[i] = c;
}

// partial[s * n_own + k] = min.NaN over the s-th slice [s * per_split, (s + 1) * per_split) of the other set of d^2(own[k], other[j])
__global__ void __launch_bounds__(KP_THREADS) kp_min_kernel(const float* __restrict__ own, int n_own, const float* __restrict__ other, int n_other,
                                                            int per_split, float* __restrict__ partial) {
    rb::pdl_wait();
    __shared__ __align__(16) float2 tile[KP_TILE];
    const int k0 = blockIdx.x * KP_THREADS * KP_ROWS + threadIdx.x;
    float px[KP_ROWS], py[KP_ROWS], m[KP_ROWS];
#pragma unroll
    for (int r = 0; r < KP_ROWS; ++r) {
        const int k = k0 + r * KP_THREADS;
        px[r] = k < n_own ? own[2 * (int64_t)k] : 0.f;
        py[r] = k < n_own ? own[2 * (int64_t)k + 1] : 0.f;
        m[r] = __int_as_float(0x7f800000);
    }
    const int j0 = blockIdx.y * per_split, j1 = min(n_other, j0 + per_split);
    for (int t0 = j0; t0 < j1; t0 += KP_TILE) {
        const int cnt = min(KP_TILE, j1 - t0);
        __syncthreads();
        for (int j = threadIdx.x; j < cnt; j += KP_THREADS)
            tile[j] = make_float2(other[2 * (int64_t)(t0 + j)], other[2 * (int64_t)(t0 + j) + 1]);
        __syncthreads();
        const float4* tile4 = reinterpret_cast<const float4*>(tile);
#pragma unroll 4
        for (int j = 0; j < cnt / 2; ++j) {
            const float4 q = tile4[j];
#pragma unroll
            for (int r = 0; r < KP_ROWS; ++r) m[r] = min_nan(min_nan(m[r], dist2(px[r], py[r], q.x, q.y)), dist2(px[r], py[r], q.z, q.w));
        }
        if (cnt & 1) {
            const float2 q = tile[cnt - 1];
#pragma unroll
            for (int r = 0; r < KP_ROWS; ++r) m[r] = min_nan(m[r], dist2(px[r], py[r], q.x, q.y));
        }
    }
    float* dst = partial + (int64_t)blockIdx.y * n_own;
#pragma unroll
    for (int r = 0; r < KP_ROWS; ++r) {
        const int k = k0 + r * KP_THREADS;
        if (k < n_own) dst[k] = m[r];
    }
}

// rowmin[k] / colmin[k] = sqrt_rn of the minimum over the slices (rowmin and colmin are adjacent in the workspace)
__global__ void __launch_bounds__(256) kp_finish_min_kernel(const float* __restrict__ part_r, const float* __restrict__ part_c, int n_a, int n_b,
                                                            int splits_r, int splits_c, float* __restrict__ mins) {
    rb::pdl_wait();
    const int k = blockIdx.x * 256 + threadIdx.x;
    if (k >= n_a + n_b) return;
    const bool row = k < n_a;
    const float* p = row ? part_r + k : part_c + (k - n_a);
    const int splits = row ? splits_r : splits_c;
    const int64_t n = row ? n_a : n_b;
    float v = p[0];
    for (int s = 1; s < splits; ++s) v = min_nan(v, p[s * n]);
    mins[k] = __fsqrt_rn(v);
}

// count (EMIT == false: offsets[i] = number of matches of row i) or write them (EMIT: at offsets[i], j ascending)
template <bool EMIT>
__global__ void __launch_bounds__(KP_THREADS) kp_pairs_kernel(const float* __restrict__ xab, const float* __restrict__ cert_A, const float* __restrict__ xb,
                                                              const float* __restrict__ rowmin, const float* __restrict__ colmin, int n_a, int n_b,
                                                              float cert_th, float max_dist, int64_t* __restrict__ offsets, int64_t* __restrict__ inds_A,
                                                              int64_t* __restrict__ inds_B) {
    rb::pdl_wait();
    const int i = blockIdx.x * KP_THREADS + threadIdx.x;
    if (i >= n_a) return;
    const float r = rowmin[i];
    int64_t o = 0;
    if (EMIT) {
        o = offsets[i];
        if (offsets[i + 1] == o) return;
    }
    int64_t c = 0;
    if (cert_A[i] > cert_th && r < max_dist) {          // false for a NaN row minimum
        const float ax = xab[2 * (int64_t)i], ay = xab[2 * (int64_t)i + 1];
#pragma unroll 8
        for (int j = 0; j < n_b; ++j) {
            if (colmin[j] == r && __fsqrt_rn(dist2(ax, ay, xb[2 * (int64_t)j], xb[2 * (int64_t)j + 1])) == r) {
                if (EMIT) {
                    inds_A[o + c] = i;
                    inds_B[o + c] = j;
                }
                ++c;
            }
        }
    }
    if (!EMIT) offsets[i] = c;
}

// slices of the other set for a min sweep over n_own points: enough CTAs to fill the GPU several times, at least one tile per slice
static int kp_splits(int n_own, int n_other) {
    const int ctas = (n_own + KP_THREADS * KP_ROWS - 1) / (KP_THREADS * KP_ROWS);
    int s = (8 * sm_count() + ctas - 1) / ctas;
    s = min(s, min(KP_MAX_SPLITS, (n_other + KP_TILE - 1) / KP_TILE));
    return max(s, 1);
}

static int kp_check(const rb_keypoints_mnn_args* a, const char* what) {
    RB_REQUIRE(a && a->x_A_to_B && a->cert_A && a->x_B && a->workspace && a->offsets, "%s: null argument", what);
    RB_REQUIRE(a->n_a > 0 && a->n_b > 0, "%s: empty point set (n_a=%d, n_b=%d)", what, a->n_a, a->n_b);
    const int64_t need = (int64_t)(KP_MAX_SPLITS + 1) * ((int64_t)a->n_a + a->n_b);
    RB_REQUIRE(a->workspace_floats >= need, "%s: workspace of %lld floats, (16 + 1) * (n_a + n_b) = %lld needed", what, (long long)a->workspace_floats,
               (long long)need);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_keypoints_sample(const rb_keypoints_sample_args* a, void* stream) {
    RB_REQUIRE(a && a->x && a->warp && a->cert && a->x_to_B && a->cert_out, "keypoints_sample: null argument");
    RB_REQUIRE(a->n > 0 && a->warp_h > 0 && a->warp_w > 0 && a->cert_h > 0 && a->cert_w > 0, "keypoints_sample: bad shape n=%d warp %dx%d cert %dx%d",
               a->n, a->warp_h, a->warp_w, a->cert_h, a->cert_w);
    rb::launch_pdl(kp_sample_kernel, dim3((a->n + KP_THREADS - 1) / KP_THREADS), dim3(KP_THREADS), 0, (cudaStream_t)stream, *a);
    return check_launch("keypoints_sample");
}

extern "C" int romab200_keypoints_mnn_count(const rb_keypoints_mnn_args* a, void* stream) {
    if (kp_check(a, "keypoints_mnn_count")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const int n_a = a->n_a, n_b = a->n_b;
    const int splits_r = kp_splits(n_a, n_b), splits_c = kp_splits(n_b, n_a);
    float* mins = a->workspace;                                 // rowmin [n_a] | colmin [n_b] | row slices [splits_r, n_a] | column slices [splits_c, n_b]
    float* part_r = mins + n_a + n_b;
    float* part_c = part_r + (int64_t)splits_r * n_a;
    const int per_r = (n_b + splits_r - 1) / splits_r, per_c = (n_a + splits_c - 1) / splits_c;
    constexpr int PER_CTA = KP_THREADS * KP_ROWS;
    rb::launch_pdl(kp_min_kernel, dim3((n_a + PER_CTA - 1) / PER_CTA, splits_r), dim3(KP_THREADS), 0, st, a->x_A_to_B, n_a, a->x_B, n_b, per_r, part_r);
    if (check_launch("keypoints_mnn_count(row minima)")) return 1;
    rb::launch_pdl(kp_min_kernel, dim3((n_b + PER_CTA - 1) / PER_CTA, splits_c), dim3(KP_THREADS), 0, st, a->x_B, n_b, a->x_A_to_B, n_a, per_c, part_c);
    if (check_launch("keypoints_mnn_count(column minima)")) return 1;
    rb::launch_pdl(kp_finish_min_kernel, dim3((n_a + n_b + 255) / 256), dim3(256), 0, st, (const float*)part_r, (const float*)part_c, n_a, n_b, splits_r,
                   splits_c, mins);
    if (check_launch("keypoints_mnn_count(finish minima)")) return 1;
    rb::launch_pdl(kp_pairs_kernel<false>, dim3((n_a + KP_THREADS - 1) / KP_THREADS), dim3(KP_THREADS), 0, st, a->x_A_to_B, a->cert_A, a->x_B,
                   (const float*)mins, (const float*)(mins + n_a), n_a, n_b, a->cert_th, a->max_dist, a->offsets, (int64_t*)nullptr, (int64_t*)nullptr);
    if (check_launch("keypoints_mnn_count(count)")) return 1;
    rb::launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->offsets, n_a);
    return check_launch("keypoints_mnn_count(scan)");
}

extern "C" int romab200_keypoints_mnn_emit(const rb_keypoints_mnn_args* a, void* stream) {
    if (kp_check(a, "keypoints_mnn_emit")) return 1;
    RB_REQUIRE(a->inds_A && a->inds_B, "keypoints_mnn_emit: null output");
    const float* mins = a->workspace;
    rb::launch_pdl(kp_pairs_kernel<true>, dim3((a->n_a + KP_THREADS - 1) / KP_THREADS), dim3(KP_THREADS), 0, (cudaStream_t)stream, a->x_A_to_B, a->cert_A,
                   a->x_B, mins, mins + a->n_a, a->n_a, a->n_b, a->cert_th, a->max_dist, a->offsets, a->inds_A, a->inds_B);
    return check_launch("keypoints_mnn_emit");
}
