// Geometric verification of a match graph (include/romab200.h): the points of each pair gathered for the fundamental-matrix
// estimator (fundamental.cu, run chunk by chunk by the caller), then only the inlier matches of accepted pairs kept.
//   check    a thread per match: its pair by binary search in match_offsets, its ids checked; info[0] |= RB_VERIFY_BAD_ID.
//   gather   a thread per match of one chunk: x0, x1 widened to float64 at (match - chunk base), and the chunk's offsets.
//            With a pair_list, one CTA first scans the listed pairs' match counts into the chunk's offsets, then a thread per
//            packed point finds its list entry by binary search in them.
//   count    a CTA per pair: num_inliers (integer sum of its mask), accepted, its kept count into out_offsets;
//            a CTA per RB_VERIFY_TILE matches: the kept matches of the tile into tile_scan; both scanned; info[1] = the total.
//   emit     the same tiles write the kept matches and scores at the scanned offsets, in match order.
// The ids of a match are checked before any access that depends on them.  Integer arithmetic only, so the result is bit-identical
// from run to run.
#include "common.cuh"

namespace rb {

constexpr int VF_THREADS = 256;
constexpr int VF_IPT = RB_VERIFY_TILE / VF_THREADS;   // consecutive matches per thread in the tile kernels
constexpr int VF_WARPS = VF_THREADS / 32;

// the pair of match m: the last k in [lo, hi] with match_offsets[k] <= m
__device__ __forceinline__ int vf_pair_of(const int64_t* match_offsets, int lo, int hi, int64_t m) {
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (match_offsets[mid] <= m) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// true when both ids of match m of pair k lie within their images' keypoints; *ra, *rb receive their rows
__device__ __forceinline__ bool vf_rows(const rb_verify_args& a, int k, int64_t m, int64_t* ra, int64_t* rb) {
    const int64_t i = a.pairs[2 * k], j = a.pairs[2 * k + 1];
    const int64_t oi = a.kp_offsets[i], oj = a.kp_offsets[j];
    const int32_t ida = a.matches[2 * m], idb = a.matches[2 * m + 1];
    if (ida < 0 || ida >= a.kp_offsets[i + 1] - oi || idb < 0 || idb >= a.kp_offsets[j + 1] - oj) return false;
    *ra = oi + ida;
    *rb = oj + idb;
    return true;
}

// exclusive block scan of one int64 per thread (VF_THREADS threads); returns the prefix, *total the sum
__device__ __forceinline__ long long vf_block_scan(long long v, long long* total) {
    __shared__ long long warp_tot[VF_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const long long u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += u;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    long long before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < VF_WARPS; ++w) {
        before += w < wid ? warp_tot[w] : 0;
        sum += warp_tot[w];
    }
    __syncthreads();
    *total = sum;
    return before + incl - v;
}

__global__ void __launch_bounds__(VF_THREADS) vf_check_kernel(rb_verify_args a) {
    pdl_wait();
    for (int64_t m = blockIdx.x * (int64_t)VF_THREADS + threadIdx.x; m < a.num_matches; m += (int64_t)gridDim.x * VF_THREADS) {
        int64_t ra, rb;
        if (!vf_rows(a, vf_pair_of(a.match_offsets, 0, a.num_pairs - 1, m), m, &ra, &rb))
            atomicOr((unsigned long long*)a.info, (unsigned long long)RB_VERIFY_BAD_ID);
    }
}

__global__ void __launch_bounds__(VF_THREADS) vf_gather_kernel(rb_verify_args a) {
    pdl_wait();
    const int64_t base = a.match_offsets[a.pair_begin], n = a.match_offsets[a.pair_end] - base;
    const int pairs = a.pair_end - a.pair_begin;
    const int64_t t0 = blockIdx.x * (int64_t)VF_THREADS + threadIdx.x, stride = (int64_t)gridDim.x * VF_THREADS;
    for (int64_t k = t0; k <= pairs; k += stride) a.chunk_offsets[k] = a.match_offsets[a.pair_begin + k] - base;
    for (int64_t q = t0; q < n; q += stride) {
        const int64_t m = base + q;
        int64_t ra, rb;
        double2 p0 = make_double2(0.0, 0.0), p1 = make_double2(0.0, 0.0);
        if (vf_rows(a, vf_pair_of(a.match_offsets, a.pair_begin, a.pair_end - 1, m), m, &ra, &rb)) {
            p0 = make_double2(a.keypoints[2 * ra], a.keypoints[2 * ra + 1]);
            p1 = make_double2(a.keypoints[2 * rb], a.keypoints[2 * rb + 1]);
        } else {
            atomicOr((unsigned long long*)a.info, (unsigned long long)RB_VERIFY_BAD_ID);
        }
        reinterpret_cast<double2*>(a.x0)[q] = p0;
        reinterpret_cast<double2*>(a.x1)[q] = p1;
    }
}

// the matches of list entry c, or 0 (and RB_VERIFY_BAD_ID) for a pair index outside [0, num_pairs)
__device__ __forceinline__ int64_t vf_list_count(const rb_verify_args& a, int c) {
    const int k = a.pair_list[a.pair_begin + c];
    if (k < 0 || k >= a.num_pairs) {
        atomicOr((unsigned long long*)a.info, (unsigned long long)RB_VERIFY_BAD_ID);
        return 0;
    }
    return a.match_offsets[k + 1] - a.match_offsets[k];
}

// one CTA: chunk_offsets = the exclusive scan of the listed pairs' match counts, each thread a contiguous run of entries
__global__ void __launch_bounds__(VF_THREADS) vf_list_offsets_kernel(rb_verify_args a) {
    pdl_wait();
    const int pairs = a.pair_end - a.pair_begin, per = (pairs + VF_THREADS - 1) / VF_THREADS;
    const int c0 = min(pairs, (int)threadIdx.x * per), c1 = min(pairs, c0 + per);
    long long run = 0;
    for (int c = c0; c < c1; ++c) run += vf_list_count(a, c);
    long long total;
    long long before = vf_block_scan(run, &total);
    for (int c = c0; c < c1; ++c) {
        a.chunk_offsets[c] = before;
        before += vf_list_count(a, c);
    }
    if (threadIdx.x == 0) a.chunk_offsets[pairs] = total;
}

// a thread per packed point q of the listed pairs: its entry c by binary search in chunk_offsets, its match, x0 and x1
__global__ void __launch_bounds__(VF_THREADS) vf_gather_list_kernel(rb_verify_args a) {
    pdl_wait();
    const int pairs = a.pair_end - a.pair_begin;
    const int64_t n = a.chunk_offsets[pairs];
    for (int64_t q = blockIdx.x * (int64_t)VF_THREADS + threadIdx.x; q < n; q += (int64_t)gridDim.x * VF_THREADS) {
        const int c = vf_pair_of(a.chunk_offsets, 0, pairs - 1, q);
        const int k = a.pair_list[a.pair_begin + c];          // in range: an entry outside it has no points
        const int64_t m = a.match_offsets[k] + (q - a.chunk_offsets[c]);
        int64_t ra, rb;
        double2 p0 = make_double2(0.0, 0.0), p1 = make_double2(0.0, 0.0);
        if (vf_rows(a, k, m, &ra, &rb)) {
            p0 = make_double2(a.keypoints[2 * ra], a.keypoints[2 * ra + 1]);
            p1 = make_double2(a.keypoints[2 * rb], a.keypoints[2 * rb + 1]);
        } else {
            atomicOr((unsigned long long*)a.info, (unsigned long long)RB_VERIFY_BAD_ID);
        }
        reinterpret_cast<double2*>(a.x0)[q] = p0;
        reinterpret_cast<double2*>(a.x1)[q] = p1;
    }
}

// CTA k: num_inliers[k] = the integer sum of pair k's mask, accepted[k], out_offsets[k] = its kept count
__global__ void __launch_bounds__(VF_THREADS) vf_pairs_kernel(rb_verify_args a) {
    pdl_wait();
    const int k = blockIdx.x;
    const int64_t m0 = a.match_offsets[k], m1 = a.match_offsets[k + 1];
    long long cnt = 0;
    for (int64_t m = m0 + threadIdx.x; m < m1; m += VF_THREADS) cnt += a.mask[m] != 0;
    long long total;
    vf_block_scan(cnt, &total);
    if (threadIdx.x == 0) {
        const bool acc = a.ok[k] != 0 && total >= a.min_inliers;
        a.num_inliers[k] = total;
        a.accepted[k] = acc;
        a.out_offsets[k] = acc ? total : 0;
    }
}

// EMIT == false: tile_scan[t] = the kept matches of tile t.  EMIT: those matches and scores at the scanned offsets.
template <bool EMIT>
__global__ void __launch_bounds__(VF_THREADS) vf_tiles_kernel(rb_verify_args a) {
    pdl_wait();
    const int64_t m0 = (int64_t)blockIdx.x * RB_VERIFY_TILE + threadIdx.x * VF_IPT;
    const int64_t m1 = min(m0 + VF_IPT, a.num_matches);
    int k = m0 < m1 ? vf_pair_of(a.match_offsets, 0, a.num_pairs - 1, m0) : 0;
    unsigned kept = 0;                                   // bit q: match m0 + q is kept
    for (int64_t m = m0; m < m1; ++m) {
        while (a.match_offsets[k + 1] <= m) ++k;
        if (a.mask[m] && a.accepted[k]) kept |= 1u << (m - m0);
    }
    long long total;
    const long long before = vf_block_scan(__popc(kept), &total);
    if (!EMIT) {
        if (threadIdx.x == 0) a.tile_scan[blockIdx.x] = total;
        return;
    }
    int64_t o = a.tile_scan[blockIdx.x] + before;
    for (; kept; kept &= kept - 1) {
        const int64_t m = m0 + __ffs(kept) - 1;
        a.out_matches[2 * o] = a.matches[2 * m];
        a.out_matches[2 * o + 1] = a.matches[2 * m + 1];
        a.out_scores[o] = a.match_scores[m];
        ++o;
    }
}
static_assert(VF_IPT <= 32, "a thread's kept matches are one 32-bit word");

static int vf_check(const rb_verify_args* a, const char* what) {
    RB_REQUIRE(a && a->kp_offsets && a->match_offsets && a->info, "%s: null argument", what);
    RB_REQUIRE(a->num_matches == 0 || (a->pairs && a->matches && a->match_scores), "%s: null match argument", what);
    RB_REQUIRE(a->num_images > 0 && a->num_pairs > 0 && a->num_matches > 0 && a->num_rows > 0,
               "%s: bad sizes num_images=%d num_pairs=%d num_matches=%lld num_rows=%lld", what, a->num_images, a->num_pairs,
               (long long)a->num_matches, (long long)a->num_rows);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_verify_check(const rb_verify_args* a, void* stream) {
    if (vf_check(a, "verify_check")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (cudaMemsetAsync(a->info, 0, 2 * sizeof(int64_t), st) != cudaSuccess) return check_launch("verify_check(info)");
    launch_pdl(vf_check_kernel, dim3(grid1d(a->num_matches, VF_THREADS, 16 * 1024)), dim3(VF_THREADS), 0, st, *a);
    return check_launch("verify_check");
}

extern "C" int romab200_verify_gather(const rb_verify_args* a, void* stream) {
    if (vf_check(a, "verify_gather")) return 1;
    RB_REQUIRE(a->keypoints && a->x0 && a->x1 && a->chunk_offsets, "verify_gather: null argument");
    RB_REQUIRE(a->pair_begin >= 0 && a->pair_begin < a->pair_end && a->pair_end <= a->num_pairs, "verify_gather: bad chunk [%d, %d) of %d pairs",
               a->pair_begin, a->pair_end, a->num_pairs);
    cudaStream_t st = (cudaStream_t)stream;
    if (a->pair_list) {
        launch_pdl(vf_list_offsets_kernel, dim3(1), dim3(VF_THREADS), 0, st, *a);
        if (check_launch("verify_gather(list offsets)")) return 1;
        launch_pdl(vf_gather_list_kernel, dim3(grid1d(a->num_matches, VF_THREADS, 16 * 1024)), dim3(VF_THREADS), 0, st, *a);
        return check_launch("verify_gather(list)");
    }
    launch_pdl(vf_gather_kernel, dim3(grid1d(a->num_matches, VF_THREADS, 16 * 1024)), dim3(VF_THREADS), 0, st, *a);
    return check_launch("verify_gather");
}

extern "C" int romab200_verify_count(const rb_verify_args* a, void* stream) {
    if (vf_check(a, "verify_count")) return 1;
    RB_REQUIRE(a->ok && a->mask && a->num_inliers && a->accepted && a->tile_scan && a->out_offsets, "verify_count: null argument");
    RB_REQUIRE(a->min_inliers >= 0, "verify_count: min_inliers %lld < 0", (long long)a->min_inliers);
    cudaStream_t st = (cudaStream_t)stream;
    launch_pdl(vf_pairs_kernel, dim3(a->num_pairs), dim3(VF_THREADS), 0, st, *a);
    if (check_launch("verify_count(pairs)")) return 1;
    const int tiles = (int)((a->num_matches + RB_VERIFY_TILE - 1) / RB_VERIFY_TILE);
    launch_pdl(vf_tiles_kernel<false>, dim3(tiles), dim3(VF_THREADS), 0, st, *a);
    if (check_launch("verify_count(tiles)")) return 1;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->out_offsets, a->num_pairs);
    if (check_launch("verify_count(pair scan)")) return 1;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->tile_scan, tiles);
    if (check_launch("verify_count(tile scan)")) return 1;
    if (cudaMemcpyAsync(a->info + 1, a->tile_scan + tiles, sizeof(int64_t), cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return check_launch("verify_count(kept matches)");
    return 0;
}

extern "C" int romab200_verify_emit(const rb_verify_args* a, void* stream) {
    if (vf_check(a, "verify_emit")) return 1;
    RB_REQUIRE(a->mask && a->accepted && a->tile_scan && a->out_matches && a->out_scores, "verify_emit: null argument");
    RB_REQUIRE(a->num_kept > 0 && a->num_kept <= a->num_matches, "verify_emit: %lld kept matches of %lld", (long long)a->num_kept,
               (long long)a->num_matches);
    cudaStream_t st = (cudaStream_t)stream;
    const int tiles = (int)((a->num_matches + RB_VERIFY_TILE - 1) / RB_VERIFY_TILE);
    launch_pdl(vf_tiles_kernel<true>, dim3(tiles), dim3(VF_THREADS), 0, st, *a);
    return check_launch("verify_emit");
}
