// Feature tracks of a match graph (include/romab200.h): the connected components of its keypoint matches, conflicting ones
// dropped, numbered by their smallest row.
//   link    init       parent[r] = r, size[r] = 0, kp_track[r] = -1, info = 0;
//           link       a thread per match: its pair by binary search in match_offsets, its ids checked, then a lock-free union of
//                      its two rows (path halving; a link points the larger root at the smaller, so a root is its component's
//                      smallest row and the labels depend on no timing);
//           flatten    parent[r] = root(r) (walks that store nothing else), size[root] += 1 (integer atomics);
//           rows       a CTA per RB_TRACKS_TILE rows counts the rows of components of >= 2 rows; scan; info[1] = the total.
//   build   rows       the same tiles write those rows as keys (root << 32 | row) in ascending row order;
//           radix      radix_sort_hi32 (common.cuh) by root: per 8-bit digit, tile histograms, a scan over (digit, tile), a stable
//                      scatter with in-tile ranks; the input is in row order, so the output is in (root, row) order;
//           conflict   an element whose predecessor has the same root and the same image flags its root (bit 31 of size[root]);
//           segments   per tile: kept track heads and kept elements (packed into one int64), scan, then track_offsets, elements
//                      and kp_track at the scanned offsets.
// Every walk of parent pointers is bounded by K steps; the ids of a match are checked before any access that depends on them.
#include "common.cuh"

namespace rb {

constexpr int TR_THREADS = 256;
constexpr int TR_IPT = RB_TRACKS_TILE / TR_THREADS;   // consecutive items per thread in the tile kernels
constexpr int TR_WARPS = TR_THREADS / 32;
constexpr uint32_t TR_CONFLICT = 0x80000000u;         // bit 31 of size[root]: the component has a conflict

__device__ __forceinline__ void tr_status(int64_t* info, int bit) { atomicOr((unsigned long long*)info, (unsigned long long)bit); }
__device__ __forceinline__ int tr_load(const int32_t* p) { return *(const volatile int32_t*)p; }

// root of row x; -1 and RB_TRACKS_WALK after more than K steps.  HALVE: halves the path on the way.  parent[y] < y for every
// non-root y, and a halving store only moves parent[y] to another member of y's set below y, so it is safe against any concurrent
// walk or link.  The flatten pass must not halve: a store of a stale grandparent could overwrite a row's final root there.
template <bool HALVE>
__device__ int tr_find(int32_t* parent, int x, int K, int64_t* info) {
    for (int64_t s = 0; s <= K; ++s) {
        const int p = tr_load(parent + x);
        if (p == x) return x;
        if (!HALVE) {
            x = p;
            continue;
        }
        const int gp = tr_load(parent + p);
        if (gp != p) *(volatile int32_t*)(parent + x) = gp;
        x = gp;
    }
    tr_status(info, RB_TRACKS_WALK);
    return -1;
}

// joins the components of rows a and b.  A failed link means another thread linked the larger root first; the larger of the two
// roots found next is smaller than before, so there are at most K retries.
__device__ void tr_unite(int32_t* parent, int a, int b, int K, int64_t* info) {
    int ra = tr_find<true>(parent, a, K, info), rb = tr_find<true>(parent, b, K, info);
    for (int64_t s = 0; s <= K; ++s) {
        if (ra < 0 || rb < 0 || ra == rb) return;
        const int hi = max(ra, rb), lo = min(ra, rb);
        const int old = atomicCAS(parent + hi, hi, lo);
        if (old == hi) return;
        ra = tr_find<true>(parent, old, K, info);
        rb = tr_find<true>(parent, lo, K, info);
    }
    tr_status(info, RB_TRACKS_WALK);
}

// image of row r < K: the last i < N with kp_offsets[i] <= r (an empty image i has kp_offsets[i + 1] == kp_offsets[i], so it is
// never the last)
__device__ __forceinline__ int tr_image(const int64_t* kp_offsets, int N, int64_t r) {
    int lo = 0, hi = N - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (kp_offsets[mid] <= r) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// exclusive block scan of one int64 per thread (TR_THREADS threads); returns the prefix, *total the sum
__device__ __forceinline__ long long tr_block_scan(long long v, long long* total) {
    __shared__ long long warp_tot[TR_WARPS];
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
    for (int w = 0; w < TR_WARPS; ++w) {
        before += w < wid ? warp_tot[w] : 0;
        sum += warp_tot[w];
    }
    __syncthreads();
    *total = sum;
    return before + incl - v;
}

__global__ void __launch_bounds__(TR_THREADS) tr_init_kernel(rb_tracks_args a) {
    pdl_wait();
    const int64_t t0 = blockIdx.x * (int64_t)TR_THREADS + threadIdx.x;
    if (t0 < 5) a.info[t0] = 0;
    for (int64_t r = t0; r < a.num_rows; r += (int64_t)gridDim.x * TR_THREADS) {
        a.parent[r] = (int32_t)r;
        a.size[r] = 0;
        a.kp_track[r] = -1;
    }
}

__global__ void __launch_bounds__(TR_THREADS) tr_link_kernel(rb_tracks_args a) {
    pdl_wait();
    for (int64_t m = blockIdx.x * (int64_t)TR_THREADS + threadIdx.x; m < a.num_matches; m += (int64_t)gridDim.x * TR_THREADS) {
        int lo = 0, hi = a.num_pairs - 1;                 // the pair of match m: the last k with match_offsets[k] <= m
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (a.match_offsets[mid] <= m) lo = mid;
            else hi = mid - 1;
        }
        const int64_t i = a.pairs[2 * lo], j = a.pairs[2 * lo + 1];
        const int64_t ri = a.kp_offsets[i], rj = a.kp_offsets[j];
        const int32_t ida = a.matches[2 * m], idb = a.matches[2 * m + 1];
        if (ida < 0 || ida >= a.kp_offsets[i + 1] - ri || idb < 0 || idb >= a.kp_offsets[j + 1] - rj) {
            tr_status(a.info, RB_TRACKS_BAD_ID);
            continue;
        }
        if (!(a.match_scores[m] > a.min_score)) continue;
        tr_unite(a.parent, (int)(ri + ida), (int)(rj + idb), a.num_rows, a.info);
    }
}

__global__ void __launch_bounds__(TR_THREADS) tr_flatten_kernel(rb_tracks_args a) {
    pdl_wait();
    for (int64_t r = blockIdx.x * (int64_t)TR_THREADS + threadIdx.x; r < a.num_rows; r += (int64_t)gridDim.x * TR_THREADS) {
        const int root = tr_find<false>(a.parent, (int)r, a.num_rows, a.info);
        if (root < 0) continue;
        *(volatile int32_t*)(a.parent + r) = root;
        atomicAdd(a.size + root, 1);
    }
}

// EMIT == false: tile_scan[t] = rows of tile t in components of >= 2 rows.  EMIT: those rows as keys at the scanned offsets.
template <bool EMIT>
__global__ void __launch_bounds__(TR_THREADS) tr_rows_kernel(rb_tracks_args a) {
    pdl_wait();
    const int64_t r0 = (int64_t)blockIdx.x * RB_TRACKS_TILE + threadIdx.x * TR_IPT;
    const int64_t r1 = min(r0 + TR_IPT, (int64_t)a.num_rows);
    int cnt = 0;
    for (int64_t r = r0; r < r1; ++r) cnt += a.size[a.parent[r]] >= 2;
    long long total;
    const long long before = tr_block_scan(cnt, &total);
    if (!EMIT) {
        if (threadIdx.x == 0) a.tile_scan[blockIdx.x] = total;
        return;
    }
    int64_t o = a.tile_scan[blockIdx.x] + before;
    for (int64_t r = r0; r < r1; ++r) {
        const uint32_t root = (uint32_t)a.parent[r];
        if (a.size[root] >= 2) a.keys[o++] = ((unsigned long long)root << 32) | (uint32_t)r;
    }
}

__global__ void __launch_bounds__(TR_THREADS) tr_conflict_kernel(rb_tracks_args a, const uint64_t* __restrict__ keys, int64_t n) {
    pdl_wait();
    for (int64_t q = 1 + blockIdx.x * (int64_t)TR_THREADS + threadIdx.x; q < n; q += (int64_t)gridDim.x * TR_THREADS) {
        const uint64_t k = keys[q], p = keys[q - 1];
        const uint32_t root = (uint32_t)(k >> 32);
        if (root != (uint32_t)(p >> 32)) continue;
        if (tr_image(a.kp_offsets, a.num_images, (uint32_t)k) != tr_image(a.kp_offsets, a.num_images, (uint32_t)p)) continue;
        if (!(tr_load(a.size + root) & TR_CONFLICT)) atomicOr((unsigned*)(a.size + root), TR_CONFLICT);
    }
}

// EMIT == false: tile_scan[t] = (kept track heads << 32) | kept elements of sorted tile t, and info[4] += conflicting heads.
// EMIT: track_offsets, elements and kp_track of the tile's kept elements; CTA 0 writes T, E and track_offsets[T].
template <bool EMIT>
__global__ void __launch_bounds__(TR_THREADS) tr_segments_kernel(rb_tracks_args a, const uint64_t* __restrict__ keys, int64_t n) {
    pdl_wait();
    const int64_t q0 = (int64_t)blockIdx.x * RB_TRACKS_TILE + threadIdx.x * TR_IPT;
    const int64_t q1 = min(q0 + TR_IPT, n);
    const auto kept = [&](uint32_t root, bool& conflict) {
        const uint32_t s = (uint32_t)a.size[root];
        conflict = (s & TR_CONFLICT) != 0;
        return (int)(s & ~TR_CONFLICT) >= a.min_length && !(a.drop_conflicts && conflict);
    };
    long long cnt = 0;
    int conflicting = 0;
    for (int64_t q = q0; q < q1; ++q) {
        const uint32_t root = (uint32_t)(keys[q] >> 32);
        const bool head = q == 0 || (uint32_t)(keys[q - 1] >> 32) != root;
        bool conflict;
        const bool k = kept(root, conflict);
        cnt += ((long long)(head && k) << 32) + k;
        conflicting += head && conflict;
    }
    long long total;
    const long long before = tr_block_scan(cnt, &total);
    if (!EMIT) {
        if (conflicting) atomicAdd((unsigned long long*)(a.info + 4), (unsigned long long)conflicting);
        if (threadIdx.x == 0) a.tile_scan[blockIdx.x] = total;
        return;
    }
    const long long pre = a.tile_scan[blockIdx.x] + before;
    int64_t track = (pre >> 32) - 1, o = pre & 0xffffffffll;
    for (int64_t q = q0; q < q1; ++q) {
        const uint32_t root = (uint32_t)(keys[q] >> 32), row = (uint32_t)keys[q];
        bool conflict;
        if (!kept(root, conflict)) continue;
        if (q == 0 || (uint32_t)(keys[q - 1] >> 32) != root) a.track_offsets[++track] = o;
        const int img = tr_image(a.kp_offsets, a.num_images, row);
        a.elements[2 * o] = img;
        a.elements[2 * o + 1] = (int32_t)(row - a.kp_offsets[img]);
        a.kp_track[row] = (int32_t)track;
        ++o;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const long long all = a.tile_scan[gridDim.x], T = all >> 32, E = all & 0xffffffffll;
        a.info[2] = T;
        a.info[3] = E;
        a.track_offsets[T] = E;
    }
}

static int tr_check(const rb_tracks_args* a, const char* what) {
    RB_REQUIRE(a && a->kp_offsets && a->match_offsets && a->parent && a->size && a->tile_scan && a->info && a->kp_track, "%s: null argument", what);
    RB_REQUIRE(a->num_matches == 0 || (a->pairs && a->matches && a->match_scores), "%s: null match argument", what);
    RB_REQUIRE(a->num_images > 0 && a->num_rows > 0 && a->num_pairs >= 0 && a->num_matches >= 0 && (a->num_matches == 0 || a->num_pairs > 0),
               "%s: bad sizes num_images=%d num_rows=%d num_pairs=%d num_matches=%lld", what, a->num_images, a->num_rows, a->num_pairs,
               (long long)a->num_matches);
    RB_REQUIRE(a->min_length >= 2 && a->min_score >= 0.f && isfinite(a->min_score), "%s: bad min_length=%d min_score=%g", what, a->min_length,
               a->min_score);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_tracks_link(const rb_tracks_args* a, void* stream) {
    if (tr_check(a, "tracks_link")) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned row_grid = grid1d(a->num_rows, TR_THREADS, 16 * 1024);
    launch_pdl(tr_init_kernel, dim3(row_grid), dim3(TR_THREADS), 0, st, *a);
    if (check_launch("tracks_link(init)")) return 1;
    if (a->num_matches > 0) {
        launch_pdl(tr_link_kernel, dim3(grid1d(a->num_matches, TR_THREADS, 16 * 1024)), dim3(TR_THREADS), 0, st, *a);
        if (check_launch("tracks_link(link)")) return 1;
    }
    launch_pdl(tr_flatten_kernel, dim3(row_grid), dim3(TR_THREADS), 0, st, *a);
    if (check_launch("tracks_link(flatten)")) return 1;
    const int tiles = (int)((a->num_rows + RB_TRACKS_TILE - 1) / RB_TRACKS_TILE);
    launch_pdl(tr_rows_kernel<false>, dim3(tiles), dim3(TR_THREADS), 0, st, *a);
    if (check_launch("tracks_link(count)")) return 1;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->tile_scan, tiles);
    if (check_launch("tracks_link(scan)")) return 1;
    if (cudaMemcpyAsync(a->info + 1, a->tile_scan + tiles, sizeof(int64_t), cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return check_launch("tracks_link(kept rows)");
    return 0;
}

extern "C" int romab200_tracks_build(const rb_tracks_args* a, void* stream) {
    if (tr_check(a, "tracks_build")) return 1;
    RB_REQUIRE(a->keys && a->keys_alt && a->hist && a->track_offsets && a->elements, "tracks_build: null argument");
    RB_REQUIRE(a->num_kept > 1 && a->num_kept <= a->num_rows, "tracks_build: %lld kept rows of %d", (long long)a->num_kept, a->num_rows);
    cudaStream_t st = (cudaStream_t)stream;
    const int row_tiles = (int)((a->num_rows + RB_TRACKS_TILE - 1) / RB_TRACKS_TILE);
    launch_pdl(tr_rows_kernel<true>, dim3(row_tiles), dim3(TR_THREADS), 0, st, *a);
    if (check_launch("tracks_build(rows)")) return 1;
    const int64_t n = a->num_kept;
    const int tiles = (int)((n + RB_TRACKS_TILE - 1) / RB_TRACKS_TILE);
    const int bits = 32 - __builtin_clz((unsigned)(a->num_rows - 1));        // roots lie in [0, num_rows), num_rows >= 2
    uint64_t* in = nullptr;
    if (radix_sort_hi32<RB_TRACKS_TILE>(a->keys, a->keys_alt, a->hist, n, bits, st, "tracks_build(radix)", &in)) return 1;
    launch_pdl(tr_conflict_kernel, dim3(grid1d(n, TR_THREADS, 16 * 1024)), dim3(TR_THREADS), 0, st, *a, (const uint64_t*)in, n);
    if (check_launch("tracks_build(conflicts)")) return 1;
    launch_pdl(tr_segments_kernel<false>, dim3(tiles), dim3(TR_THREADS), 0, st, *a, (const uint64_t*)in, n);
    if (check_launch("tracks_build(count)")) return 1;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->tile_scan, tiles);
    if (check_launch("tracks_build(scan)")) return 1;
    launch_pdl(tr_segments_kernel<true>, dim3(tiles), dim3(TR_THREADS), 0, st, *a, (const uint64_t*)in, n);
    return check_launch("tracks_build(emit)");
}
