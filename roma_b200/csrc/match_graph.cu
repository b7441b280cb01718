// Structure-from-motion match graph from sampled dense matches (include/romab200.h): every sample side is snapped to a pixel cell of
// its image, one keypoint per occupied cell, and each pair keeps its mutual-best (a, b) keypoint matches.
//   keypoints  per group of images whose cell grids fit the caller's workspace:
//              side_max    a thread per sample side: 32-bit atomicMax of the certainty's bits into its cell (the certainty is > 0,
//                          so its bits order like its value);
//              side_min_g  sides whose certainty equals their cell's maximum: 64-bit atomicMin of g, the tie-break;
//              tile_count  a CTA per RB_MG_TILE cells of one image counts the occupied ones;
//              scan        exclusive tile offsets, and the group's entries of kp_offsets;
//              tile_emit   ranks the occupied cells of the tile in raster order, writes the winner's position and score, and
//                          overwrites the cell's bits with its id;
//              side_id     a thread per sample side writes its cell's id (or -1) to sid.
//   pairs      a CTA per pair sorts 64-bit keys with a bitonic network, in shared memory or, for large n, in scratch:
//              rank        (~certainty bits, s) -> rank r of every used sample (certainty descending, s ascending);
//              by b        (b, r): the first of each run is best_a(b)'s sample -> flag[r];
//              by a        (a, r): the first of each run is best_b(a)'s sample; kept iff flagged; counted or written in a order.
// Only integer atomics on keys whose maximum / minimum is unique: deterministic, independent of how the work is grouped.
#include "common.cuh"
#include "tma.cuh"

namespace rb {

constexpr int MG_THREADS = 256;
constexpr int MG_CELLS = RB_MG_TILE / MG_THREADS;     // consecutive cells per thread in the tile kernels
constexpr int MG_PAIR_THREADS = 512;
constexpr unsigned long long MG_NONE = ~0ull;

__host__ __device__ inline int64_t mg_pow2(int64_t n) {
    int64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}
__host__ __device__ inline int64_t mg_pair_bytes(int n) { return (8 * mg_pow2(n) + 5 * (int64_t)n + 15) / 16 * 16; }

// The side `gs` = (k * n + s) * 2 + side: -1 if its image is outside [img_begin, img_end), 0 if ignored, 1 with its cell's index
// in the group's grid, its pixel position and its certainty's bits.
__device__ __forceinline__ int mg_side(const rb_match_graph_keypoints_args& a, int64_t gs, int64_t& cell, float& x, float& y, uint32_t& bits) {
    const int side = (int)(gs & 1);
    const int64_t ks = gs >> 1, k = ks / a.n;
    const int img = (int)a.pairs[2 * k + side];
    if (img < a.img_begin || img >= a.img_end) return -1;
    const float c = a.certainty[ks];
    const float u = a.matches[4 * ks + 2 * side], v = a.matches[4 * ks + 2 * side + 1];
    if (!(c > a.min_certainty) || !isfinite(c) || !isfinite(u) || !isfinite(v)) return 0;
    const int H = a.image_sizes[2 * img], W = a.image_sizes[2 * img + 1];
    x = __fmul_rn((float)W * 0.5f, __fadd_rn(u, 1.f));
    y = __fmul_rn((float)H * 0.5f, __fadd_rn(v, 1.f));
    const int cx = (int)fminf(fmaxf(floorf(x), 0.f), (float)(W - 1)) / a.cell_size;
    const int cy = (int)fminf(fmaxf(floorf(y), 0.f), (float)(H - 1)) / a.cell_size;
    const int gw = (W + a.cell_size - 1) / a.cell_size;
    cell = a.cell_start[img] - a.cell_start[a.img_begin] + (int64_t)cy * gw + cx;
    bits = __float_as_uint(c);
    return 1;
}

// PASS 0: cell maximum of the certainty bits; 1: smallest g among the sides at that maximum; 2: sid
template <int PASS>
__global__ void __launch_bounds__(MG_THREADS) mg_side_kernel(rb_match_graph_keypoints_args a) {
    pdl_wait();
    const int64_t total = (int64_t)a.num_pairs * a.n * 2;
    for (int64_t gs = blockIdx.x * (int64_t)MG_THREADS + threadIdx.x; gs < total; gs += (int64_t)gridDim.x * MG_THREADS) {
        int64_t cell;
        float x, y;
        uint32_t bits;
        const int st = mg_side(a, gs, cell, x, y, bits);
        if (PASS == 0 && st == 1) atomicMax(&a.grid_bits[cell], bits);
        if (PASS == 1 && st == 1 && a.grid_bits[cell] == bits) atomicMin((unsigned long long*)&a.grid_g[cell], (unsigned long long)gs);
        if (PASS == 2 && st >= 0) a.sid[gs] = st ? (int32_t)a.grid_bits[cell] : -1;
    }
}

// the image of the group's tile t: the last img in [img_begin, img_end) with tile_start[img] <= tile_start[img_begin] + t
__device__ __forceinline__ int mg_tile_image(const rb_match_graph_keypoints_args& a, int64_t t) {
    const int64_t g = a.tile_start[a.img_begin] + t;
    int lo = a.img_begin, hi = a.img_end - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.tile_start[mid] <= g) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

// exclusive block scan of one int per thread (MG_THREADS threads); returns the prefix, *total the sum
__device__ __forceinline__ int mg_block_scan(int v, int* total) {
    __shared__ int warp_tot[MG_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += u;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < MG_THREADS / 32; ++w) {
        before += w < wid ? warp_tot[w] : 0;
        sum += warp_tot[w];
    }
    __syncthreads();
    *total = sum;
    return before + incl - v;
}

// EMIT == false: tile_scan[t] = occupied cells of tile t.  EMIT: ids, keypoints and scores of the tile's occupied cells.
template <bool EMIT>
__global__ void __launch_bounds__(MG_THREADS) mg_tile_kernel(rb_match_graph_keypoints_args a) {
    pdl_wait();
    const int64_t t = blockIdx.x;
    const int img = mg_tile_image(a, t);
    const int64_t first = (a.tile_start[a.img_begin] + t - a.tile_start[img]) * RB_MG_TILE;        // first cell of the tile in the image
    const int64_t cells = a.cell_start[img + 1] - a.cell_start[img];
    const int64_t base = a.cell_start[img] - a.cell_start[a.img_begin] + first;                      // the same in the group's grid
    const int64_t c0 = (int64_t)threadIdx.x * MG_CELLS;
    uint32_t bits[MG_CELLS];
    int cnt = 0;
#pragma unroll
    for (int q = 0; q < MG_CELLS; ++q) {
        bits[q] = first + c0 + q < cells ? a.grid_bits[base + c0 + q] : 0u;
        cnt += bits[q] != 0u;
    }
    int total;
    const int before = mg_block_scan(cnt, &total);
    if (!EMIT) {
        if (threadIdx.x == 0) a.tile_scan[t] = total;
        return;
    }
    // the tile's first id within the image: occupied cells of the image's earlier tiles
    int64_t id = a.tile_scan[t] - a.tile_scan[a.tile_start[img] - a.tile_start[a.img_begin]] + before;
    const int64_t kp0 = a.kp_offsets[img];
    const int H = a.image_sizes[2 * img], W = a.image_sizes[2 * img + 1];
#pragma unroll
    for (int q = 0; q < MG_CELLS; ++q) {
        if (bits[q] == 0u) continue;
        const int64_t c = base + c0 + q, gs = (int64_t)a.grid_g[c], ks = gs >> 1, side = gs & 1;
        const float u = a.matches[4 * ks + 2 * side], v = a.matches[4 * ks + 2 * side + 1];
        const int64_t o = kp0 + id;
        if (o < a.kp_capacity) {
            a.keypoints[2 * o] = __fmul_rn((float)W * 0.5f, __fadd_rn(u, 1.f));
            a.keypoints[2 * o + 1] = __fmul_rn((float)H * 0.5f, __fadd_rn(v, 1.f));
            a.kp_scores[o] = __uint_as_float(bits[q]);
        }
        a.grid_bits[c] = (uint32_t)id;
        ++id;
    }
}

// one CTA: kp_offsets[img + 1] of the group's images from the scanned tile counts
__global__ void __launch_bounds__(1024) mg_kp_offsets_kernel(rb_match_graph_keypoints_args a) {
    pdl_wait();
    const int64_t t0 = a.tile_start[a.img_begin], k0 = a.kp_offsets[a.img_begin];
    for (int img = a.img_begin + threadIdx.x; img < a.img_end; img += blockDim.x)
        a.kp_offsets[img + 1] = k0 + a.tile_scan[a.tile_start[img + 1] - t0];
}

// ---- pairs --------------------------------------------------------------------------------------------------------------------

// ascending bitonic sort of keys[0, n2), n2 a power of two, by the whole CTA
__device__ __forceinline__ void mg_sort(unsigned long long* keys, int n2) {
    for (int k = 2; k <= n2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n2 / 2; i += MG_PAIR_THREADS) {
                const int lo = ((i & ~(j - 1)) << 1) | (i & (j - 1)), hi = lo + j;
                const unsigned long long x = keys[lo], y = keys[hi];
                if ((x > y) == ((lo & k) == 0)) {
                    keys[lo] = y;
                    keys[hi] = x;
                }
            }
            __syncthreads();
        }
    }
}

// EMIT == false: match_offsets[k] = kept matches of pair k.  EMIT: writes them at match_offsets[k].
// Storage: keys [n2] | ord [n] (sample of rank r) | flag [n] (rank r is best_a of its b), in shared memory or in the pair's scratch.
template <bool EMIT>
__global__ void __launch_bounds__(MG_PAIR_THREADS, 1) mg_pair_kernel(rb_match_graph_pairs_args a, int in_smem) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char mg_smem[];
    __shared__ int s_used, s_total[MG_PAIR_THREADS / 32];
    const int n = a.n;
    const int64_t k = a.pair_begin + (int64_t)blockIdx.x;
    const int64_t n2_full = mg_pow2(n);
    unsigned char* store = in_smem ? mg_smem : a.scratch + (int64_t)blockIdx.x * mg_pair_bytes(n);
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(store);
    uint32_t* ord = reinterpret_cast<uint32_t*>(store + 8 * n2_full);
    unsigned char* flag = store + 8 * n2_full + 4 * (int64_t)n;
    const int32_t* sid = a.sid + k * n * 2;
    const float* cert = a.certainty + k * n;
    if (threadIdx.x == 0) s_used = 0;
    __syncthreads();
    int used = 0;
    for (int s = threadIdx.x; s < n; s += MG_PAIR_THREADS) {
        const bool ok = sid[2 * s] >= 0 && sid[2 * s + 1] >= 0;
        keys[s] = ok ? ((unsigned long long)(~__float_as_uint(cert[s])) << 32) | (uint32_t)s : MG_NONE;
        flag[s] = 0;
        used += ok;
    }
    atomicAdd(&s_used, used);
    __syncthreads();
    const int V = s_used;
    for (int s = n + threadIdx.x; s < n2_full; s += MG_PAIR_THREADS) keys[s] = MG_NONE;
    __syncthreads();
    mg_sort(keys, (int)n2_full);
    const int n2 = (int)mg_pow2(V);           // the two sorts by id hold keys at ranks r < V: pow2(V) of them need sorting
    for (int r = threadIdx.x; r < V; r += MG_PAIR_THREADS) ord[r] = (uint32_t)keys[r];
    __syncthreads();
#pragma unroll 1
    for (int side = 1; side >= 0; --side) {
        for (int r = threadIdx.x; r < n2; r += MG_PAIR_THREADS)
            keys[r] = r < V ? ((unsigned long long)(uint32_t)sid[2 * (int64_t)ord[r] + side] << 32) | (uint32_t)r : MG_NONE;
        __syncthreads();
        mg_sort(keys, n2);
        if (side == 1) {
            for (int q = threadIdx.x; q < V; q += MG_PAIR_THREADS)
                if (q == 0 || (keys[q] >> 32) != (keys[q - 1] >> 32)) flag[(uint32_t)keys[q]] = 1;
            __syncthreads();
        }
    }
    // runs of a in ascending order; a contiguous chunk of them per thread
    const int per = (V + MG_PAIR_THREADS - 1) / MG_PAIR_THREADS;
    const int q0 = min(V, (int)threadIdx.x * per), q1 = min(V, q0 + per);
    int cnt = 0;
    for (int q = q0; q < q1; ++q) cnt += (q == 0 || (keys[q] >> 32) != (keys[q - 1] >> 32)) && flag[(uint32_t)keys[q]];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int incl = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += u;
    }
    if (lane == 31) s_total[wid] = incl;
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < MG_PAIR_THREADS / 32; ++w) {
        before += w < wid ? s_total[w] : 0;
        total += s_total[w];
    }
    if (!EMIT) {
        if (threadIdx.x == 0) a.match_offsets[k] = total;
        return;
    }
    int64_t o = a.match_offsets[k] + before + incl - cnt;
    for (int q = q0; q < q1; ++q) {
        const uint32_t r = (uint32_t)keys[q];
        if ((q == 0 || (keys[q] >> 32) != (keys[q - 1] >> 32)) && flag[r]) {
            const int64_t s = ord[r];
            if (o < a.match_capacity) {
                a.matches[2 * o] = sid[2 * s];
                a.matches[2 * o + 1] = sid[2 * s + 1];
                a.match_scores[o] = cert[s];
            }
            ++o;
        }
    }
}

static int mg_pairs_check(const rb_match_graph_pairs_args* a, const char* what, int& in_smem) {
    RB_REQUIRE(a && a->sid && a->certainty && a->match_offsets, "%s: null argument", what);
    RB_REQUIRE(a->num_pairs > 0 && a->n > 0 && a->pair_begin >= 0 && a->pair_begin < a->pair_end && a->pair_end <= a->num_pairs,
               "%s: bad pair range [%d, %d) of %d pairs, n=%d", what, a->pair_begin, a->pair_end, a->num_pairs, a->n);
    const int64_t bytes = mg_pair_bytes(a->n);
    in_smem = bytes <= RB_MG_PAIR_SMEM;
    RB_REQUIRE(in_smem || (a->scratch && a->scratch_bytes >= bytes * (a->pair_end - a->pair_begin)),
               "%s: n=%d needs %lld scratch bytes per pair, %lld given for %d pairs", what, a->n, (long long)bytes, (long long)a->scratch_bytes,
               a->pair_end - a->pair_begin);
    return 0;
}

template <bool EMIT>
static int mg_pairs_launch(const rb_match_graph_pairs_args* a, int in_smem, cudaStream_t st) {
    const size_t smem = in_smem ? (size_t)mg_pair_bytes(a->n) : 0;
    if (ensure_smem<mg_pair_kernel<EMIT>>(RB_MG_PAIR_SMEM, "match_graph pairs")) return 1;
    launch_pdl(mg_pair_kernel<EMIT>, dim3(a->pair_end - a->pair_begin), dim3(MG_PAIR_THREADS), smem, st, *a, in_smem);
    return 0;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_match_graph_keypoints(const rb_match_graph_keypoints_args* a, void* stream) {
    RB_REQUIRE(a && a->pairs && a->matches && a->certainty && a->image_sizes && a->cell_start && a->tile_start && a->grid_bits && a->grid_g &&
               a->tile_scan && a->kp_offsets && a->keypoints && a->kp_scores && a->sid, "match_graph_keypoints: null argument");
    RB_REQUIRE(a->num_pairs > 0 && a->n > 0 && a->cell_size > 0 && a->min_certainty >= 0.f, "match_graph_keypoints: bad arguments "
               "num_pairs=%d n=%d cell_size=%d min_certainty=%g", a->num_pairs, a->n, a->cell_size, a->min_certainty);
    RB_REQUIRE(0 <= a->img_begin && a->img_begin < a->img_end && a->img_end <= a->num_images, "match_graph_keypoints: bad image group [%d, %d) of %d",
               a->img_begin, a->img_end, a->num_images);
    RB_REQUIRE(a->grid_cells >= 0 && a->grid_tiles >= 0 && a->grid_tiles < (1ll << 31), "match_graph_keypoints: bad grid of %lld cells, %lld tiles",
               (long long)a->grid_cells, (long long)a->grid_tiles);
    cudaStream_t st = (cudaStream_t)stream;
    if (a->grid_cells > 0 && (cudaMemsetAsync(a->grid_bits, 0, (size_t)a->grid_cells * 4, st) != cudaSuccess ||
                              cudaMemsetAsync(a->grid_g, 0xff, (size_t)a->grid_cells * 8, st) != cudaSuccess))
        return check_launch("match_graph_keypoints(clear grid)");
    const unsigned grid = grid1d((int64_t)a->num_pairs * a->n * 2, MG_THREADS, 16 * 1024);
    launch_pdl(mg_side_kernel<0>, dim3(grid), dim3(MG_THREADS), 0, st, *a);
    if (check_launch("match_graph_keypoints(cell maximum)")) return 1;
    launch_pdl(mg_side_kernel<1>, dim3(grid), dim3(MG_THREADS), 0, st, *a);
    if (check_launch("match_graph_keypoints(cell winner)")) return 1;
    const int tiles = (int)a->grid_tiles;
    if (tiles > 0) {
        launch_pdl(mg_tile_kernel<false>, dim3(tiles), dim3(MG_THREADS), 0, st, *a);
        if (check_launch("match_graph_keypoints(tile count)")) return 1;
    }
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->tile_scan, tiles);
    if (check_launch("match_graph_keypoints(tile scan)")) return 1;
    launch_pdl(mg_kp_offsets_kernel, dim3(1), dim3(1024), 0, st, *a);
    if (check_launch("match_graph_keypoints(offsets)")) return 1;
    if (tiles > 0) {
        launch_pdl(mg_tile_kernel<true>, dim3(tiles), dim3(MG_THREADS), 0, st, *a);
        if (check_launch("match_graph_keypoints(emit)")) return 1;
    }
    launch_pdl(mg_side_kernel<2>, dim3(grid), dim3(MG_THREADS), 0, st, *a);
    return check_launch("match_graph_keypoints(ids)");
}

extern "C" int romab200_match_graph_count(const rb_match_graph_pairs_args* a, void* stream) {
    int in_smem = 0;
    if (mg_pairs_check(a, "match_graph_count", in_smem)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    if (mg_pairs_launch<false>(a, in_smem, st) || check_launch("match_graph_count")) return 1;
    if (a->pair_end < a->num_pairs) return 0;
    launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->match_offsets, a->num_pairs);
    return check_launch("match_graph_count(scan)");
}

extern "C" int romab200_match_graph_emit(const rb_match_graph_pairs_args* a, void* stream) {
    int in_smem = 0;
    if (mg_pairs_check(a, "match_graph_emit", in_smem)) return 1;
    RB_REQUIRE(a->matches && a->match_scores, "match_graph_emit: null output");
    if (mg_pairs_launch<true>(a, in_smem, (cudaStream_t)stream)) return 1;
    return check_launch("match_graph_emit");
}
