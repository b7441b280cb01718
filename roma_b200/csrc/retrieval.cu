// Image retrieval on the device: DINOv2 global descriptors and the nearest-neighbour pair list (rules in include/romab200.h).
//   descriptor  one CTA per image, one thread per channel: class token, mean of the patch tokens in ascending token order, two
//               L2 norms summed in ascending channel order by one thread, every operation fp32 round-to-nearest, no contraction;
//   select      one CTA per row of a block of scores: exact radix select over the 48-bit key (order-preserving score bits << 16 |
//               0xffff - j) with 12-bit digits, until the keys at or above the selected digit prefix fit the shared candidate list;
//               those are collected, bitonic-sorted in shared memory and the first k written.  Keys are unique (j is part of
//               them), so ties between scores need no second pass and the result does not depend on thread timing;
//   pairs       (min, max) keys of every listed neighbour, radix_sort_hi32, adjacent duplicates dropped by a count, a scan and an
//               emit.  No float atomics anywhere.
#include "common.cuh"

namespace rb {

constexpr int DESC_THREADS = 1024;
constexpr float DESC_SQRT2 = 1.41421354f;        // fp32(sqrt(2))

// out = c / (sqrt2 * |c|), or 0 when |c| = 0.  sq: the CTA's shared squares, summed by thread 0 in ascending channel order.
__device__ __forceinline__ float desc_normalize(float v, float* sq, float* norm, int dim) {
    sq[threadIdx.x] = __fmul_rn(v, v);
    __syncthreads();
    if (threadIdx.x == 0) {
        float s = 0.f;
        for (int c = 0; c < dim; ++c) s = __fadd_rn(s, sq[c]);
        *norm = __fsqrt_rn(s);
    }
    __syncthreads();
    const float n = *norm;
    __syncthreads();                                 // sq and norm are reused by the second half
    return n == 0.f ? 0.f : __fdiv_rn(v, __fmul_rn(DESC_SQRT2, n));
}

template <typename T>
__global__ void __launch_bounds__(DESC_THREADS) global_descriptor_kernel(const T* __restrict__ tokens, int n_tokens, int dim, float* __restrict__ out) {
    rb::pdl_wait();
    __shared__ float sq[DESC_THREADS];
    __shared__ float norm;
    const int e = blockIdx.x, ch = threadIdx.x;
    const T* t = tokens + (int64_t)e * n_tokens * dim + ch;
    float c = 0.f, s = 0.f;
    if (ch < dim) {
        c = to_f(t[0]);
#pragma unroll 8
        for (int k = 1; k < n_tokens; ++k) s = __fadd_rn(s, to_f(t[(int64_t)k * dim]));
    }
    const float m = __fdiv_rn(s, (float)(n_tokens - 1));
    const float dc = desc_normalize(ch < dim ? c : 0.f, sq, &norm, dim);
    const float dm = desc_normalize(ch < dim ? m : 0.f, sq, &norm, dim);
    if (ch < dim) {
        out[(int64_t)e * 2 * dim + ch] = dc;
        out[(int64_t)e * 2 * dim + dim + ch] = dm;
    }
}

// ---- neighbour selection ------------------------------------------------------------------------------------------------------
constexpr int SEL_THREADS = 512;
constexpr int SEL_WARPS = SEL_THREADS / 32;
constexpr int SEL_BITS = 12;
constexpr int SEL_BINS = 1 << SEL_BITS;
constexpr int SEL_PER = SEL_BINS / SEL_THREADS;  // bins per thread in the crossing search
constexpr int SEL_CAND = 2048;                   // shared candidate list (16 KB)
static_assert(SEL_CAND >= 128 && (SEL_CAND & (SEL_CAND - 1)) == 0, "the candidate list holds k <= 128 keys and is bitonic-sorted");

// 48-bit key of score s at column j: the order-preserving bit pattern of s (-0 taken as +0) above 0xffff - j, so that larger keys
// come first in (score descending, j ascending).  Never 0 for j <= 65534: 0 marks the row's own column.
__device__ __forceinline__ uint64_t sel_key(float s, int j) {
    uint32_t u = __float_as_uint(s == 0.f ? 0.f : s);
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((uint64_t)u << 16) | (uint32_t)(0xffff - j);
}
__device__ __forceinline__ float sel_score(uint64_t key) {
    const uint32_t u = (uint32_t)(key >> 16);
    return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void __launch_bounds__(SEL_THREADS) retrieval_select_kernel(const float* __restrict__ S, int64_t lds, int n, int row0, int k,
                                                                      int64_t* __restrict__ neighbors, float* __restrict__ scores,
                                                                      int32_t* __restrict__ status) {
    rb::pdl_wait();
    __shared__ int hist[SEL_BINS];
    __shared__ uint64_t cand[SEL_CAND];
    __shared__ int warp_tot[SEL_WARPS];
    __shared__ int sel_bin, sel_gt, n_cand, bad;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int i = row0 + blockIdx.x;
    const float* row = S + (int64_t)blockIdx.x * lds;
    if (threadIdx.x == 0) { bad = 0; n_cand = 0; }
    uint64_t prefix = 0, mask = 0;
    int need = k, taken = 0;                         // taken: keys above the current prefix range, all selected
    for (int pass = 0; pass < 4; ++pass) {
        const int shift = 36 - SEL_BITS * pass;
        for (int b = threadIdx.x; b < SEL_BINS; b += SEL_THREADS) hist[b] = 0;
        __syncthreads();
        bool nonfinite = false;
        for (int j0 = 0; j0 < n; j0 += SEL_THREADS) {
            const int j = j0 + threadIdx.x;
            int digit = -1;
            if (j < n) {
                const float s = row[j];
                nonfinite |= !isfinite(s);
                const uint64_t key = j == i ? 0ull : sel_key(s, j);
                if ((key & mask) == prefix) digit = (int)((key >> shift) & (SEL_BINS - 1));
            }
            const unsigned peers = __match_any_sync(0xffffffffu, digit);       // one shared atomic per distinct digit of the warp
            if (digit >= 0 && __ffs(peers) - 1 == lane) atomicAdd(&hist[digit], __popc(peers));
        }
        if (pass == 0 && nonfinite) bad = 1;
        __syncthreads();
        // the bin holding the need-th largest key of the range: suffix counts over bins, thread t owning [SEL_PER t, SEL_PER (t + 1))
        int local = 0;
#pragma unroll
        for (int q = 0; q < SEL_PER; ++q) local += hist[threadIdx.x * SEL_PER + q];
        int incl = local;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, d);
            if (lane >= d) incl += u;
        }
        if (lane == 31) warp_tot[wid] = incl;
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < SEL_WARPS; ++w) {
            const int t = warp_tot[w];
            if (w < wid) before += t;
            total += t;
        }
        const int above = total - (before + incl);   // keys of the range in the bins of later threads
        if (above < need && need <= above + local) {
            int cum = above;
            for (int q = SEL_PER - 1; q >= 0; --q) {
                const int h = hist[threadIdx.x * SEL_PER + q];
                if (cum + h >= need) { sel_bin = threadIdx.x * SEL_PER + q; sel_gt = cum; break; }
                cum += h;
            }
        }
        __syncthreads();
        const int b = sel_bin, gt = sel_gt, in_bin = hist[b];
        prefix |= (uint64_t)b << shift;
        mask |= (uint64_t)(SEL_BINS - 1) << shift;
        taken += gt;
        need -= gt;
        __syncthreads();                             // hist, sel_bin and sel_gt are rewritten by the next pass
        if (taken + in_bin <= SEL_CAND) break;
    }
    // collect every key at or above the prefix range (taken + the range's keys <= SEL_CAND), in no particular order
    for (int j = threadIdx.x; j < n; j += SEL_THREADS) {
        if (j == i) continue;
        const uint64_t key = sel_key(row[j], j);
        if ((key & mask) >= prefix) cand[atomicAdd(&n_cand, 1)] = key;
    }
    __syncthreads();
    const int m = n_cand;
    int len = 1;
    while (len < m) len <<= 1;
    for (int q = m + threadIdx.x; q < len; q += SEL_THREADS) cand[q] = 0ull;
    __syncthreads();
    // bitonic sort, descending
    for (int size = 2; size <= len; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int q = threadIdx.x; q < len / 2; q += SEL_THREADS) {
                const int lo = 2 * q - (q & (stride - 1)), hi = lo + stride;
                const bool desc = (lo & size) == 0;
                const uint64_t a = cand[lo], c = cand[hi];
                if ((a < c) == desc) { cand[lo] = c; cand[hi] = a; }
            }
            __syncthreads();
        }
    }
    if (threadIdx.x < k) {
        const uint64_t key = cand[threadIdx.x];
        neighbors[(int64_t)i * k + threadIdx.x] = 0xffff - (int)(key & 0xffff);
        scores[(int64_t)i * k + threadIdx.x] = sel_score(key);
    }
    if (threadIdx.x == 0 && bad) *status = 1;
}

// ---- pair list ----------------------------------------------------------------------------------------------------------------
constexpr int PAIR_THREADS = 256;

__global__ void __launch_bounds__(PAIR_THREADS) retrieval_keys_kernel(const int64_t* __restrict__ neighbors, int64_t total, int k, int n,
                                                                    uint64_t* __restrict__ keys) {
    rb::pdl_wait();
    for (int64_t q = (int64_t)blockIdx.x * PAIR_THREADS + threadIdx.x; q < total; q += (int64_t)gridDim.x * PAIR_THREADS) {
        const int64_t i = q / k, j = neighbors[q];
        const int64_t a = i < j ? i : j, b = i < j ? j : i;
        keys[q] = (uint64_t)(a * n + b) << 32;
    }
}

// flags[q] = 1 when sorted key q differs from key q - 1 (the first of a run), scanned afterwards into offsets
__global__ void __launch_bounds__(PAIR_THREADS) retrieval_flags_kernel(const uint64_t* __restrict__ sorted, int64_t total, int64_t* __restrict__ flags) {
    rb::pdl_wait();
    for (int64_t q = (int64_t)blockIdx.x * PAIR_THREADS + threadIdx.x; q < total; q += (int64_t)gridDim.x * PAIR_THREADS)
        flags[q] = (q == 0 || (sorted[q] >> 32) != (sorted[q - 1] >> 32)) ? 1 : 0;
}

__global__ void __launch_bounds__(PAIR_THREADS) retrieval_emit_kernel(const uint64_t* __restrict__ sorted, int64_t total, int n,
                                                                    const int64_t* __restrict__ offsets, int64_t* __restrict__ pairs) {
    rb::pdl_wait();
    for (int64_t q = (int64_t)blockIdx.x * PAIR_THREADS + threadIdx.x; q < total; q += (int64_t)gridDim.x * PAIR_THREADS) {
        const int64_t o = offsets[q];
        if (offsets[q + 1] == o) continue;
        const int64_t v = (int64_t)(sorted[q] >> 32);
        pairs[2 * o] = v / n;
        pairs[2 * o + 1] = v % n;
    }
}

// bits of the largest pair key (n - 2) n + n - 1 = n^2 - n - 1, and the buffer radix_sort_hi32 leaves the sorted keys in
static int pair_key_bits(int n) {
    const uint64_t top = (uint64_t)n * n - n - 1;
    int bits = 1;
    while (bits < 32 && (top >> bits)) ++bits;
    return bits;
}
static uint64_t* pair_sorted(const rb_retrieval_args* a) {
    const int passes = (pair_key_bits(a->num_images) + 7) / 8;
    return (uint64_t*)(passes % 2 ? a->keys_alt : a->keys);
}

static int retrieval_check(const rb_retrieval_args* a, const char* what) {
    RB_REQUIRE(a && a->neighbors, "%s: null argument", what);
    RB_REQUIRE(a->num_images >= 2 && a->num_images <= RB_RETRIEVAL_MAX_IMAGES, "%s: num_images %d outside [2, %d]", what, a->num_images,
               RB_RETRIEVAL_MAX_IMAGES);
    RB_REQUIRE(a->k >= 1 && a->k <= RB_RETRIEVAL_MAX_K && a->k <= a->num_images - 1, "%s: k %d outside [1, min(%d, num_images - 1)]", what, a->k,
               RB_RETRIEVAL_MAX_K);
    return 0;
}

static unsigned pair_grid(int64_t total) { return grid1d(total, PAIR_THREADS, 4096); }

}  // namespace rb

using namespace rb;

extern "C" int romab200_global_descriptor(const rb_global_descriptor_args* a, void* stream) {
    RB_REQUIRE(a && a->tokens && a->out, "global_descriptor: null argument");
    RB_REQUIRE(a->batch >= 1 && a->batch <= 65535 && a->n_tokens >= 2 && a->dim >= 1 && a->dim <= DESC_THREADS,
               "global_descriptor: bad shape batch=%d n_tokens=%d dim=%d (dim <= %d)", a->batch, a->n_tokens, a->dim, DESC_THREADS);
    return with_dtype<float, __half, __nv_bfloat16>(a->tokens_dtype, "global_descriptor", [&](auto tag) {
        using T = typename decltype(tag)::type;
        rb::launch_pdl(global_descriptor_kernel<T>, dim3(a->batch), dim3(DESC_THREADS), 0, (cudaStream_t)stream, (const T*)a->tokens, a->n_tokens,
                       a->dim, a->out);
        return check_launch("global_descriptor");
    });
}

extern "C" int romab200_retrieval_select(const rb_retrieval_args* a, void* stream) {
    if (retrieval_check(a, "retrieval_select")) return 1;
    RB_REQUIRE(a->scores && a->neighbor_scores && a->status, "retrieval_select: null argument");
    RB_REQUIRE(a->row_begin >= 0 && a->row_begin < a->row_end && a->row_end <= a->num_images && a->ld_scores >= a->num_images,
               "retrieval_select: rows [%d, %d) of %d images, ld_scores %lld", a->row_begin, a->row_end, a->num_images, (long long)a->ld_scores);
    rb::launch_pdl(retrieval_select_kernel, dim3(a->row_end - a->row_begin), dim3(SEL_THREADS), 0, (cudaStream_t)stream, a->scores, a->ld_scores,
                   a->num_images, a->row_begin, a->k, a->neighbors, a->neighbor_scores, a->status);
    return check_launch("retrieval_select");
}

extern "C" int romab200_retrieval_pairs_count(const rb_retrieval_args* a, void* stream) {
    if (retrieval_check(a, "retrieval_pairs_count")) return 1;
    RB_REQUIRE(a->keys && a->keys_alt && a->hist && a->offsets, "retrieval_pairs_count: null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t total = (int64_t)a->num_images * a->k;
    rb::launch_pdl(retrieval_keys_kernel, dim3(pair_grid(total)), dim3(PAIR_THREADS), 0, st, (const int64_t*)a->neighbors, total, a->k, a->num_images,
                   (uint64_t*)a->keys);
    if (check_launch("retrieval_pairs_count(keys)")) return 1;
    uint64_t* sorted = nullptr;
    if (radix_sort_hi32<RB_RETRIEVAL_TILE>((uint64_t*)a->keys, (uint64_t*)a->keys_alt, a->hist, total, pair_key_bits(a->num_images), st,
                                           "retrieval_pairs_count(sort)", &sorted))
        return 1;
    RB_REQUIRE(sorted == pair_sorted(a), "retrieval_pairs_count: sorted keys in an unexpected buffer");
    rb::launch_pdl(retrieval_flags_kernel, dim3(pair_grid(total)), dim3(PAIR_THREADS), 0, st, (const uint64_t*)sorted, total, a->offsets);
    if (check_launch("retrieval_pairs_count(flags)")) return 1;
    rb::launch_pdl(scan_counts_kernel<int64_t>, dim3(1), dim3(1024), 0, st, a->offsets, (int)total);
    return check_launch("retrieval_pairs_count(scan)");
}

extern "C" int romab200_retrieval_pairs_emit(const rb_retrieval_args* a, void* stream) {
    if (retrieval_check(a, "retrieval_pairs_emit")) return 1;
    RB_REQUIRE(a->keys && a->keys_alt && a->offsets && a->pairs, "retrieval_pairs_emit: null argument");
    const int64_t total = (int64_t)a->num_images * a->k;
    rb::launch_pdl(retrieval_emit_kernel, dim3(pair_grid(total)), dim3(PAIR_THREADS), 0, (cudaStream_t)stream, (const uint64_t*)pair_sorted(a), total,
                   a->num_images, (const int64_t*)a->offsets, a->pairs);
    return check_launch("retrieval_pairs_emit");
}
