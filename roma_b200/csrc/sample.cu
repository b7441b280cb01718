// Weighted sampling without replacement on the device — the two `torch.multinomial(..., replacement=False)` draws of
// `RegressionMatcher.sample` (romatch/models/matcher.py:613-617, 626-628), SURVEY 8f-1.
//
// Exponential race (Efraimidis-Spirakis): key_i = -log(u_i) / w_i with u_i ~ U(0,1); the k smallest keys are a draw of k items
// without replacement with probabilities proportional to w (the same construction torch.multinomial uses on CUDA: w / Exp(1),
// top-k).  Grid-wide kernels (a single CTA needs 0.6 ms for the 1.5 M keys of one pair):
//   keys     from a counter-based generator (Philox4x32-10 keyed by the seed, counter = element index), written to the
//            workspace; the weight transform of the caller is applied on the fly (certainty threshold / density balancing), so
//            no intermediate tensor is materialised; the histogram of bits [31:21] is accumulated on the way;
//   select   (one CTA per batch item, three times) radix select of the k-th smallest key over bits [31:21], [20:10], [9:0] of
//            the (order-preserving) bit pattern of the positive float keys; `hist` re-histograms the surviving candidates;
//            then three more times over the bits of the INDICES of the keys equal to the k-th one, so that ties at the cut are
//            resolved by index (smallest first) and the drawn set does not depend on thread timing;
//   compact  indices of all keys below the k-th one and of the tied keys up to the selected index (in no particular order).
// The keys of a 1.5 M-pixel certainty map are 6 MB: L2-resident across the passes.  Items of zero weight have key = +inf and are
// only drawn when fewer than k positive weights exist.
#include "common.cuh"

namespace rb {

// Philox4x32-10: counter (c0, c1, 0, 0), key (k0, k1); returns the first output word
__device__ __forceinline__ uint32_t philox_u32(uint32_t c0, uint32_t c1, uint32_t k0, uint32_t k1) {
    return philox4x32_10(make_uint4(c0, c1, 0u, 0u), k0, k1).x;
}

// weight transforms (matcher.py:604-607, 622-625)
__device__ __forceinline__ float sample_weight(float v, int transform, float param) {
    if (transform == RB_SAMPLE_THRESHOLD) return v > param ? 1.0f : v;                       // certainty[certainty > thresh] = 1
    if (transform == RB_SAMPLE_BALANCE) return v < 10.0f ? 1e-7f : 1.0f / (v + 1.0f);        // p = 1/(density+1); p[density < 10] = 1e-7
    return v;
}

constexpr int SMP_THREADS = 256;
constexpr int SMP_BINS = 2048;
// scratch layout per batch item (int32 words): [0, 2048) histogram, 2048: prefix, 2049: need, 2050: mask, 2051: output count,
// 2053: the k-th smallest key (set by the last key pass).  Passes 0-2 select over key bits, passes 3-5 over index bits of the ties.
constexpr int SMP_SCRATCH = SMP_BINS + 8;
constexpr int SMP_PASSES = 6;

__device__ __forceinline__ void flush_hist(uint32_t* smem_hist, uint32_t* gh, int bins) {
    __syncthreads();
    for (int i = threadIdx.x; i < bins; i += blockDim.x) {
        const uint32_t c = smem_hist[i];
        if (c) atomicAdd(&gh[i], c);
    }
}

// pass 0: keys (grid-wide) + histogram of bits [31:21]
// item b: seed from seed_dev[b * seed_stride] (own seed, key as a batch-1 call with it) or, with seed_stride = 0, the shared seed with
// b mixed into the key; weights from row b / repeats of `values` (the `repeats` draws of one pair read one map)
__global__ void __launch_bounds__(SMP_THREADS) sample_keys_kernel(const float* __restrict__ values, int64_t n, int64_t stride, uint64_t seed, const uint64_t* __restrict__ seed_dev,
                                                                  int64_t seed_stride, int repeats, int transform, float param, float* __restrict__ keys_ws,
                                                                  uint32_t* __restrict__ scratch) {
    rb::pdl_wait();
    __shared__ uint32_t hist[SMP_BINS];
    const int b = blockIdx.y;
    if (seed_dev) seed = seed_dev[(int64_t)b * seed_stride];
    for (int i = threadIdx.x; i < SMP_BINS; i += SMP_THREADS) hist[i] = 0;
    __syncthreads();
    const float* v = values + (int64_t)(b / repeats) * stride;
    float* keys = keys_ws + (int64_t)b * n;
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32) ^ (seed_stride ? 0u : (uint32_t)b * 0x9E3779B9u);
    for (int64_t i = (int64_t)blockIdx.x * SMP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * SMP_THREADS) {
        const float w = sample_weight(v[i], transform, param);
        const uint32_t r = philox_u32((uint32_t)i, (uint32_t)(i >> 32), k0, k1);
        const float u = ((float)(r >> 8) + 0.5f) * (1.0f / 16777216.0f);          // (0, 1), 24 random bits
        const float key = w > 0.f ? -__logf(u) / w : __int_as_float(0x7f800000);
        keys[i] = key;
        atomicAdd(&hist[__float_as_uint(key) >> 21], 1u);
    }
    flush_hist(hist, scratch + (int64_t)b * SMP_SCRATCH, SMP_BINS);
}

// between the passes: one CTA per batch item finds the bin holding the `need`-th smallest candidate, extends the prefix, clears the histogram
__global__ void __launch_bounds__(SMP_THREADS) sample_select_kernel(uint32_t* __restrict__ scratch, int pass, int k) {
    rb::pdl_wait();
    __shared__ uint32_t part[SMP_THREADS];
    uint32_t* sc = scratch + (int64_t)blockIdx.x * SMP_SCRATCH;
    const int shifts[3] = {21, 10, 0}, nbits[3] = {11, 11, 10};
    const int sh = shifts[pass % 3], bins = 1 << nbits[pass % 3];
    const bool first = pass % 3 == 0;                  // a new radix select starts: empty prefix / mask
    const uint32_t need = pass == 0 ? (uint32_t)k : sc[SMP_BINS + 1];
    // 8 consecutive bins per thread: local sums, scan of the 256 partial sums, then the thread that holds the crossing finds the bin
    constexpr int PER = SMP_BINS / SMP_THREADS;
    uint32_t local[PER], sum = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) { const int i = threadIdx.x * PER + j; local[j] = i < bins ? sc[i] : 0u; sum += local[j]; }
    part[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t run = 0;
        for (int t = 0; t < SMP_THREADS; ++t) { const uint32_t c = part[t]; part[t] = run; run += c; }     // exclusive scan (256 steps)
    }
    __syncthreads();
    const uint32_t before = part[threadIdx.x];
    if (before < need && need <= before + sum) {
        uint32_t cum = before;
#pragma unroll
        for (int j = 0; j < PER; ++j) {
            if (cum + local[j] >= need) {
                const uint32_t prefix = (first ? 0u : sc[SMP_BINS]) | ((uint32_t)(threadIdx.x * PER + j) << sh);
                const uint32_t mask = (first ? 0u : sc[SMP_BINS + 2]) | ((uint32_t)(bins - 1) << sh);
                sc[SMP_BINS] = prefix; sc[SMP_BINS + 1] = need - cum; sc[SMP_BINS + 2] = mask;
                if (pass == 2) sc[SMP_BINS + 5] = prefix;     // the k-th smallest key; need - cum of its ties are drawn
                break;
            }
            cum += local[j];
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < SMP_BINS; i += SMP_THREADS) sc[i] = 0;
    if (threadIdx.x == 0) sc[SMP_BINS + 3] = 0;
}

// passes 1, 2: histogram of the next key bits over the candidates (keys whose masked bits equal the prefix); passes 3-5: histogram
// of the index bits of the keys equal to the k-th one (whose masked index bits equal the prefix; none masked in pass 3)
__global__ void __launch_bounds__(SMP_THREADS) sample_hist_kernel(const float* __restrict__ keys_ws, int64_t n, uint32_t* __restrict__ scratch, int pass) {
    rb::pdl_wait();
    __shared__ uint32_t hist[SMP_BINS];
    const int b = blockIdx.y;
    uint32_t* sc = scratch + (int64_t)b * SMP_SCRATCH;
    for (int i = threadIdx.x; i < SMP_BINS; i += SMP_THREADS) hist[i] = 0;
    __syncthreads();
    const bool ties = pass >= 3;
    const uint32_t prefix = pass == 3 ? 0u : sc[SMP_BINS], mask = pass == 3 ? 0u : sc[SMP_BINS + 2], kth = sc[SMP_BINS + 5];
    const int shifts[3] = {21, 10, 0};
    const int sh = shifts[pass % 3], bins = pass % 3 == 2 ? 1024 : 2048;
    const float* keys = keys_ws + (int64_t)b * n;
    for (int64_t i = (int64_t)blockIdx.x * SMP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * SMP_THREADS) {
        const uint32_t x = __float_as_uint(keys[i]);
        if (!ties) {
            if ((x & mask) == prefix) atomicAdd(&hist[(x >> sh) & (bins - 1)], 1u);
        } else if (x == kth && ((uint32_t)i & mask) == prefix) {
            atomicAdd(&hist[((uint32_t)i >> sh) & (bins - 1)], 1u);
        }
    }
    flush_hist(hist, sc, bins);
}

// compaction: every key below the k-th smallest, and the ties up to the selected index
__global__ void __launch_bounds__(SMP_THREADS) sample_compact_kernel(const float* __restrict__ values, const float* __restrict__ keys_ws, int64_t n, int k, int64_t stride,
                                                                     int repeats, int transform, float param, uint32_t* __restrict__ scratch,
                                                                     int32_t* __restrict__ out_idx, float* __restrict__ out_w) {
    rb::pdl_wait();
    const int b = blockIdx.y;
    uint32_t* sc = scratch + (int64_t)b * SMP_SCRATCH;
    const uint32_t kth = sc[SMP_BINS + 5], last_tie = sc[SMP_BINS];
    const float* keys = keys_ws + (int64_t)b * n;
    const float* v = values + (int64_t)(b / repeats) * stride;
    for (int64_t i = (int64_t)blockIdx.x * SMP_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * SMP_THREADS) {
        const uint32_t x = __float_as_uint(keys[i]);
        const bool take = x < kth || (x == kth && (uint32_t)i <= last_tie);
        if (take) {
            const uint32_t pos = atomicAdd(&sc[SMP_BINS + 3], 1u);
            if (pos < (uint32_t)k) {
                out_idx[(int64_t)b * k + pos] = (int32_t)i;
                if (out_w) out_w[(int64_t)b * k + pos] = sample_weight(v[i], transform, param);
            }
        }
    }
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_weighted_sample(const rb_sample_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->values && a->out_idx && a->keys && a->scratch, "weighted_sample: null argument");
    RB_REQUIRE(a->n > 0 && a->k > 0 && a->k <= a->n && a->n < (1ll << 31) && a->batch > 0 && a->batch <= 65535, "weighted_sample: bad shape n=%lld k=%d batch=%d",
               (long long)a->n, a->k, a->batch);
    RB_REQUIRE(a->transform >= RB_SAMPLE_IDENTITY && a->transform <= RB_SAMPLE_BALANCE, "weighted_sample: unknown transform %d", a->transform);
    RB_REQUIRE(a->seed_stride >= 0 && (a->seed_stride == 0 || a->seed_dev), "weighted_sample: seed_stride %lld needs seed_dev", (long long)a->seed_stride);
    RB_REQUIRE(a->repeats >= 0, "weighted_sample: repeats %d < 0", a->repeats);
    const int repeats = a->repeats > 0 ? a->repeats : 1;
    uint32_t* scratch = reinterpret_cast<uint32_t*>(a->scratch);
    RB_REQUIRE(cudaMemsetAsync(scratch, 0, (size_t)a->batch * SMP_SCRATCH * sizeof(uint32_t), st) == cudaSuccess, "weighted_sample: memset failed");
    const int64_t stride = a->stride > 0 ? a->stride : a->n;
    int gx = (int)((a->n + SMP_THREADS * 8 - 1) / (SMP_THREADS * 8));
    if (gx > 592) gx = 592;
    if (gx < 1) gx = 1;
    const dim3 grid(gx, a->batch);
    rb::launch_pdl(sample_keys_kernel, grid, dim3(SMP_THREADS), 0, st, a->values, a->n, stride, a->seed, a->seed_dev, a->seed_stride, repeats, a->transform,
                   a->param, a->keys, scratch);
    if (check_launch("weighted_sample(keys)")) return 1;
    for (int pass = 0; pass < SMP_PASSES; ++pass) {
        rb::launch_pdl(sample_select_kernel, dim3(a->batch), dim3(SMP_THREADS), 0, st, scratch, pass, a->k);
        if (check_launch("weighted_sample(select)")) return 1;
        if (pass < SMP_PASSES - 1) {
            rb::launch_pdl(sample_hist_kernel, grid, dim3(SMP_THREADS), 0, st, (const float*)a->keys, a->n, scratch, pass + 1);
            if (check_launch("weighted_sample(hist)")) return 1;
        }
    }
    rb::launch_pdl(sample_compact_kernel, grid, dim3(SMP_THREADS), 0, st, a->values, (const float*)a->keys, a->n, a->k, stride, repeats, a->transform, a->param, scratch,
                   a->out_idx, a->out_weights);
    return check_launch("weighted_sample(compact)");
}

namespace rb {

// out[item, j] = row idx[item, j] of pair item / repeats; the certainty thresholded as `c > thresh ? 1 : c` when `threshold`
__global__ void __launch_bounds__(256) sample_gather_kernel(const float4* __restrict__ matches, const float* __restrict__ certainty, int64_t n,
                                                            const int32_t* __restrict__ idx, int64_t total, int k, int repeats, int threshold, float thresh,
                                                            float4* __restrict__ out_m, float* __restrict__ out_c) {
    rb::pdl_wait();
    for (int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x; t < total; t += (int64_t)gridDim.x * 256) {
        const int64_t row = (int64_t)((int)(t / k) / repeats) * n + idx[t];
        const float c = certainty[row];
        out_m[t] = matches[row];
        out_c[t] = threshold && c > thresh ? 1.0f : c;
    }
}

}  // namespace rb

extern "C" int romab200_sample_gather(const rb_sample_gather_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->matches && a->certainty && a->idx && a->out_matches && a->out_certainty, "sample_gather: null argument");
    RB_REQUIRE(a->n > 0 && a->k > 0 && a->items > 0 && a->repeats >= 0, "sample_gather: bad shape n=%lld k=%d items=%d repeats=%d", (long long)a->n, a->k,
               a->items, a->repeats);
    RB_REQUIRE(((uintptr_t)a->matches | (uintptr_t)a->out_matches) % 16 == 0, "sample_gather: matches and out_matches must be 16-byte aligned");
    const int64_t total = (int64_t)a->items * a->k;
    int64_t blocks = (total + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    rb::launch_pdl(sample_gather_kernel, dim3((unsigned)blocks), dim3(256), 0, st, (const float4*)a->matches, a->certainty, a->n, a->idx, total, a->k,
                   a->repeats > 0 ? a->repeats : 1, a->threshold, a->thresh, (float4*)a->out_matches, a->out_certainty);
    return check_launch("sample_gather");
}
