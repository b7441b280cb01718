// Shared helpers for libromab200 kernels (sm_90a only).
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <type_traits>
#include <math_constants.h>
#include "../../include/romab200.h"

namespace rb {

void set_error(const char* fmt, ...);
int check_launch(const char* what);

#define RB_REQUIRE(cond, ...)                         \
    do {                                              \
        if (!(cond)) {                                \
            rb::set_error(__VA_ARGS__);               \
            return 1;                                 \
        }                                             \
    } while (0)

template <typename T> struct DT;
template <> struct DT<float> { static constexpr int id = RB_F32; };
template <> struct DT<__half> { static constexpr int id = RB_F16; };
template <> struct DT<__nv_bfloat16> { static constexpr int id = RB_BF16; };
template <> struct DT<double> { static constexpr int id = RB_F64; };

// Dtype dispatch of the entry points: returns f(type_tag<T>{}) for the T among Ts whose code is `code`; any other code is refused
// with "<what>: unsupported dtype <code>" and 1.  List exactly the types the caller has kernels for: a generic lambda instantiates
// its body (and the kernels it launches) once per listed type.
template <typename T> struct type_tag { using type = T; };
template <typename... Ts, typename F>
inline int with_dtype(int code, const char* what, F&& f) {
    int rc = 0;
    if (((code == DT<Ts>::id ? (rc = f(type_tag<Ts>{}), true) : false) || ...)) return rc;
    set_error("%s: unsupported dtype %d", what, code);
    return 1;
}
// the same refusal for kernels that take the code itself and convert at run time
template <typename... Ts>
inline int check_dtype(int code, const char* what) { return with_dtype<Ts...>(code, what, [](auto) { return 0; }); }

// The same for an integer template parameter (window radius, lanes per pixel): f(std::integral_constant<int, V>{}) for the V among
// Vs equal to v; any other value: "<what> <v> unsupported (<Vs>)", 1.
template <int... Vs, typename F>
inline int with_value(int v, const char* what, F&& f) {
    int rc = 0;
    if (((v == Vs ? (rc = f(std::integral_constant<int, Vs>{}), true) : false) || ...)) return rc;
    const int vs[] = {Vs...};
    char list[64] = "";
    for (int i = 0, n = 0; i < (int)sizeof...(Vs); ++i) n += snprintf(list + n, sizeof(list) - n, i ? ", %d" : "%d", vs[i]);
    set_error("%s %d unsupported (%s)", what, v, list);
    return 1;
}

// 1-D grid of `block`-thread CTAs over `total` elements: at least one CTA and at most `cap` (the kernels loop over the rest)
inline unsigned grid1d(int64_t total, int block, int64_t cap) {
    const int64_t g = (total + block - 1) / block;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}

__device__ __forceinline__ float to_f(float v) { return v; }
__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_f<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_f<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float load_any(const void* p, int64_t i, int dtype) {
    if (dtype == RB_F32) return ((const float*)p)[i];
    if (dtype == RB_F16) return __half2float(((const __half*)p)[i]);
    return __bfloat162float(((const __nv_bfloat16*)p)[i]);
}
__device__ __forceinline__ void store_any(void* p, int64_t i, int dtype, float v) {
    if (dtype == RB_F32) ((float*)p)[i] = v;
    else if (dtype == RB_F16) ((__half*)p)[i] = __float2half_rn(v);
    else ((__nv_bfloat16*)p)[i] = __float2bfloat16_rn(v);
}

// Philox4x32-10 (Salmon et al. 2011, Random123): the four output words of counter c under key (k0, k1)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c.x, p1 = (uint64_t)0xCD9E8D57u * c.z;
        c = make_uint4((uint32_t)(p1 >> 32) ^ c.y ^ k0, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k1, (uint32_t)p0);
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return c;
}

// bytes per element of one plane (RB_F16S = two fp16 planes of the same pitch)
__host__ __device__ __forceinline__ int dtype_size(int dtype) { return dtype == RB_F64 ? 8 : (dtype == RB_F32 ? 4 : 2); }

// ---- split-fp16 pair: x ~ hi + lo * 2^-11 with hi = fp16(x), lo = fp16((x - hi) * 2^11) -------------------------------
// 22 significand bits, the exponent range of fp16, and no underflow of the low part (it is stored at the magnitude of x).
// Re-splitting a reconstructed value is exact, so kernels may pass maps through unchanged (max-pool, copies).
constexpr float RB_SPLIT_SCALE = 2048.0f;
__device__ __forceinline__ void split_f16s(float x, __half& hi, __half& lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn((x - __half2float(hi)) * RB_SPLIT_SCALE);
}
__device__ __forceinline__ float join_f16s(__half hi, __half lo) { return fmaf(__half2float(lo), 1.0f / RB_SPLIT_SCALE, __half2float(hi)); }
// stores `v` as `dtype` at element i of p (and of p_lo for RB_F16S)
__device__ __forceinline__ void store_split_any(void* p, void* p_lo, int64_t i, int dtype, float v) {
    if (dtype == RB_F16S) {
        __half hi, lo;
        split_f16s(v, hi, lo);
        ((__half*)p)[i] = hi; ((__half*)p_lo)[i] = lo;
    } else {
        store_any(p, i, dtype, v);
    }
}
inline int current_device() { int d = 0; cudaGetDevice(&d); return d; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// two independent fp32 FMAs on a channel pair (c + a * b per component, round-to-nearest)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }

// exact-erf GELU (nn.GELU default, mlp.py:26)
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }

// ------------------------------------------------------------------------------------------------
// GEMM epilogue shared by the SIMT and tensor-core back-ends
// ------------------------------------------------------------------------------------------------
struct Epilogue {
    void* C; void* C_lo; int64_t ldc; int dtype_c;
    float alpha;
    const float* bias; const float* col_scale;
    const void* R; int64_t ldr; int dtype_r;
    int act, epi;
    const float* norm_a; const float* norm_b;
    float eps, inv_t, diag_add; int cos_normalized;
    int rowmap, pad_h, pad_w, seg_in, seg_out, seg_off;
    int M, N;

    // maps the logical row m to the stored row, or -1 when the row is not stored
    __device__ __forceinline__ int64_t map_row(int m) const {
        if (rowmap == RB_ROWMAP_NONE) return m;
        if (rowmap == RB_ROWMAP_SEGMENT) return (int64_t)(m / seg_in) * seg_out + (m % seg_in) + seg_off;
        int plane = pad_h * pad_w;
        int img = m / plane, rem = m - img * plane;
        int yp = rem / pad_w, xp = rem - yp * pad_w;
        if (yp == 0 || xp == 0 || yp == pad_h - 1 || xp == pad_w - 1) return -1;
        if (rowmap == RB_ROWMAP_PAD_KEEP) return m;
        return (int64_t)img * (pad_h - 2) * (pad_w - 2) + (int64_t)(yp - 1) * (pad_w - 2) + (xp - 1);
    }
    __device__ __forceinline__ float apply(float acc, int m, int n, int64_t orow) const {
        float v;
        if (epi == RB_EPI_COSKERNEL) {
            float p = norm_a[m] * norm_b[n];
            float s = cos_normalized ? p / (p + eps) : 1.0f / (p + eps);
            v = expf((acc * s - 1.0f) * inv_t);
            if (m == n) v += diag_add;
            return v;
        }
        v = alpha * acc;
        if (bias) v += bias[n];
        if (act == RB_ACT_RELU) v = fmaxf(v, 0.0f);
        else if (act == RB_ACT_GELU) v = gelu_erf(v);
        if (col_scale) v *= col_scale[n];
        if (R) v += load_any(R, orow * ldr + n, dtype_r);
        return v;
    }
    __device__ __forceinline__ void store(float acc, int m, int n) const {
        if (m >= M || n >= N) return;
        int64_t orow = map_row(m);
        if (orow < 0) return;
        store_split_any(C, C_lo, orow * ldc + n, dtype_c, apply(acc, m, n, orow));
    }
};

// ------------------------------------------------------------------------------------------------
// Programmatic dependent launch: every kernel of the library is launched with the stream-serialization attribute and
// starts with pdl_wait(), so that its launch latency and per-CTA set-up overlap the tail of the previous kernel in the
// stream (the ~680 launches of one match() are otherwise separated by a few microseconds each).
// ------------------------------------------------------------------------------------------------
// No early griddepcontrol.launch_dependents: the next grid's CTAs would take SM slots and issue bandwidth while they spin in
// their wait; the implicit trigger at grid exit already hides the launch.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// ROMAB200_NO_PDL=1 launches every kernel fully serialised (debugging knob; griddepcontrol.* are no-ops then)
inline int pdl_mode() { static const int m = [] { const char* e = getenv("ROMAB200_NO_PDL"); return e ? atoi(e) : 0; }(); return m; }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl_mode() ? 0 : 1;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// In place: v[0..n) counts -> exclusive prefix sums, v[n] = total.  One CTA of 1024 threads, a contiguous chunk per thread.  A
// template so that every translation unit that launches it carries its own copy.
template <typename T>
__global__ void __launch_bounds__(1024) scan_counts_kernel(T* __restrict__ v, int n) {
    pdl_wait();
    __shared__ T warp_tot[32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int per = (n + 1023) / 1024;
    const int b = min(n, (int)threadIdx.x * per), e = min(n, b + per);
    T s = 0;
    for (int k = b; k < e; ++k) s += v[k];
    T incl = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T u = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += u;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        const T t = warp_tot[lane];
        T wi = t;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const T u = __shfl_up_sync(0xffffffffu, wi, d);
            if (lane >= d) wi += u;
        }
        warp_tot[lane] = wi - t;
    }
    __syncthreads();
    T run = warp_tot[wid] + incl - s;
    for (int k = b; k < e; ++k) {
        const T c = v[k];
        v[k] = run;
        run += c;
    }
    if (threadIdx.x == 1023) v[n] = run;
}

// Exp(w) by Rodrigues (bundle rule 3, absolute-pose rule 5), with the small-angle branch I + [w]x for theta^2 <= 2^-52
__device__ __forceinline__ void so3_exp(const double (&w)[3], double (&E)[3][3]) {
    const double t2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    if (t2 > 0x1p-52) {
        const double th = sqrt(t2), k0 = w[0] / th, k1 = w[1] / th, k2 = w[2] / th;
        double s, c;
        sincospi(th * (1.0 / CUDART_PI), &s, &c);      // sincospi: its argument reduction is exact and needs no stack
        const double c1 = 1.0 - c;
        E[0][0] = c + c1 * k0 * k0;      E[0][1] = c1 * k0 * k1 - s * k2; E[0][2] = c1 * k0 * k2 + s * k1;
        E[1][0] = c1 * k1 * k0 + s * k2; E[1][1] = c + c1 * k1 * k1;      E[1][2] = c1 * k1 * k2 - s * k0;
        E[2][0] = c1 * k2 * k0 - s * k1; E[2][1] = c1 * k2 * k1 + s * k0; E[2][2] = c + c1 * k2 * k2;
    } else {
        E[0][0] = 1.0;   E[0][1] = -w[2]; E[0][2] = w[1];
        E[1][0] = w[2];  E[1][1] = 1.0;   E[1][2] = -w[0];
        E[2][0] = -w[1]; E[2][1] = w[0];  E[2][2] = 1.0;
    }
}

// ---- stable LSD radix sort of 64-bit keys by their high 32 bits, 8-bit digits, tiles of TILE keys --------------------------------
// Templates, so that every translation unit that launches them carries its own copy.
constexpr int RADIX_THREADS = 256;
constexpr int RADIX_WARPS = RADIX_THREADS / 32;
constexpr int RADIX_DIGITS = 256;
static_assert(RADIX_DIGITS == RADIX_THREADS, "the radix kernels give one digit to each thread");

// hist[d * tiles + t] = keys of tile t whose high word has digit d at `shift`
template <int TILE>
__global__ void __launch_bounds__(RADIX_THREADS) radix_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift, int32_t* hist) {
    pdl_wait();
    __shared__ int h[RADIX_DIGITS];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t q0 = (int64_t)blockIdx.x * TILE;
    for (int k = 0; k < TILE / RADIX_THREADS; ++k) {
        const int64_t q = q0 + k * RADIX_THREADS + threadIdx.x;
        if (q < n) atomicAdd(&h[(keys[q] >> (32 + shift)) & (RADIX_DIGITS - 1)], 1);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// Stable scatter of tile t: rounds of RADIX_THREADS consecutive keys; within a warp, the rank among equal digits from
// __match_any_sync; across warps and rounds, a running offset per digit that starts at the scanned hist entry of (digit, tile).
template <int TILE>
__global__ void __launch_bounds__(RADIX_THREADS) radix_scatter_kernel(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, int64_t n,
                                                                      int shift, const int32_t* __restrict__ hist) {
    pdl_wait();
    __shared__ int base[RADIX_DIGITS];
    __shared__ int wcnt[RADIX_WARPS][RADIX_DIGITS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    base[threadIdx.x] = hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x];
    const int64_t q0 = (int64_t)blockIdx.x * TILE;
    for (int k = 0; k < TILE / RADIX_THREADS; ++k) {
#pragma unroll
        for (int w = 0; w < RADIX_WARPS; ++w) wcnt[w][threadIdx.x] = 0;
        __syncthreads();
        const int64_t q = q0 + k * RADIX_THREADS + threadIdx.x;
        const bool valid = q < n;
        const uint64_t key = valid ? in[q] : 0;
        const int d = valid ? (int)((key >> (32 + shift)) & (RADIX_DIGITS - 1)) : RADIX_DIGITS;
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (valid && rank == 0) wcnt[wid][d] = __popc(peers);
        __syncthreads();
        int run = base[threadIdx.x];                     // column of digit threadIdx.x: exclusive over the warps, from base
#pragma unroll
        for (int w = 0; w < RADIX_WARPS; ++w) {
            const int c = wcnt[w][threadIdx.x];
            wcnt[w][threadIdx.x] = run;
            run += c;
        }
        base[threadIdx.x] = run;
        __syncthreads();
        if (valid) out[wcnt[wid][d] + rank] = key;
        __syncthreads();
    }
}

// Sorts keys[0, n) stably by the low `bits` bits of their high words, ping-ponging between keys and keys_alt; hist holds
// RADIX_DIGITS ceil(n / TILE) + 1 ints.  *sorted receives the buffer that holds the result.  0, or 1 after a failed launch.
template <int TILE>
inline int radix_sort_hi32(uint64_t* keys, uint64_t* keys_alt, int32_t* hist, int64_t n, int bits, cudaStream_t st, const char* what,
                           uint64_t** sorted) {
    const int tiles = (int)((n + TILE - 1) / TILE);
    uint64_t* in = keys;
    uint64_t* out = keys_alt;
    for (int shift = 0; shift < bits; shift += 8) {
        launch_pdl(radix_hist_kernel<TILE>, dim3(tiles), dim3(RADIX_THREADS), 0, st, (const uint64_t*)in, n, shift, hist);
        if (check_launch(what)) return 1;
        launch_pdl(scan_counts_kernel<int32_t>, dim3(1), dim3(1024), 0, st, hist, RADIX_DIGITS * tiles);
        if (check_launch(what)) return 1;
        launch_pdl(radix_scatter_kernel<TILE>, dim3(tiles), dim3(RADIX_THREADS), 0, st, (const uint64_t*)in, out, n, shift, (const int32_t*)hist);
        if (check_launch(what)) return 1;
        uint64_t* t = in;
        in = out;
        out = t;
    }
    *sorted = in;
    return 0;
}

int gemm_simt(const rb_gemm_args* a, cudaStream_t stream, int lower_only = 0);
int gemm_tc(const rb_gemm_args* a, cudaStream_t stream);
int dwconv_tma(const rb_dwconv_args* a, cudaStream_t stream);     // dwconv_tma.cu: TMA-fed persistent depthwise kernel (16-bit maps)
Epilogue make_epilogue(const rb_gemm_args* a);
int split_f16s_batched(const float* x, void* hi, void* lo, int64_t rows, int cols, int64_t ldx, int64_t ldd, int batch, int64_t sx, int64_t sd, cudaStream_t st);

}  // namespace rb
