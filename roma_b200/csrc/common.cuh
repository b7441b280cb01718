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
__host__ __device__ __forceinline__ int dtype_size(int dtype) { return dtype == RB_F32 ? 4 : 2; }

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

int gemm_simt(const rb_gemm_args* a, cudaStream_t stream, int lower_only = 0);
int gemm_tc(const rb_gemm_args* a, cudaStream_t stream);
int dwconv_tma(const rb_dwconv_args* a, cudaStream_t stream);     // dwconv_tma.cu: TMA-fed persistent depthwise kernel (16-bit maps)
Epilogue make_epilogue(const rb_gemm_args* a);
int split_f16s_batched(const float* x, void* hi, void* lo, int64_t rows, int cols, int64_t ldx, int64_t ldd, int batch, int64_t sx, int64_t sd, cudaStream_t st);

}  // namespace rb
