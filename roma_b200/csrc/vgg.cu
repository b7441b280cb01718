// VGG19-BN pieces that are not GEMMs (romatch/models/encoders.py:17-27):
//   * the first 3->64 convolution (K = 27 is too thin for a GEMM tile): direct conv from the NCHW fp32
//     image into the zero-padded channels-last layout every later 3x3 layer uses;
//   * 2x2 max-pool between zero-padded channels-last maps.
// Both are HBM-bound streaming kernels.
#include "common.cuh"

namespace rb {

// one thread per output pixel, 64 output channels in 4 groups of 16 accumulators; weights in shared memory
// (every lane reads the same address -> broadcast).  Inputs are read coalesced along x from the 3 planes.
template <typename TO, bool SPLIT = false>
__global__ void __launch_bounds__(128) conv3x3_first_kernel(const float* __restrict__ img, TO* __restrict__ out,
                                                            const float* __restrict__ wgt, const float* __restrict__ bias,
                                                            int B, int H, int W, int COUT, TO* __restrict__ out_lo = nullptr) {
    rb::pdl_wait();
    extern __shared__ float sw[];   // [COUT][27] + [COUT]
    for (int i = threadIdx.x; i < COUT * 27; i += blockDim.x) sw[i] = wgt[i];
    for (int i = threadIdx.x; i < COUT; i += blockDim.x) sw[COUT * 27 + i] = bias[i];
    __syncthreads();
    int x = blockIdx.x * blockDim.x + threadIdx.x;
    int y = blockIdx.y, b = blockIdx.z;
    if (x >= W) return;
    float in[27];
#pragma unroll
    for (int c = 0; c < 3; ++c)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
                int yy = y + ky - 1, xx = x + kx - 1;
                float v = 0.f;
                if (yy >= 0 && yy < H && xx >= 0 && xx < W) v = img[(((int64_t)b * 3 + c) * H + yy) * W + xx];
                in[c * 9 + ky * 3 + kx] = v;
            }
    TO* o = out + (((int64_t)b * (H + 2) + (y + 1)) * (W + 2) + (x + 1)) * COUT;
    for (int g = 0; g < COUT; g += 8) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            float a = sw[COUT * 27 + g + j];
            const float* wj = sw + (g + j) * 27;
#pragma unroll
            for (int t = 0; t < 27; ++t) a = fmaf(in[t], wj[t], a);
            acc[j] = fmaxf(a, 0.f);
        }
        if constexpr (SPLIT) {                // RB_F16S: hi and lo planes, 8 channels = one 16-byte store each
            __half hi[8], lo[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) split_f16s(acc[j], hi[j], lo[j]);
            *reinterpret_cast<uint4*>(o + g) = *reinterpret_cast<uint4*>(hi);
            *reinterpret_cast<uint4*>(out_lo + (o - out) + g) = *reinterpret_cast<uint4*>(lo);
        } else if constexpr (sizeof(TO) == 2) {      // 8 channels = one 16-byte store
            TO pk[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) pk[j] = from_f<TO>(acc[j]);
            *reinterpret_cast<uint4*>(o + g) = *reinterpret_cast<uint4*>(pk);
        } else {
            *reinterpret_cast<float4*>(o + g) = make_float4(acc[0], acc[1], acc[2], acc[3]);
            *reinterpret_cast<float4*>(o + g + 4) = make_float4(acc[4], acc[5], acc[6], acc[7]);
        }
    }
}

// thread per (output pixel, channel); channels fastest -> coalesced
template <typename T>
__global__ void maxpool2x2_padded_kernel(const T* __restrict__ in, T* __restrict__ out, int B, int H, int W, int C) {
    rb::pdl_wait();
    int Ho = H / 2, Wo = W / 2;
    int64_t total = (int64_t)B * Ho * Wo * C;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(idx % C); int64_t p = idx / C;
        int xo = (int)(p % Wo); int yo = (int)((p / Wo) % Ho); int b = (int)(p / ((int64_t)Wo * Ho));
        const T* s = in + (((int64_t)b * (H + 2) + (2 * yo + 1)) * (W + 2) + (2 * xo + 1)) * C + c;
        int64_t rs = (int64_t)(W + 2) * C;
        float v = fmaxf(fmaxf(to_f(s[0]), to_f(s[C])), fmaxf(to_f(s[rs]), to_f(s[rs + C])));
        out[(((int64_t)b * (Ho + 2) + (yo + 1)) * (Wo + 2) + (xo + 1)) * C + c] = from_f<T>(v);
    }
}

// 16-bit maps with C % 8 == 0: thread per (output pixel, 8-channel vector), 16-byte loads / stores, packed half2 / bf162 max
// (the scalar kernel above spends its time in 64-bit index arithmetic per 2-byte element: 73 us average against a
// 34 us HBM bound for the 864^2 x 64 map).
template <typename T2>
__device__ __forceinline__ uint4 max4(const uint4 a, const uint4 b) {
    uint4 r;
    const T2* pa = reinterpret_cast<const T2*>(&a); const T2* pb = reinterpret_cast<const T2*>(&b);
    T2* pr = reinterpret_cast<T2*>(&r);
#pragma unroll
    for (int i = 0; i < 4; ++i) pr[i] = __hmax2(pa[i], pb[i]);
    return r;
}
template <typename T> struct Pair2;     // the packed pair type of a 16-bit element type
template <> struct Pair2<__half> { using type = __half2; };
template <> struct Pair2<__nv_bfloat16> { using type = __nv_bfloat162; };
template <typename T2>
__global__ void __launch_bounds__(256) maxpool2x2_padded_vec_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int B, int H, int W, int C8) {
    rb::pdl_wait();
    const int Ho = H / 2, Wo = W / 2;
    const int64_t total = (int64_t)B * Ho * Wo * C8;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % C8); const int64_t p = idx / C8;
    const int xo = (int)(p % Wo); const int64_t q = p / Wo;
    const int yo = (int)(q % Ho), b = (int)(q / Ho);
    const int64_t rs = (int64_t)(W + 2) * C8;
    const uint4* s = in + (((int64_t)b * (H + 2) + (2 * yo + 1)) * (W + 2) + (2 * xo + 1)) * C8 + c;
    const uint4 v00 = s[0], v01 = s[C8], v10 = s[rs], v11 = s[rs + C8];
    out[(((int64_t)b * (Ho + 2) + (yo + 1)) * (Wo + 2) + (xo + 1)) * C8 + c] = max4<T2>(max4<T2>(v00, v01), max4<T2>(v10, v11));
}

// RB_F16S maps (C % 8 == 0): the pair (hi, lo) with the largest value hi + lo * 2^-11 is copied through unchanged
__global__ void __launch_bounds__(256) maxpool2x2_padded_split_kernel(const uint4* __restrict__ in_hi, const uint4* __restrict__ in_lo,
                                                                      uint4* __restrict__ out_hi, uint4* __restrict__ out_lo, int B, int H, int W, int C8) {
    rb::pdl_wait();
    const int Ho = H / 2, Wo = W / 2;
    const int64_t total = (int64_t)B * Ho * Wo * C8;
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= total) return;
    const int c = (int)(idx % C8); const int64_t p = idx / C8;
    const int xo = (int)(p % Wo); const int64_t q = p / Wo;
    const int yo = (int)(q % Ho), b = (int)(q / Ho);
    const int64_t rs = (int64_t)(W + 2) * C8;
    const int64_t si = (((int64_t)b * (H + 2) + (2 * yo + 1)) * (W + 2) + (2 * xo + 1)) * C8 + c;
    const int64_t offs[4] = {0, C8, rs, rs + C8};
    uint4 bh = in_hi[si], bl = in_lo[si];
#pragma unroll
    for (int t = 1; t < 4; ++t) {
        const uint4 h = in_hi[si + offs[t]], l = in_lo[si + offs[t]];
        const __half* ph = reinterpret_cast<const __half*>(&h); const __half* pl = reinterpret_cast<const __half*>(&l);
        __half* qh = reinterpret_cast<__half*>(&bh); __half* ql = reinterpret_cast<__half*>(&bl);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            if (join_f16s(ph[j], pl[j]) > join_f16s(qh[j], ql[j])) { qh[j] = ph[j]; ql[j] = pl[j]; }
    }
    const int64_t so = (((int64_t)b * (Ho + 2) + (yo + 1)) * (Wo + 2) + (xo + 1)) * C8 + c;
    out_hi[so] = bh; out_lo[so] = bl;
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_conv3x3_first(const rb_conv_first_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->cout % 8 == 0 && a->cout <= 256, "conv3x3_first: cout=%d", a->cout);
    RB_REQUIRE(a->height <= 65535 && a->batch <= 65535, "conv3x3_first: grid too large");
    dim3 grid((a->width + 127) / 128, a->height, a->batch);
    size_t smem = (size_t)a->cout * 28 * sizeof(float);
    if (a->dtype_out == RB_F16S) {
        RB_REQUIRE(a->out_lo, "conv3x3_first: RB_F16S output needs out_lo");
        rb::launch_pdl(conv3x3_first_kernel<__half, true>, dim3(grid), dim3(128), smem, st, a->image, (__half*)a->out, a->weight, a->bias, a->batch, a->height, a->width, a->cout, (__half*)a->out_lo);
        return check_launch("conv3x3_first");
    }
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype_out, "conv3x3_first", [&](auto t) {
        using TO = typename decltype(t)::type;
        rb::launch_pdl(conv3x3_first_kernel<TO, false>, grid, dim3(128), smem, st, a->image, (TO*)a->out, a->weight, a->bias, a->batch, a->height, a->width, a->cout, (TO*)nullptr);
        return check_launch("conv3x3_first");
    });
}

extern "C" int romab200_maxpool2x2_padded(const rb_maxpool_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int64_t total = (int64_t)a->batch * (a->height / 2) * (a->width / 2) * a->channels;
    RB_REQUIRE(total > 0, "maxpool: empty");
    if (a->dtype == RB_F16S) {
        RB_REQUIRE(a->in_lo && a->out_lo && a->channels % 8 == 0 && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0 &&
                   ((uintptr_t)a->in_lo) % 16 == 0 && ((uintptr_t)a->out_lo) % 16 == 0, "maxpool: RB_F16S needs both planes, C %% 8 == 0, 16-byte alignment");
        const int64_t tv = total / 8, gv = (tv + 255) / 256;
        RB_REQUIRE(gv < (1ll << 31), "maxpool: grid too large");
        rb::launch_pdl(maxpool2x2_padded_split_kernel, dim3((unsigned)gv), dim3(256), 0, st, (const uint4*)a->in, (const uint4*)a->in_lo, (uint4*)a->out, (uint4*)a->out_lo,
                       a->batch, a->height, a->width, a->channels / 8);
        return check_launch("maxpool2x2_padded");
    }
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "maxpool2x2_padded", [&](auto t) {
        using T = typename decltype(t)::type;
        if constexpr (sizeof(T) == 2) {
            if (a->channels % 8 == 0 && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0) {
                const int64_t tv = total / 8, gv = (tv + 255) / 256;
                RB_REQUIRE(gv < (1ll << 31), "maxpool: grid too large");
                rb::launch_pdl(maxpool2x2_padded_vec_kernel<typename Pair2<T>::type>, dim3((unsigned)gv), dim3(256), 0, st, (const uint4*)a->in, (uint4*)a->out,
                               a->batch, a->height, a->width, a->channels / 8);
                return check_launch("maxpool2x2_padded");
            }
        }
        rb::launch_pdl(maxpool2x2_padded_kernel<T>, dim3(grid1d(total, 256, 132 * 64)), dim3(256), 0, st, (const T*)a->in, (T*)a->out, a->batch, a->height, a->width, a->channels);
        return check_launch("maxpool2x2_padded");
    });
}
