// Fused ConvRefiner block for the stride-2 maps (C = 144):  out = PW_{144x144}( ReLU( BN( DW5x5(in) ) ) ) + bias
// (create_block, romatch/models/matcher.py:92-122) in ONE kernel: the activation map is read once and written once.
// Un-fused, this block is a depthwise kernel plus a GEMM that together move the 107 MB map four times and spend most
// of their time in per-tile overheads; here
//   * 1 thread TMA-loads the 12x20 pixel input window of an 8x16 tile (4-D tensor map over [B,H,W,C]: the image border
//     is the map's out-of-bounds zero fill, no address arithmetic, no registers);
//   * 9 depthwise warps run the 5x5 stage on the CUDA cores (channel pairs) and write the ReLU'd 128 x 144 result
//     straight into the 128B-swizzled K-major layout of a wgmma A operand;
//   * 1 warpgroup multiplies it with the pointwise weights (TMA-loaded into shared memory once, resident for the whole
//     persistent kernel): per 64-pixel half 9 wgmma (M=64, N=144, K=16) into registers, then + bias -> 16-bit rows.
#include "tma.cuh"
#include "wgmma.cuh"
#include <type_traits>

namespace rb {

#ifdef RB_FZ_CLK
__device__ long long g_fz_clk[64];
#define FZCLK(var) const long long var = clock64();
#else
#define FZCLK(var)
#endif

struct FusedParams {
    const void* in; void* out; int64_t ld;
    const float* dw_w; int64_t ldw; const float* dw_b; const float* pw_b;
    int batch, H, W, tiles_x, tiles_y, total_tiles, is_bf16;
};

constexpr int FZ_C = 144, FZ_CP = 72, FZ_TH = 8, FZ_TW = 16, FZ_IH = 12, FZ_IW = 20;
constexpr int FZ_DW_THREADS = 288;                    // 72 channel pairs x 4 row groups
constexpr int FZ_THREADS = 128 + 32 + FZ_DW_THREADS;  // warps 0-3: weights + MMA + epilogue, warp 4: input TMA, warps 5-13: depthwise
constexpr int FZ_IN_BYTES = FZ_IH * FZ_IW * FZ_C * 2;              // 69120
constexpr int FZ_A_BYTES = 3 * 128 * 128;                          // 49152: 3 k-blocks of 64 channels, 128 pixel rows
constexpr int FZ_B_KB = FZ_C * 128;                                // 18432 per k-block
constexpr int FZ_B_BYTES = 3 * FZ_B_KB;                            // 55296
constexpr int FZ_W_BYTES = 25 * FZ_C * 4;                          // depthwise taps, fp32, tap-major
constexpr int FZ_SMEM = FZ_A_BYTES + FZ_B_BYTES + FZ_IN_BYTES + FZ_W_BYTES + 1024 + 1024;

template <typename T>
__global__ void __launch_bounds__(FZ_THREADS, 1) refiner_block_c144_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_in, const FusedParams p) {
    rb::pdl_wait();
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - ((uint32_t)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);   // offset on the array: keeps ld/st.shared
    uint8_t* sA = smem;
    uint8_t* sB = sA + FZ_A_BYTES;
    uint8_t* sIn = sB + FZ_B_BYTES;
    float* s_dw = reinterpret_cast<float*>(sIn + FZ_IN_BYTES);            // [25][144]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sIn + FZ_IN_BYTES + FZ_W_BYTES);
    uint64_t* w_full = bars;            // weights landed
    uint64_t* a_full = bars + 1;        // depthwise tile written (9 warp arrivals)
    uint64_t* a_empty = bars + 2;       // MMAs that read it retired
    uint64_t* in_full = bars + 3;       // input window landed (TMA transaction bytes)
    uint64_t* in_empty = bars + 4;      // depthwise warps have read it (9 warp arrivals)
    float* s_bias = reinterpret_cast<float*>(bars + 6);     // [144]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        mbar_init(w_full, 1); mbar_init(a_full, FZ_DW_THREADS / 32); mbar_init(a_empty, 1);
        mbar_init(in_full, 1); mbar_init(in_empty, FZ_DW_THREADS / 32);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    for (int i = threadIdx.x; i < FZ_C; i += FZ_THREADS) s_bias[i] = p.pw_b[i];
    for (int i = threadIdx.x; i < 25 * FZ_C; i += FZ_THREADS) s_dw[i] = p.dw_w[(int64_t)(i / FZ_C) * p.ldw + (i % FZ_C)];
    for (int i = threadIdx.x; i < FZ_A_BYTES / 16; i += FZ_THREADS) reinterpret_cast<uint4*>(sA)[i] = make_uint4(0u, 0u, 0u, 0u);   // K padding stays 0
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const int tiles_per_img = p.tiles_x * p.tiles_y;

    if (warp < 4) {
        // ===== pointwise GEMM + epilogue: the warpgroup takes the 128-pixel tile in two halves of 64 rows =====
        const int t = threadIdx.x;
        if (t == 0) {
            // pointwise weights [144 x 144] -> three K-major k-blocks, loaded once for the whole persistent kernel
            mbar_expect_tx(w_full, FZ_B_BYTES);
            for (int kb = 0; kb < 3; ++kb) tma_load_2d(sB + kb * FZ_B_KB, &map_w, w_full, kb * 64, 0);
        }
        mbar_wait(w_full, 0);
        const uint32_t a_addr = smem_u32(sA), b_addr = smem_u32(sB);
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
            const int img = tile / tiles_per_img, r = tile - img * tiles_per_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
            mbar_wait(a_full, it & 1);
#pragma unroll 1
            for (int half = 0; half < 2; ++half) {
                float acc[FZ_C / 2];
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < FZ_C / 16; ++k) {
                    const uint32_t aoff = (k >> 2) * (128 * 128) + half * (64 * 128) + (k & 3) * 32, boff = (k >> 2) * FZ_B_KB + (k & 3) * 32;
                    Wgmma<FZ_C, std::is_same<T, __nv_bfloat16>::value>::template ss<0>(acc, gmma_desc(a_addr + aoff, 16, 1024), gmma_desc(b_addr + boff, 16, 1024), k != 0);
                }
                wgmma_commit();
                wgmma_wait<0>();
                wgmma_fence_regs(acc);
                if (half == 1 && t == 0) mbar_arrive(a_empty);     // the depthwise warps may overwrite sA
                // accumulator fragment: pixels m and m + 8 of this half, channel pairs 8 i + 2 (t % 4)
                const int m0 = half * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int m = m0 + 8 * h;
                    const int yy = ty * FZ_TH + m / FZ_TW, xx = tx * FZ_TW + m % FZ_TW;
                    if (yy >= p.H || xx >= p.W) continue;
                    T* orow = (T*)p.out + (((int64_t)img * p.H + yy) * p.W + xx) * p.ld + 2 * (t & 3);
#pragma unroll
                    for (int i = 0; i < FZ_C / 8; ++i) {
                        T pr[2] = {from_f<T>(acc[4 * i + 2 * h] + s_bias[8 * i + 2 * (t & 3)]), from_f<T>(acc[4 * i + 2 * h + 1] + s_bias[8 * i + 2 * (t & 3) + 1])};
                        *reinterpret_cast<uint32_t*>(orow + 8 * i) = *reinterpret_cast<uint32_t*>(pr);
                    }
                }
            }
        }
    } else if (warp == 4) {
        // ===== input loader: one TMA box per tile, re-armed as soon as the depthwise warps have read the previous window =====
        if (lane == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
                const int img = tile / tiles_per_img, r = tile - img * tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                if (it > 0) mbar_wait(in_empty, (it - 1) & 1);
                mbar_expect_tx(in_full, FZ_IN_BYTES);
                tma_load_4d(sIn, &map_in, in_full, 0, tx * FZ_TW - 2, ty * FZ_TH - 2, img);
            }
        }
    } else {
        // ===== depthwise producers: thread = (channel pair, 2 output rows) =====
        const int t = threadIdx.x - 160;                   // 0 .. 287
        const int cp = t % FZ_CP, rg = t / FZ_CP;
        const float2 bv = make_float2(p.dw_b[2 * cp], p.dw_b[2 * cp + 1]);
        // A-operand address pieces of this thread's two channels (K-major, 128B swizzle): k-block, 16-byte chunk, byte in chunk
        const int kb = cp >> 5, chunk = (cp & 31) >> 2, inb = (cp & 3) * 4;
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
            FZCLK(t0)
            mbar_wait(in_full, it & 1);
            FZCLK(t1)
            // filter taps: re-read from shared memory per tile so that they are not live during the load phase
            float2 wv[25];
#pragma unroll
            for (int k = 0; k < 25; ++k) wv[k] = *reinterpret_cast<const float2*>(&s_dw[k * FZ_C + 2 * cp]);
            float2 acc2[2][FZ_TW];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                for (int i = 0; i < FZ_TW; ++i) acc2[rr][i] = bv;
#pragma unroll
            for (int iy = 0; iy < 6; ++iy) {
#pragma unroll
                for (int ix = 0; ix < FZ_IW; ++ix) {
                    T pr[2];
                    *reinterpret_cast<uint32_t*>(pr) = *reinterpret_cast<const uint32_t*>(sIn + ((2 * rg + iy) * FZ_IW + ix) * (FZ_C * 2) + cp * 4);
                    const float2 v = make_float2(to_f(pr[0]), to_f(pr[1]));
#pragma unroll
                    for (int rr = 0; rr < 2; ++rr) {
                        const int ky = iy - rr;
                        if (ky >= 0 && ky < 5) {
#pragma unroll
                            for (int kx = 0; kx < 5; ++kx) {
                                const int ox = ix - kx;
                                if (ox >= 0 && ox < FZ_TW) { const float2 w2 = wv[ky * 5 + kx]; acc2[rr][ox].x = fmaf(w2.x, v.x, acc2[rr][ox].x); acc2[rr][ox].y = fmaf(w2.y, v.y, acc2[rr][ox].y); }
                            }
                        }
                    }
                }
            }
            FZCLK(t2)
            __syncwarp();
            if (lane == 0) mbar_arrive(in_empty);          // this warp's reads of the input window are done
            mbar_wait(a_empty, (it & 1) ^ 1);
            FZCLK(t3)              // the MMAs of the previous tile no longer read sA
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
                for (int i = 0; i < FZ_TW; ++i) {
                    const int m = (2 * rg + rr) * FZ_TW + i;
                    T pair[2] = {from_f<T>(fmaxf(acc2[rr][i].x, 0.f)), from_f<T>(fmaxf(acc2[rr][i].y, 0.f))};
                    *reinterpret_cast<uint32_t*>(sA + kb * (128 * 128) + m * 128 + ((chunk ^ (m & 7)) << 4) + inb) = *reinterpret_cast<uint32_t*>(pair);
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            __syncwarp();
            if (lane == 0) mbar_arrive(a_full);
#ifdef RB_FZ_CLK
            if (blockIdx.x == 0 && lane == 0) { const long long t4 = clock64(); long long* g = g_fz_clk + (warp - 5) * 5; g[0] += t1 - t0; g[1] += t2 - t1; g[2] += t3 - t2; g[3] += t4 - t3; g[4] += 1; }
#endif
        }
    }
}
}  // namespace rb

using namespace rb;

#ifdef RB_FZ_CLK
extern "C" int romab200_debug_fzclk(long long* out, int reset) {
    if (reset) { long long z[64] = {0}; return (int)cudaMemcpyToSymbol(rb::g_fz_clk, z, sizeof(z)); }
    return (int)cudaMemcpyFromSymbol(out, rb::g_fz_clk, sizeof(long long) * 64);
}
#endif

extern "C" int romab200_refiner_block_c144(const rb_refiner_block_c144_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->c == FZ_C, "refiner_block_c144: C must be 144 (got %d)", a->c);
    RB_REQUIRE(a->dtype == RB_F16 || a->dtype == RB_BF16, "refiner_block_c144: 16-bit activations only");
    RB_REQUIRE(a->ld % 8 == 0 && a->ld >= FZ_C && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0 && a->in != a->out,
               "refiner_block_c144: bad activation layout");
    RB_REQUIRE(a->ld_pw % 8 == 0 && a->ld_pw >= FZ_C && ((uintptr_t)a->pw_weight) % 16 == 0, "refiner_block_c144: bad weight layout");
    const CUtensorMapDataType dt = a->dtype == RB_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    CUtensorMap map;
    cuuint64_t dims[2] = {(cuuint64_t)FZ_C, (cuuint64_t)FZ_C};
    cuuint64_t strides[1] = {(cuuint64_t)a->ld_pw * 2};
    cuuint32_t box[2] = {64, (cuuint32_t)FZ_C};
    if (encode_tiled(&map, "refiner_block_c144", dt, 2, a->pw_weight, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
    CUtensorMap map_in;          // activation [B, H, W, C] with pitch ld: box = 12 x 20 pixels x 144 channels, borders zero-filled
    {
        cuuint64_t d4[4] = {(cuuint64_t)FZ_C, (cuuint64_t)a->w, (cuuint64_t)a->h, (cuuint64_t)a->batch};
        cuuint64_t s4[3] = {(cuuint64_t)a->ld * 2, (cuuint64_t)a->w * a->ld * 2, (cuuint64_t)a->h * a->w * a->ld * 2};
        cuuint32_t b4[4] = {(cuuint32_t)FZ_C, (cuuint32_t)FZ_IW, (cuuint32_t)FZ_IH, 1};
        if (encode_tiled(&map_in, "refiner_block_c144 (input)", dt, 4, a->in, d4, s4, b4, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
    }
    FusedParams p;
    p.in = a->in; p.out = a->out; p.ld = a->ld; p.dw_w = a->dw_weight; p.ldw = a->ldw; p.dw_b = a->dw_bias; p.pw_b = a->pw_bias;
    p.batch = a->batch; p.H = a->h; p.W = a->w; p.tiles_x = (a->w + FZ_TW - 1) / FZ_TW; p.tiles_y = (a->h + FZ_TH - 1) / FZ_TH;
    const long long total = (long long)p.tiles_x * p.tiles_y * a->batch;
    RB_REQUIRE(total > 0 && total < (1ll << 31), "refiner_block_c144: bad tile count");
    p.total_tiles = (int)total; p.is_bf16 = a->dtype == RB_BF16;
    const int sms = sm_count();
    const int grid = p.total_tiles < sms ? p.total_tiles : sms;
    if (a->dtype == RB_F16) {
        if (ensure_smem<refiner_block_c144_kernel<__half>>(FZ_SMEM, "refiner_block_c144")) return 1;
        rb::launch_pdl(refiner_block_c144_kernel<__half>, dim3(grid), dim3(FZ_THREADS), FZ_SMEM, st, map, map_in, p);
    } else {
        if (ensure_smem<refiner_block_c144_kernel<__nv_bfloat16>>(FZ_SMEM, "refiner_block_c144")) return 1;
        rb::launch_pdl(refiner_block_c144_kernel<__nv_bfloat16>, dim3(grid), dim3(FZ_THREADS), FZ_SMEM, st, map, map_in, p);
    }
    return check_launch("refiner_block_c144");
}
