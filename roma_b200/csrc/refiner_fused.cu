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
// The parity mode (fp32 maps, split-fp16 pointwise operands) has its own kernel below, refiner_block_c144_split_kernel.
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

// ===== parity mode: the same block on fp32 maps with split-fp16 pointwise operands =====
// Bit-identical to the two launches it replaces, dwconv5x5_relu_tma_kernel<float> (fp32 map -> RB_F16S pair) followed by
// gemm_tc_kernel<144, true> (RB_F16S pair x RB_F16S weights -> fp32 map + bias): every result goes through the same operations
// in the same order, only the intermediate pair stays in shared memory.  The block moves 8 B per map element (read 4, write 4)
// instead of 16.  The fp32 input window and the two planes of both operands are twice the size of the fast-mode kernel's, so
//   * the tile is 4 x 16 = 64 pixels (one m64 wgmma row block; the warpgroup's accumulators acc / acc2 take 144 registers);
//   * the input window (8 x 20 pixels) arrives in chunks of 16 channels through a TMA ring of 7 slots, one per depthwise warp;
//   * the 7 depthwise warps take the chunks in turn (chunk g: warp and slot g % 7; lane = channel x row pair, 2 rows x 16
//     pixels each) and write the ReLU'd, split result as one k-step (16 channels, 32-byte swizzle) of a double-buffered A
//     operand, so the next tile's depthwise stage overlaps this tile's MMAs and stores.  A slot has one consumer, which waits
//     for its phases in order: with more consumers than slots a warp could wait on a phase two ahead and pass early;
//   * the pointwise weights stay resident as 9 k-steps of 16 channels per plane (32-byte swizzle: no zero-padded k-block).
struct FusedSplitParams {
    float* out; int64_t ld;
    const float* dw_w; int64_t ldw; const float* dw_b; const float* pw_b;
    int H, W, tiles_x, tiles_per_img, total_tiles;
};

constexpr int FS_TH = 4, FS_TW = 16, FS_IH = FS_TH + 4, FS_IW = FS_TW + 4, FS_CH = 16, FS_KSTEPS = FZ_C / FS_CH;   // 9 chunks
constexpr int FS_DW_WARPS = 7, FS_STAGES = FS_DW_WARPS;           // one ring slot per depthwise warp
constexpr int FS_THREADS = 128 + 32 + 32 * FS_DW_WARPS;               // warps 0-3: MMA + epilogue, warp 4: input TMA, 5-11: depthwise
constexpr int FS_STAGE_BYTES = FS_IH * FS_IW * FS_CH * 4;             // 10240: one fp32 chunk of the window
constexpr int FS_A_KS = 64 * 32, FS_A_PLANE = FS_KSTEPS * FS_A_KS, FS_A_BYTES = 2 * FS_A_PLANE;            // 36864 per A buffer
constexpr int FS_B_KS = FZ_C * 32, FS_B_PLANE = FS_KSTEPS * FS_B_KS, FS_B_BYTES = 2 * FS_B_PLANE;          // 82944
constexpr int FS_OFF_A = FS_B_BYTES, FS_OFF_RING = FS_OFF_A + 2 * FS_A_BYTES, FS_OFF_BIAS = FS_OFF_RING + FS_STAGES * FS_STAGE_BYTES;
constexpr int FS_OFF_BARS = FS_OFF_BIAS + FZ_C * 4;
constexpr int FS_SMEM = FS_OFF_BARS + 256 + 1024;
static_assert(FS_OFF_A % 1024 == 0 && FS_OFF_RING % 1024 == 0 && FS_SMEM <= 232448, "shared memory layout");

__global__ void __launch_bounds__(FS_THREADS, 1) refiner_block_c144_split_kernel(const __grid_constant__ CUtensorMap map_w, const __grid_constant__ CUtensorMap map_w_lo,
                                                                               const __grid_constant__ CUtensorMap map_in, const FusedSplitParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - ((uint32_t)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);   // offset on the array: keeps ld/st.shared
    uint8_t* sB = smem;
    uint8_t* sA = smem + FS_OFF_A;
    uint8_t* ring = smem + FS_OFF_RING;
    float* s_pwb = reinterpret_cast<float*>(smem + FS_OFF_BIAS);          // [144] pointwise bias
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FS_OFF_BARS);
    uint64_t* full = bars;                          // input chunk landed (TMA transaction bytes)
    uint64_t* empty = bars + FS_STAGES;             // its depthwise warp has read it
    uint64_t* a_full = bars + 2 * FS_STAGES;        // [2] all 9 k-steps of the A buffer written (one arrival per chunk)
    uint64_t* a_empty = a_full + 2;                 // [2] the MMAs that read the A buffer retired
    uint64_t* w_full = a_empty + 2;                 // pointwise weights landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < FS_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
        for (int b = 0; b < 2; ++b) { mbar_init(&a_full[b], FS_KSTEPS); mbar_init(&a_empty[b], 1); }
        mbar_init(w_full, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    rb::pdl_wait();                                    // everything above overlapped the previous kernel's tail
    for (int i = threadIdx.x; i < FZ_C; i += FS_THREADS) s_pwb[i] = p.pw_b[i];
    __syncthreads();
    const int my_tiles = p.total_tiles > (int)blockIdx.x ? (p.total_tiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;

    if (warp < 4) {
        // ===== pointwise GEMM + epilogue, as gemm_tc_kernel<144, true> issues it for one 64-row half of its tile =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");     // acc + acc2: 144 registers a thread
        const int t = threadIdx.x;
        if (t == 0) {
            mbar_expect_tx(w_full, FS_B_BYTES);
            for (int j = 0; j < FS_KSTEPS; ++j) {
                tma_load_2d(sB + j * FS_B_KS, &map_w, w_full, j * FS_CH, 0);
                tma_load_2d(sB + FS_B_PLANE + j * FS_B_KS, &map_w_lo, w_full, j * FS_CH, 0);
            }
        }
        mbar_wait(w_full, 0);
        const uint32_t b_addr = smem_u32(sB);
        float acc[FZ_C / 2], acc2[FZ_C / 2];
        for (int it = 0; it < my_tiles; ++it) {
            const int tile = blockIdx.x + it * gridDim.x;
            const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
            const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
            const int ab = it & 1;
            const uint32_t a_addr = smem_u32(sA + ab * FS_A_BYTES);
            mbar_wait(&a_full[ab], (it >> 1) & 1);
            // K = 144 in 9 k-steps of 16 channels, ascending.  gemm_tc_kernel also issues the three k-steps of channels 144-191
            // of its last k-block; their operands are TMA zero fill, and adding zero products leaves an accumulator unchanged
            // (up to the sign of a zero), so they are not issued here.
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < FS_KSTEPS; ++j) {
                const uint64_t a_hi = gmma_desc(a_addr + j * FS_A_KS, 16, 256, GMMA_SW32);
                const uint64_t a_lo = gmma_desc(a_addr + FS_A_PLANE + j * FS_A_KS, 16, 256, GMMA_SW32);
                const uint64_t b_hi = gmma_desc(b_addr + j * FS_B_KS, 16, 256, GMMA_SW32);
                const uint64_t b_lo = gmma_desc(b_addr + FS_B_PLANE + j * FS_B_KS, 16, 256, GMMA_SW32);
                Wgmma<FZ_C, false>::ss<0>(acc, a_hi, b_hi, j != 0);
                Wgmma<FZ_C, false>::ss<0>(acc2, a_hi, b_lo, j != 0);
                Wgmma<FZ_C, false>::ss<0>(acc2, a_lo, b_hi, 1);
            }
            wgmma_commit();
            wgmma_wait<0>();
            wgmma_fence_regs(acc);
            wgmma_fence_regs(acc2);
            if (t == 0) mbar_arrive(&a_empty[ab]);          // the depthwise warps may overwrite this A buffer
            // epilogue (Epilogue::apply with alpha = 1, bias, fp32 out): acc + acc2 * 2^-11, then + bias.  Accumulator fragment:
            // pixels m and m + 8, channel pairs 8 i + 2 (t % 4).
            const int m0 = (t >> 5) * 16 + ((t & 31) >> 2), cn = 2 * (t & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = m0 + 8 * h;
                const int yy = ty * FS_TH + m / FS_TW, xx = tx * FS_TW + m % FS_TW;
                if (yy >= p.H || xx >= p.W) continue;
                float* orow = p.out + (((int64_t)img * p.H + yy) * p.W + xx) * p.ld + cn;
#pragma unroll
                for (int i = 0; i < FZ_C / 8; ++i) {
                    const float v0 = fmaf(acc2[4 * i + 2 * h], 1.0f / RB_SPLIT_SCALE, acc[4 * i + 2 * h]);
                    const float v1 = fmaf(acc2[4 * i + 2 * h + 1], 1.0f / RB_SPLIT_SCALE, acc[4 * i + 2 * h + 1]);
                    *reinterpret_cast<float2*>(orow + 8 * i) = make_float2(__fadd_rn(v0, s_pwb[8 * i + cn]), __fadd_rn(v1, s_pwb[8 * i + cn + 1]));
                }
            }
        }
    } else {
        // 12 warps leave 3 on some SM sub-partition, whose register file then caps a thread at 168 registers: warpgroups 1-2
        // (loader, depthwise) hand theirs to the MMA warpgroup
        asm volatile("setmaxnreg.dec.sync.aligned.u32 104;");
        if (warp == 4) {
            // ===== input loader: chunk j of tile it is ring slot (9 it + j) % FS_STAGES =====
            if (lane == 0) {
                uint32_t g = 0;
                for (int it = 0; it < my_tiles; ++it) {
                    const int tile = blockIdx.x + it * gridDim.x;
                    const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
                    const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                    for (int j = 0; j < FS_KSTEPS; ++j, ++g) {
                        const uint32_t s = g % FS_STAGES, round = g / FS_STAGES;
                        if (round > 0) mbar_wait(&empty[s], (round - 1) & 1);
                        mbar_expect_tx(&full[s], FS_STAGE_BYTES);
                        tma_load_4d(ring + s * FS_STAGE_BYTES, &map_in, &full[s], j * FS_CH, tx * FS_TW - 2, ty * FS_TH - 2, img);
                    }
                }
            }
        } else {
            // ===== depthwise warps: warp w takes chunks g = w, w + 7, ... (tile g / 9, channels 16 (g % 9) ..), all from slot w =====
            // lane = (channel c of the chunk, row pair rp): output rows 2 rp, 2 rp + 1 x 16 pixels.  The arithmetic is that of
            // dwconv5x5_relu_tma_kernel<float>: bias, then fmaf over the taps ky-major, kx-minor, ReLU, split_f16s.
            const int c = lane & 15, rp = lane >> 4;
            const uint32_t n_chunks = (uint32_t)my_tiles * FS_KSTEPS;
            for (uint32_t g = warp - 5; g < n_chunks; g += FS_DW_WARPS) {
                const int it = g / FS_KSTEPS, j = g - it * FS_KSTEPS;
                const uint32_t s = g % FS_STAGES;
                const int ch = j * FS_CH + c;
                float wv[25];
    #pragma unroll
                for (int k = 0; k < 25; ++k) wv[k] = __ldg(&p.dw_w[(int64_t)k * p.ldw + ch]);    // 14 KB for all chunks: L1 hits
                const float bv = __ldg(&p.dw_b[ch]);
                float acc[2][FS_TW];
    #pragma unroll
                for (int rr = 0; rr < 2; ++rr)
    #pragma unroll
                    for (int i = 0; i < FS_TW; ++i) acc[rr][i] = bv;
                mbar_wait(&full[s], (g / FS_STAGES) & 1);
                const float* win = reinterpret_cast<const float*>(ring + s * FS_STAGE_BYTES) + c;
    #pragma unroll
                for (int iy = 0; iy < 6; ++iy) {                   // window rows 2 rp + iy feed output rows 2 rp + {0, 1}
    #pragma unroll
                    for (int ix = 0; ix < FS_IW; ++ix) {
                        const float v = win[((2 * rp + iy) * FS_IW + ix) * FS_CH];
    #pragma unroll
                        for (int rr = 0; rr < 2; ++rr) {
                            const int ky = iy - rr;
                            if (ky >= 0 && ky < 5) {
    #pragma unroll
                                for (int kx = 0; kx < 5; ++kx) {
                                    const int ox = ix - kx;
                                    if (ox >= 0 && ox < FS_TW) acc[rr][ox] = fmaf(wv[ky * 5 + kx], v, acc[rr][ox]);
                                }
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);             // this warp no longer reads the slot
                const int ab = it & 1;
                mbar_wait(&a_empty[ab], ((it >> 1) & 1) ^ 1);     // the MMAs of tile it - 2 no longer read the buffer
                // k-step j of both planes: row m (pixel) is 32 B, channel c at 16-byte chunk (c / 8) ^ ((m / 4) % 2), element c % 8
                uint8_t* a_hi = sA + ab * FS_A_BYTES + j * FS_A_KS;
    #pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
    #pragma unroll
                    for (int i = 0; i < FS_TW; ++i) {
                        const int m = (2 * rp + rr) * FS_TW + i;
                        __half hi, lo;
                        split_f16s(fmaxf(acc[rr][i], 0.f), hi, lo);
                        const int off = m * 32 + ((((c >> 3) ^ (m >> 2)) & 1) << 4) + (c & 7) * 2;
                        *reinterpret_cast<__half*>(a_hi + off) = hi;
                        *reinterpret_cast<__half*>(a_hi + FS_A_PLANE + off) = lo;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(&a_full[ab]);
            }
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
    return with_dtype<__half, __nv_bfloat16>(a->dtype, "refiner_block_c144", [&](auto t) {
        using T = typename decltype(t)::type;
        RB_REQUIRE(a->ld % 8 == 0 && a->ld >= FZ_C && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0 && a->in != a->out,
                   "refiner_block_c144: bad activation layout");
        RB_REQUIRE(a->ld_pw % 8 == 0 && a->ld_pw >= FZ_C && ((uintptr_t)a->pw_weight) % 16 == 0, "refiner_block_c144: bad weight layout");
        const CUtensorMapDataType dt = tma_dtype(a->dtype);
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
        if (ensure_smem<refiner_block_c144_kernel<T>>(FZ_SMEM, "refiner_block_c144")) return 1;
        rb::launch_pdl(refiner_block_c144_kernel<T>, dim3(grid), dim3(FZ_THREADS), FZ_SMEM, st, map, map_in, p);
        return check_launch("refiner_block_c144");
    });
}

extern "C" int romab200_refiner_block_c144_split(const rb_refiner_block_c144_split_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->c == FZ_C, "refiner_block_c144_split: C must be 144 (got %d)", a->c);
    RB_REQUIRE(a->in != a->out, "refiner_block_c144_split: in and out must differ (the block reads a 5x5 halo)");
    RB_REQUIRE(a->ld % 8 == 0 && a->ld >= FZ_C && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0,
               "refiner_block_c144_split: bad activation layout (ld %lld)", (long long)a->ld);
    RB_REQUIRE(a->ld_pw % 8 == 0 && a->ld_pw >= FZ_C && ((uintptr_t)a->pw_weight) % 16 == 0 && ((uintptr_t)a->pw_weight_lo) % 16 == 0,
               "refiner_block_c144_split: bad weight layout (ld_pw %lld)", (long long)a->ld_pw);
    RB_REQUIRE(a->ldw >= FZ_C, "refiner_block_c144_split: ldw %lld < 144", (long long)a->ldw);
    CUtensorMap map_w, map_w_lo;       // pointwise weights [144 x 144] per plane: boxes of 16 channels x 144 rows, 32-byte swizzle
    {
        cuuint64_t dims[2] = {(cuuint64_t)FZ_C, (cuuint64_t)FZ_C};
        cuuint64_t strides[1] = {(cuuint64_t)a->ld_pw * 2};
        cuuint32_t box[2] = {FS_CH, (cuuint32_t)FZ_C};
        if (encode_tiled(&map_w, "refiner_block_c144_split", CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, a->pw_weight, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
        if (encode_tiled(&map_w_lo, "refiner_block_c144_split", CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, a->pw_weight_lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_32B)) return 1;
    }
    CUtensorMap map_in;          // fp32 activation [B, H, W, C] with pitch ld: box = 8 x 20 pixels x 16 channels, borders zero-filled
    {
        cuuint64_t d4[4] = {(cuuint64_t)FZ_C, (cuuint64_t)a->w, (cuuint64_t)a->h, (cuuint64_t)a->batch};
        cuuint64_t s4[3] = {(cuuint64_t)a->ld * 4, (cuuint64_t)a->w * a->ld * 4, (cuuint64_t)a->h * a->w * a->ld * 4};
        cuuint32_t b4[4] = {FS_CH, FS_IW, FS_IH, 1};
        if (encode_tiled(&map_in, "refiner_block_c144_split (input)", CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, a->in, d4, s4, b4, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
    }
    FusedSplitParams p;
    p.out = a->out; p.ld = a->ld; p.dw_w = a->dw_weight; p.ldw = a->ldw; p.dw_b = a->dw_bias; p.pw_b = a->pw_bias;
    p.H = a->h; p.W = a->w; p.tiles_x = (a->w + FS_TW - 1) / FS_TW; p.tiles_per_img = p.tiles_x * ((a->h + FS_TH - 1) / FS_TH);
    const long long total = (long long)p.tiles_per_img * a->batch;
    RB_REQUIRE(a->h > 0 && a->w > 0 && total > 0 && total < (1ll << 31) / FS_KSTEPS, "refiner_block_c144_split: bad tile count");
    p.total_tiles = (int)total;
    const int sms = sm_count();
    const int grid = p.total_tiles < sms ? p.total_tiles : sms;
    if (ensure_smem<refiner_block_c144_split_kernel>(FS_SMEM, "refiner_block_c144_split")) return 1;
    rb::launch_pdl(refiner_block_c144_split_kernel, dim3(grid), dim3(FS_THREADS), FS_SMEM, st, map_w, map_w_lo, map_in, p);
    return check_launch("refiner_block_c144_split");
}
