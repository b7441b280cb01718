// Depthwise 5x5 + folded BN + ReLU of the ConvRefiner blocks (create_block, romatch/models/matcher.py:92-122) for the
// wide maps (C = 569 / 1137 / 1377 at strides 4 / 8 / 16; C = 144 / 24 in the parity mode), TMA-fed and persistent.
// Two instantiations: 16-bit map -> 16-bit map (fast mode, 8x16 tiles, 3 stages, two CTAs per SM) and fp32 map -> RB_F16S
// pair (parity mode: the result is the A operand of the split-fp16 pointwise GEMM; 16x16 tiles, 2 stages of 100 KB, one CTA
// with 8 compute warps per SM).
//
// The kernel is FP32-FMA bound by construction (25 FMA per output element, issued as packed FFMA2 on channel pairs),
// so everything that is not an FMA is kept out of the compute warps:
//   * the 12x20 pixel x 64 channel input window of an 8x16 tile is ONE cp.async.bulk.tensor.4d issued by a loader
//     thread into a 3-stage shared-memory ring (the image border and the channel tail are the tensor map's
//     out-of-bounds zero fill: no address arithmetic, no bounds checks, no staging registers);
//   * CTAs are persistent per 64-channel group, so the 2 x 25 filter taps of a lane's channel pair are loaded once;
//   * 4 compute warps each own two output rows of the tile: 120 LDS.32 + 800 FFMA2 per 64 outputs.
// ncu on the previous version (software loads in the compute warps): 2690 instructions per warp and tile of which 800
// FFMA2, FMA pipe 50 % busy, 115 us for the 216x216x569 map; see DESIGN.md for the numbers of this one.
#include "tma.cuh"

namespace rb {

constexpr int DT_TW = 16, DT_CH = 64, DT_IW = DT_TW + 4;

template <typename TIN> struct DwCfg {
    static constexpr int TH = sizeof(TIN) == 4 ? 16 : 8;                 // output rows per tile (two per compute warp)
    static constexpr int IH = TH + 4;
    static constexpr int NWARPS = TH / 2;
    static constexpr int STAGES = sizeof(TIN) == 4 ? 2 : 3;
    static constexpr int STAGE_BYTES = IH * DT_IW * DT_CH * (int)sizeof(TIN);   // 30720 (16-bit, 12 rows) / 102400 (fp32, 20 rows)
    static constexpr int THREADS = 32 * (NWARPS + 1);                    // compute warps + loader warp
    static constexpr int SMEM = STAGES * STAGE_BYTES + 128 + 128;        // ring + alignment slack + barriers
};

#ifdef RB_FZ_CLK
__device__ long long g_dw_clk[16];
#endif

struct DwTmaParams {
    void* out; void* out_lo; int64_t ldo;
    const float* wgt; int64_t ldw; const float* bias;
    int H, W, C, tiles_x, tiles_per_img, total_tiles;
};

// TIN = __half / __nv_bfloat16: output in the same type.  TIN = float: output as an RB_F16S pair (out = hi plane, out_lo).
template <typename TIN>
__global__ void __launch_bounds__(DwCfg<TIN>::THREADS) dwconv5x5_relu_tma_kernel(const __grid_constant__ CUtensorMap map_in, const DwTmaParams p) {
    using Cfg = DwCfg<TIN>;
    constexpr int STAGES = Cfg::STAGES, STAGE_BYTES = Cfg::STAGE_BYTES, TH = Cfg::TH, NW = Cfg::NWARPS;
    constexpr bool F32IN = sizeof(TIN) == 4;
    extern __shared__ uint8_t dsm_raw[];
    uint8_t* ring = dsm_raw + ((128u - ((uint32_t)__cvta_generic_to_shared(dsm_raw) & 127u)) & 127u);   // offset on the array: keeps ld.shared
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + STAGES * STAGE_BYTES);
    uint64_t* empty = full + STAGES;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NW); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    rb::pdl_wait();                                    // everything above overlapped the previous kernel's tail
    const int c0 = blockIdx.y * DT_CH;

    if (wid == NW) {
        if (lane == 0) {
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
                const int s = it % STAGES, round = it / STAGES;
                const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
                const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
                if (round > 0) mbar_wait(&empty[s], (round - 1) & 1);
                mbar_expect_tx(&full[s], STAGE_BYTES);
                tma_load_4d(ring + s * STAGE_BYTES, &map_in, &full[s], c0, tx * DT_TW - 2, ty * TH - 2, img);
            }
        }
        return;
    }
    const int c = c0 + 2 * lane;
    const bool ok0 = c < p.C, ok1 = c + 1 < p.C;
    float2 wv[25];                                        // (channel c, channel c+1) taps: operands of the packed FFMA2
#pragma unroll
    for (int t = 0; t < 25; ++t) wv[t] = make_float2(ok0 ? p.wgt[(int64_t)t * p.ldw + c] : 0.f, ok1 ? p.wgt[(int64_t)t * p.ldw + c + 1] : 0.f);
    const float2 bv = make_float2(ok0 ? p.bias[c] : 0.f, ok1 ? p.bias[c + 1] : 0.f);
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x, ++it) {
        const int s = it % STAGES, round = it / STAGES;
        const int img = tile / p.tiles_per_img, r = tile - img * p.tiles_per_img;
        const int ty = r / p.tiles_x, tx = r - ty * p.tiles_x;
        const int x0 = tx * DT_TW, y0 = ty * TH;
        const TIN* tile_s = reinterpret_cast<const TIN*>(ring + s * STAGE_BYTES);
#ifdef RB_FZ_CLK
        const long long t0 = clock64();
#endif
        mbar_wait(&full[s], round & 1);
#ifdef RB_FZ_CLK
        const long long t1 = clock64();
#endif
        float2 acc[2][DT_TW];
#pragma unroll
        for (int rr = 0; rr < 2; ++rr)
#pragma unroll
            for (int i = 0; i < DT_TW; ++i) acc[rr][i] = bv;
#pragma unroll
        for (int iy = 0; iy < 6; ++iy) {                      // input rows 2*wid + iy of the window feed output rows 2*wid + {0, 1}
#pragma unroll
            for (int px = 0; px < DT_IW; ++px) {
                float2 v;
                if constexpr (F32IN) {
                    v = *reinterpret_cast<const float2*>(&tile_s[((2 * wid + iy) * DT_IW + px) * DT_CH + 2 * lane]);
                } else {
                    TIN pr[2];
                    *reinterpret_cast<uint32_t*>(pr) = *reinterpret_cast<const uint32_t*>(&tile_s[((2 * wid + iy) * DT_IW + px) * DT_CH + 2 * lane]);
                    v = make_float2(to_f(pr[0]), to_f(pr[1]));
                }
#pragma unroll
                for (int rr = 0; rr < 2; ++rr) {
                    const int ky = iy - rr;
                    if (ky >= 0 && ky < 5) {
#pragma unroll
                        for (int kx = 0; kx < 5; ++kx) {
                            const int ox = px - kx;
                            if (ox >= 0 && ox < DT_TW) acc[rr][ox] = rb::fma2(wv[ky * 5 + kx], v, acc[rr][ox]);
                        }
                    }
                }
            }
        }
#ifdef RB_FZ_CLK
        const long long t2 = clock64();
#endif
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[s]);                // this warp no longer reads the stage
        if (ok0) {
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int yy = y0 + 2 * wid + rr;
                if (yy < p.H) {
                    const int64_t o0 = ((int64_t)img * p.H * p.W + (int64_t)yy * p.W) * p.ldo + c;
#pragma unroll
                    for (int i = 0; i < DT_TW; ++i) {
                        if (x0 + i < p.W) {
                            const float r0 = fmaxf(acc[rr][i].x, 0.f), r1 = ok1 ? fmaxf(acc[rr][i].y, 0.f) : 0.f;
                            if constexpr (F32IN) {
                                __half hi[2], lo[2];
                                split_f16s(r0, hi[0], lo[0]); split_f16s(r1, hi[1], lo[1]);
                                *reinterpret_cast<uint32_t*>((__half*)p.out + o0 + (int64_t)(x0 + i) * p.ldo) = *reinterpret_cast<uint32_t*>(hi);
                                *reinterpret_cast<uint32_t*>((__half*)p.out_lo + o0 + (int64_t)(x0 + i) * p.ldo) = *reinterpret_cast<uint32_t*>(lo);
                            } else {
                                TIN pair[2] = {from_f<TIN>(r0), from_f<TIN>(r1)};
                                *reinterpret_cast<uint32_t*>((TIN*)p.out + o0 + (int64_t)(x0 + i) * p.ldo) = *reinterpret_cast<uint32_t*>(pair);
                            }
                        }
                    }
                }
            }
        }
#ifdef RB_FZ_CLK
        if (blockIdx.x == 0 && blockIdx.y == 0 && lane == 0 && wid == 0) { const long long t3 = clock64(); g_dw_clk[0] += t1 - t0; g_dw_clk[1] += t2 - t1; g_dw_clk[2] += t3 - t2; g_dw_clk[3] += 1; }
#endif
    }
}

#ifdef RB_FZ_CLK
extern "C" int romab200_debug_dwclk(long long* out, int reset) {
    if (reset) { long long z[16] = {0}; return (int)cudaMemcpyToSymbol(g_dw_clk, z, sizeof(z)); }
    return (int)cudaMemcpyFromSymbol(out, g_dw_clk, sizeof(long long) * 16);
}
#endif

// 16-bit maps (same type out), or fp32 maps with an RB_F16S result (a->out_lo != NULL); the caller has checked the pitches
// (ldi * element size % 16 == 0, ldo % 2 == 0) and the 16-byte alignment of the input.
int dwconv_tma(const rb_dwconv_args* a, cudaStream_t st) {
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "dwconv", [&](auto t) {
        using TIN = typename decltype(t)::type;
        using Cfg = DwCfg<TIN>;
        constexpr bool f32 = std::is_same_v<TIN, float>;
        RB_REQUIRE(!f32 || a->out_lo, "dwconv_tma: fp32 maps need the RB_F16S output planes");
        const uint64_t es = sizeof(TIN);
        CUtensorMap map;             // activation [B, H, W, C] with pitch ldi: box = (TH+4) x 20 pixels x 64 channels, borders zero-filled
        cuuint64_t d4[4] = {(cuuint64_t)a->c, (cuuint64_t)a->w, (cuuint64_t)a->h, (cuuint64_t)a->batch};
        cuuint64_t s4[3] = {(cuuint64_t)a->ldi * es, (cuuint64_t)a->w * a->ldi * es, (cuuint64_t)a->h * a->w * a->ldi * es};
        cuuint32_t b4[4] = {(cuuint32_t)DT_CH, (cuuint32_t)DT_IW, (cuuint32_t)(Cfg::TH + 4), 1};
        if (encode_tiled(&map, "dwconv", tma_dtype(a->dtype), 4, a->in, d4, s4, b4, CU_TENSOR_MAP_SWIZZLE_NONE)) return 1;
        DwTmaParams p;
        p.out = a->out; p.out_lo = a->out_lo; p.ldo = a->ldo; p.wgt = a->weight; p.ldw = a->ldw; p.bias = a->bias;
        p.H = a->h; p.W = a->w; p.C = a->c;
        p.tiles_x = (a->w + DT_TW - 1) / DT_TW;
        p.tiles_per_img = p.tiles_x * ((a->h + Cfg::TH - 1) / Cfg::TH);
        const long long total = (long long)p.tiles_per_img * a->batch;
        RB_REQUIRE(total > 0 && total < (1ll << 31), "dwconv: bad tile count");
        p.total_tiles = (int)total;
        const int groups = (a->c + DT_CH - 1) / DT_CH;
        RB_REQUIRE(groups <= 65535, "dwconv: too many channel groups");
        int per_group = (f32 ? 1 : 2) * sm_count() / groups;             // resident CTAs per SM (one for the fp32 ring), never more CTAs than fit at once
        if (per_group < 1) per_group = 1;
        if (per_group > p.total_tiles) per_group = p.total_tiles;
        if (ensure_smem<dwconv5x5_relu_tma_kernel<TIN>>(Cfg::SMEM, "dwconv")) return 1;
        rb::launch_pdl(dwconv5x5_relu_tma_kernel<TIN>, dim3(per_group, groups), dim3(Cfg::THREADS), Cfg::SMEM, st, map, p);
        return check_launch("dwconv5x5_relu_tma");
    });
}

}  // namespace rb
