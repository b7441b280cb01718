// Tensor-core (wgmma) / TMA back-end of romab200_gemm: fp16 / bf16 operands, fp32 accumulation in registers.
//
// Persistent kernel; one CTA computes one 128 x BN output tile at a time (BN in {32, 64, 128, 144, 192, 256}).  Warp roles:
//   warps 0-7   two consumer warpgroups, 64 rows of the tile each: wgmma.mma_async (m64 x BN x k16, 4 per k-block) from the
//               STAGES-deep 128B-swizzled shared-memory ring into fp32 register accumulators, then the fused epilogue: 32
//               columns at a time, the accumulators go through the warpgroup's shared-memory staging buffer, and a rolled loop
//               in which each thread owns 8 consecutive columns of a row applies the epilogue and stores 16-byte vectors;
//   warps 8-11  TMA producer: one lane issues cp.async.bulk.tensor loads of the A (128 x 64) and B (BN x 64, or 64 x BN when B
//               is [K,N]) tiles; it runs ahead into the next tile while the consumers are in their epilogue.  The producer
//               warpgroup hands its registers to the consumers (setmaxnreg), whose accumulators take up to 144 per thread.
// A-operand "taps" (the 9 shifted row blocks of a 3x3 convolution on a zero-padded channels-last map) are just a per-k-block row
// offset on the TMA coordinate; out-of-range rows/columns are zero-filled by TMA, which also handles M/N/K tails, so no operand is
// ever padded or copied.  Batched GEMMs (attention heads) use the 3rd/4th tensor-map dimension.
//
// SPLIT variant (dtype_ab == RB_F16S): fp32-class accuracy on the f16 tensor pipe.  Every operand element x is stored as two fp16
// planes, hi = fp16(x) and lo = fp16((x - hi) * 2^11), i.e. 22 significand bits with the exponent range of fp16 and no underflow of
// the low part.  Per k-step each warpgroup issues three MMAs into two accumulators, acc0 += A_hi.B_hi and acc1 += A_hi.B_lo +
// A_lo.B_hi; the epilogue forms acc0 + acc1 * 2^-11 (the dropped A_lo.B_lo term is 2^-22 relative).  Products of fp16 values are
// exact in the fp32 accumulator, so the only error left is the 2^-22 operand representation and the fp32 accumulation itself.
#include "tma.cuh"
#include "wgmma.cuh"

namespace rb {

// ------------------------------------------------------------------------------------------------
struct TcParams {
    int M, N, K;
    int batch1;
    int ntaps, k_per_tap; int tap_rows[9];
    int tiles_m, tiles_n, total_tiles;
    int band_m;                   // M-tiles per band of the tile order (tile_coords); tiles_m: plain m-fastest order
    int n_zero_to;                // columns [N, n_zero_to) of every stored row are written with zeros (pad up to a 16-byte granule)
    int64_t sc0, sc1, sr0, sr1, sna0, snb0;
    Epilogue epi;
};

constexpr int TC_BM = 128, TC_BK = 64;
constexpr int TC_THREADS = 384;                    // two consumer warpgroups + one producer warpgroup
// epilogue staging: each consumer warpgroup owns a 64 x TC_CW fp32 buffer; rows are TC_SP floats apart (40: the accumulator
// fragments' float2 writes and the row readers' float4 reads are both free of bank conflicts)
constexpr int TC_CW = 32, TC_SP = 40;
constexpr int TC_STAGING = 2 * 64 * TC_SP * 4;

template <int BN, bool SPLIT> struct TcCfg {
    static constexpr int NOPS = SPLIT ? 2 : 1;                           // operand planes per matrix
    static constexpr int A_BYTES = TC_BM * TC_BK * 2;
    static constexpr int B_BYTES = BN * TC_BK * 2;                       // a multiple of 1024: every plane stays swizzle-atom aligned
    static constexpr int STAGE_BYTES = NOPS * (A_BYTES + B_BYTES);
    static constexpr int RING_MAX = 232448 - TC_STAGING - 1024 /*align*/ - 256 /*barriers*/;
    static constexpr int STAGES = RING_MAX / STAGE_BYTES > 8 ? 8 : RING_MAX / STAGE_BYTES;
    static constexpr int SMEM = STAGES * STAGE_BYTES + TC_STAGING + 1024 + 256;
    static_assert(STAGES >= 3 && SMEM <= 232448, "shared memory budget");
};

// cnt (<= 8) consecutive elements of a 16-bit or fp32 matrix as floats: two 16-byte loads (fp32) or one (16-bit) when all 8 are
// wanted and the address allows it
__device__ __forceinline__ void load8(const void* p, int64_t i, int dtype, int cnt, float (&v)[8]) {
    if (dtype == RB_F32) {
        const float* s = (const float*)p + i;
        if (cnt == 8 && (reinterpret_cast<uintptr_t>(s) & 15) == 0) {
            const float4 a = reinterpret_cast<const float4*>(s)[0], b = reinterpret_cast<const float4*>(s)[1];
            v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = k < cnt ? s[k] : 0.f;
        }
        return;
    }
    const uint16_t* s = (const uint16_t*)p + i;
    uint16_t h[8];
    if (cnt == 8 && (reinterpret_cast<uintptr_t>(s) & 15) == 0) {
        const uint4 q = *reinterpret_cast<const uint4*>(s);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) { h[2 * k] = (uint16_t)w[k]; h[2 * k + 1] = (uint16_t)(w[k] >> 16); }
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) h[k] = k < cnt ? s[k] : 0;
    }
    if (dtype == RB_F16) {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __half2float(__ushort_as_half(h[k]));
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __bfloat162float(__ushort_as_bfloat16(h[k]));
    }
}

// cnt (<= 8) consecutive output elements starting at element i of C (and C_lo): 16-byte stores when all 8 go out and the address
// allows it, scalar stores otherwise.  Rounding is that of store_split_any.
__device__ __forceinline__ void store8(const Epilogue& e, int64_t i, int cnt, const float (&v)[8]) {
    if (e.dtype_c == RB_F32) {
        float* c = (float*)e.C + i;
        if (cnt == 8 && (reinterpret_cast<uintptr_t>(c) & 15) == 0) {
            reinterpret_cast<float4*>(c)[0] = make_float4(v[0], v[1], v[2], v[3]);
            reinterpret_cast<float4*>(c)[1] = make_float4(v[4], v[5], v[6], v[7]);
        } else {
#pragma unroll
            for (int k = 0; k < 8; ++k) if (k < cnt) c[k] = v[k];
        }
        return;
    }
    uint16_t h[8], l[8];
    const bool two = e.dtype_c == RB_F16S;
    if (e.dtype_c == RB_BF16) {
#pragma unroll
        for (int k = 0; k < 8; ++k) h[k] = __bfloat16_as_ushort(__float2bfloat16_rn(v[k]));
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            __half hi, lo;
            split_f16s(v[k], hi, lo);
            h[k] = __half_as_ushort(hi); l[k] = __half_as_ushort(lo);
        }
    }
    uint16_t* c = (uint16_t*)e.C + i;
    uint16_t* cl = two ? (uint16_t*)e.C_lo + i : nullptr;
    if (cnt == 8 && (reinterpret_cast<uintptr_t>(c) & 15) == 0 && (!two || (reinterpret_cast<uintptr_t>(cl) & 15) == 0)) {
        *reinterpret_cast<uint4*>(c) = make_uint4(h[0] | (uint32_t)h[1] << 16, h[2] | (uint32_t)h[3] << 16, h[4] | (uint32_t)h[5] << 16,
                                                  h[6] | (uint32_t)h[7] << 16);
        if (two) *reinterpret_cast<uint4*>(cl) = make_uint4(l[0] | (uint32_t)l[1] << 16, l[2] | (uint32_t)l[3] << 16,
                                                            l[4] | (uint32_t)l[5] << 16, l[6] | (uint32_t)l[7] << 16);
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) if (k < cnt) { c[k] = h[k]; if (two) cl[k] = l[k]; }
    }
}

// Epilogue of 8 consecutive columns n .. n + 7 of one stored row (logical row m, stored row orow): the same operations in the same
// order as Epilogue::apply (the _rn intrinsics keep the multiplies and adds from being contracted into FMAs), with every per-launch
// option tested once for the 8 values.  cb / cs hold bias (COSKERNEL: norm_b) and col_scale of the 8 columns, na norm_a[m].
// Columns in [N, nz) become zeros; cnt = the number of columns below nz.
__device__ __forceinline__ void epilogue8(const Epilogue& e, int m, int n, int64_t orow, int cnt, const float (&cb)[8],
                                          const float (&cs)[8], float na, float (&v)[8]) {
    const int nv = min(8, e.N - n);                  // columns holding results
    if (e.epi == RB_EPI_COSKERNEL) {
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float p = na * cb[k];
            const float s = e.cos_normalized ? p / (p + e.eps) : 1.0f / (p + e.eps);
            v[k] = expf((v[k] * s - 1.0f) * e.inv_t);
            if (m == n + k) v[k] += e.diag_add;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = __fmul_rn(e.alpha, v[k]);
        if (e.bias) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __fadd_rn(v[k], cb[k]);
        }
        if (e.act == RB_ACT_RELU) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = fmaxf(v[k], 0.0f);
        } else if (e.act == RB_ACT_GELU) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = gelu_erf(v[k]);
        }
        if (e.col_scale) {
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __fmul_rn(v[k], cs[k]);
        }
        if (e.R) {
            float r[8];
            load8(e.R, orow * e.ldr + n, e.dtype_r, nv, r);
#pragma unroll
            for (int k = 0; k < 8; ++k) v[k] = __fadd_rn(v[k], r[k]);
        }
    }
    if (nv < 8) {
#pragma unroll
        for (int k = 0; k < 8; ++k) if (k >= nv) v[k] = 0.f;
    }
    store8(e, orow * e.ldc + n, cnt, v);
}

// Output tile of work index w: z outermost; inside one z, bands of p.band_m consecutive M-tiles (the last band may be shorter), each
// band walked m-fastest over all tiles_n N-tiles.  band_m == tiles_m is the plain m-fastest order.
__device__ __forceinline__ void tile_coords(const TcParams& p, int w, int& z, int& mt, int& nt) {
    const int per_z = p.tiles_m * p.tiles_n;
    z = w / per_z;
    const int r = w - z * per_z;
    const int m_lo = r / (p.band_m * p.tiles_n) * p.band_m;
    const int rows = min(p.band_m, p.tiles_m - m_lo);
    const int rb = r - m_lo * p.tiles_n;
    nt = rb / rows;
    mt = m_lo + (rb - nt * rows);
}

// Persistent kernel: every CTA walks work indices w = blockIdx.x, blockIdx.x + gridDim.x, ... in the order of tile_coords.  The
// host picks the band height (launch_tc): m-fastest (one band), so that CTAs that run together share the weight tile in L2, unless
// the activation A is too big to stay in L2 while the N-tiles sweep over it; then bands of about one wave of the grid read each
// A row from HBM once while the weights stay resident.  Only the assignment of tiles to CTAs changes: every tile's result is
// computed by the same instructions on the same data, so the results are bit-identical in either order.
template <int BN, bool SPLIT, bool BF16, int TB>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_a_lo, const __grid_constant__ CUtensorMap map_b_lo, const TcParams p) {
    using Cfg = TcCfg<BN, SPLIT>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int A_BYTES = Cfg::A_BYTES, B_BYTES = Cfg::B_BYTES;
    constexpr int OFF_A_LO = A_BYTES, OFF_B = Cfg::NOPS * A_BYTES, OFF_B_LO = Cfg::NOPS * A_BYTES + B_BYTES;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - ((uint32_t)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);   // offset on the array: keeps ld/st.shared
    float* staging = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + TC_STAGING);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int kblocks = (p.K + TC_BK - 1) / TC_BK;

    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    // programmatic dependent launch: the set-up above overlapped the tail of the previous kernel in the stream; its results may only
    // be touched after this point
    rb::pdl_wait();

    if (warp >= 8) {
        // ===== TMA producer =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            const int kb_per_tap = p.ntaps > 1 ? p.k_per_tap / TC_BK : kblocks;
            uint32_t it = 0;
            for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
                int z, mt, nt;
                tile_coords(p, tile, z, mt, nt);
                const int m0 = mt * TC_BM, n0 = nt * BN, z0 = z / p.batch1, z1 = z - z0 * p.batch1;
                for (int kb = 0; kb < kblocks; ++kb, ++it) {
                    const int s = it % STAGES;
                    const uint32_t ph = (it / STAGES) & 1;
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
                    int tap = 0, kin = kb * TC_BK, shift = 0;
                    if (p.ntaps > 1) { tap = kb / kb_per_tap; kin = (kb - tap * kb_per_tap) * TC_BK; shift = p.tap_rows[tap]; }
                    uint8_t* st = smem + s * Cfg::STAGE_BYTES;
                    tma_load_4d(st, &map_a, &full_bar[s], kin, m0 + shift, z1, z0);
                    if constexpr (SPLIT) tma_load_4d(st + OFF_A_LO, &map_a_lo, &full_bar[s], kin, m0 + shift, z1, z0);
                    if constexpr (!TB) {
                        tma_load_4d(st + OFF_B, &map_b, &full_bar[s], kb * TC_BK, n0, z1, z0);
                        if constexpr (SPLIT) tma_load_4d(st + OFF_B_LO, &map_b_lo, &full_bar[s], kb * TC_BK, n0, z1, z0);
                    } else {
                        // B is [K, N]: boxes of 64 (n) x 64 (k); one box per 64 columns of the tile
#pragma unroll
                        for (int j = 0; j < (BN + 63) / 64; ++j) {
                            tma_load_4d(st + OFF_B + j * (64 * 128), &map_b, &full_bar[s], n0 + j * 64, kb * TC_BK, z1, z0);
                            if constexpr (SPLIT) tma_load_4d(st + OFF_B_LO + j * (64 * 128), &map_b_lo, &full_bar[s], n0 + j * 64, kb * TC_BK, z1, z0);
                        }
                    }
                }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2, t = threadIdx.x & 127;
    float acc[BN / 2];
    float acc2[SPLIT ? BN / 2 : 1];
    uint32_t it = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
        int z, mt, nt;
        tile_coords(p, tile, z, mt, nt);
        const int m0 = mt * TC_BM, n0 = nt * BN, z0 = z / p.batch1, z1 = z - z0 * p.batch1;
        int prev = -1;
        for (int kb = 0; kb < kblocks; ++kb, ++it) {
            const int s = it % STAGES;
            mbar_wait(&full_bar[s], (it / STAGES) & 1);
            const uint32_t st = smem_u32(smem + s * Cfg::STAGE_BYTES);
            // all four k-steps are issued: those beyond K multiply TMA zero fill (a branch here would serialise the wgmmas)
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_BK / 16; ++k) {
                // K-major SW128: 8-row groups are 1024 B apart (SBO); a K step of 16 elements = +32 B inside the atom.  MN-major B
                // ([K,N] boxes of 64 columns): 16 k-rows = 2048 B, the next 64 columns 8 KB further (LBO).
                const uint32_t koff_a = wg * (64 * 128) + k * 32;
                const uint32_t koff_b = TB ? k * 2048 : k * 32;
                const uint32_t lbo_b = TB ? 64 * 128 : 16;
                const uint64_t a_hi = gmma_desc(st + koff_a, 16, 1024);
                const uint64_t b_hi = gmma_desc(st + OFF_B + koff_b, lbo_b, 1024);
                const int accum = (kb | k) != 0;
                Wgmma<BN, BF16>::template ss<TB>(acc, a_hi, b_hi, accum);
                if constexpr (SPLIT) {
                    const uint64_t a_lo = gmma_desc(st + OFF_A_LO + koff_a, 16, 1024);
                    const uint64_t b_lo = gmma_desc(st + OFF_B_LO + koff_b, lbo_b, 1024);
                    Wgmma<BN, BF16>::template ss<TB>(acc2, a_hi, b_lo, accum);
                    Wgmma<BN, BF16>::template ss<TB>(acc2, a_lo, b_hi, 1);
                }
            }
            wgmma_commit();
            // keep this k-block's MMAs in flight; the previous k-block's have retired, so its ring slot is free
            wgmma_wait<1>();
            if (prev >= 0 && t == 0) mbar_arrive(&empty_bar[prev]);
            prev = s;
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if constexpr (SPLIT) wgmma_fence_regs(acc2);
        if (t == 0) mbar_arrive(&empty_bar[prev]);

        // ===== epilogue, TC_CW columns at a time: the warpgroup copies its accumulator fragments (thread t: rows fr, fr + 8, column
        // pairs 8 j + 2 (t % 4)) into its staging buffer, then every thread takes 8 consecutive columns of rows rr and rr + 32 of the
        // chunk and runs the fused epilogue on them with 16-byte stores.  Named barriers: the other warpgroup and the producer run on.
        Epilogue e = p.epi;
        e.C = (char*)e.C + (z0 * p.sc0 + z1 * p.sc1) * dtype_size(e.dtype_c);
        if (e.C_lo) e.C_lo = (char*)e.C_lo + (z0 * p.sc0 + z1 * p.sc1) * 2;
        if (e.R) e.R = (const char*)e.R + (z0 * p.sr0 + z1 * p.sr1) * dtype_size(e.dtype_r);
        if (e.norm_a) e.norm_a += z0 * p.sna0;
        if (e.norm_b) e.norm_b += z0 * p.snb0;
        float* stg = staging + wg * (64 * TC_SP);
        const int fr = (t >> 5) * 16 + ((t & 31) >> 2), fc = 2 * (t & 3);
        const int g = t & 3, rr = t >> 2;
        // the two rows this thread stores: logical row, stored row (-1: not stored) and norm_a
        int mrow[2]; int64_t orow[2]; float na[2] = {0.f, 0.f};
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mrow[h] = m0 + wg * 64 + rr + 32 * h;
            orow[h] = mrow[h] < e.M ? e.map_row(mrow[h]) : -1;
            if (orow[h] >= 0 && e.epi == RB_EPI_COSKERNEL) na[h] = e.norm_a[mrow[h]];
        }
        constexpr int NCH = (BN + TC_CW - 1) / TC_CW;
#pragma unroll 1
        for (int ch = 0; ch < NCH; ++ch) {
            if (n0 + ch * TC_CW >= p.n_zero_to) break;
            bar_named(1 + wg, 128);                 // the previous chunk's readers are done with the buffer
#pragma unroll
            for (int c = 0; c < NCH; ++c) {
                if (c != ch) continue;
#pragma unroll
                for (int jj = 0; jj < TC_CW / 8; ++jj) {
                    const int j = c * (TC_CW / 8) + jj;
                    if (j >= BN / 8) break;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
                        if constexpr (SPLIT) {
                            v0 = fmaf(acc2[4 * j + 2 * h], 1.0f / RB_SPLIT_SCALE, v0);
                            v1 = fmaf(acc2[4 * j + 2 * h + 1], 1.0f / RB_SPLIT_SCALE, v1);
                        }
                        *reinterpret_cast<float2*>(stg + (fr + 8 * h) * TC_SP + 8 * jj + fc) = make_float2(v0, v1);
                    }
                }
            }
            bar_named(1 + wg, 128);
            const int n = n0 + ch * TC_CW + 8 * g;
            if (ch * TC_CW + 8 * g >= BN || n >= p.n_zero_to) continue;
            const int cnt = min(8, p.n_zero_to - n);
            float cb[8], cs[8];
            const float* colb = e.epi == RB_EPI_COSKERNEL ? e.norm_b : e.bias;
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const bool in = n + k < e.N;
                cb[k] = colb && in ? colb[n + k] : 0.f;
                cs[k] = e.col_scale && in ? e.col_scale[n + k] : 0.f;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (orow[h] < 0) continue;
                // odd rows read their two halves in the other order: the 8 lanes of a 16-byte load phase then hit 32 distinct banks
                const float* src = stg + (rr + 32 * h) * TC_SP + 8 * g;
                const int q = (rr & 1) * 4;
                const float4 a = *reinterpret_cast<const float4*>(src + q), b = *reinterpret_cast<const float4*>(src + (4 - q));
                float v[8];
                if (q == 0) { v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w; }
                else        { v[0] = b.x; v[1] = b.y; v[2] = b.z; v[3] = b.w; v[4] = a.x; v[5] = a.y; v[6] = a.z; v[7] = a.w; }
                epilogue8(e, mrow[h], n, orow[h], cnt, cb, cs, na[h], v);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// 4-D map over (inner, rows, batch1, batch0) of a 16-bit matrix of dtype code `dtype` (RB_F16S: either plane)
static int make_map(CUtensorMap* map, const void* base, int dtype, uint64_t inner, uint64_t rows, uint64_t pitch_elems, uint64_t b1,
                    uint64_t s1_elems, uint64_t b0, uint64_t s0_elems, uint32_t box_inner, uint32_t box_rows) {
    RB_REQUIRE(((uintptr_t)base) % 16 == 0 && (pitch_elems * 2) % 16 == 0, "gemm_tc: operand base/pitch must be 16-byte aligned (pitch %llu elems)", (unsigned long long)pitch_elems);
    RB_REQUIRE((b1 <= 1 || (s1_elems * 2) % 16 == 0) && (b0 <= 1 || (s0_elems * 2) % 16 == 0), "gemm_tc: batch strides must be 16-byte aligned");
    cuuint64_t dims[4] = {inner, rows, b1 > 0 ? b1 : 1, b0 > 0 ? b0 : 1};
    cuuint64_t strides[3] = {pitch_elems * 2, (b1 > 1 ? s1_elems : pitch_elems * rows) * 2, (b0 > 1 ? s0_elems : pitch_elems * rows) * 2};
    cuuint32_t box[4] = {box_inner, box_rows, 1, 1};
    return encode_tiled(map, "gemm_tc", tma_dtype(dtype), 4, base, dims, strides, box,
                        CU_TENSOR_MAP_SWIZZLE_128B);
}

struct TcMaps { CUtensorMap a, b, a_lo, b_lo; };

template <int BN, bool SPLIT, bool BF16, int TB>
static int launch_tc(const TcMaps& maps, TcParams& p, int zdim, int max_ctas, cudaStream_t st) {
    using Cfg = TcCfg<BN, SPLIT>;
    auto kernel = gemm_tc_kernel<BN, SPLIT, BF16, TB>;
    if (ensure_smem<gemm_tc_kernel<BN, SPLIT, BF16, TB>>(Cfg::SMEM, "gemm_tc")) return 1;
    p.tiles_m = (p.M + TC_BM - 1) / TC_BM;
    p.tiles_n = (p.N + BN - 1) / BN;
    const long long total = (long long)p.tiles_m * p.tiles_n * zdim;
    RB_REQUIRE(total < (1ll << 31), "gemm_tc: too many tiles");
    p.total_tiles = (int)total;
    int resident = sm_count();
    if (max_ctas > 0 && max_ctas < resident) resident = max_ctas;
    const int grid = p.total_tiles < resident ? p.total_tiles : resident;
    // Tile order.  m-fastest comes back to an A row once per N-tile, after a sweep over all of A (per z) and the C it writes: when
    // A is more than half the L2, the row has been evicted and is read from HBM tiles_n times.  Bands of grid / tiles_n M-tiles
    // (one wave: every CTA that reads a band's A rows runs at once) read A from HBM once; every band reads all of B, so B must
    // stay resident beside the band (at most half the L2).  Measured with scripts/bench_gemm.py on the parity-mode step (H100,
    // 50 MB L2): the refiner pointwise GEMMs at C = 569 / 1137 (A 45-212 MB) run 6-14% faster in bands, and launches with A
    // between a half and one L2 (41-50 MB) from 3% slower to 27% faster, most of them faster; the ViT qkv / fc1 and decoder GEMMs (A <= 18 MB) keep m-fastest.
    const int64_t a_bytes = (int64_t)p.M * (p.ntaps > 1 ? p.k_per_tap : p.K) * Cfg::NOPS * 2;
    const int64_t b_bytes = (int64_t)p.N * p.K * Cfg::NOPS * 2;
    const bool bands = p.tiles_n > 1 && 2 * a_bytes > l2_bytes() && 2 * b_bytes <= l2_bytes();
    const int band_m = grid / p.tiles_n > 1 ? grid / p.tiles_n : 1;
    p.band_m = bands && band_m < p.tiles_m ? band_m : p.tiles_m;
    cudaError_t err = rb::launch_pdl(kernel, dim3(grid), dim3(TC_THREADS), Cfg::SMEM, st, maps.a, maps.b, maps.a_lo, maps.b_lo, (const TcParams)p);
    if (err != cudaSuccess) { set_error("gemm_tc: launch failed: %s", cudaGetErrorString(err)); return 1; }
    return check_launch("gemm_tc");
}

template <bool SPLIT, bool BF16>
static int dispatch_tc(int BN, int trans_b, const TcMaps& maps, TcParams& p, int zdim, int max_ctas, cudaStream_t st) {
    if (trans_b) return BN == 64 ? launch_tc<64, SPLIT, BF16, 1>(maps, p, zdim, max_ctas, st) : launch_tc<128, SPLIT, BF16, 1>(maps, p, zdim, max_ctas, st);
    switch (BN) {
        case 32: return launch_tc<32, SPLIT, BF16, 0>(maps, p, zdim, max_ctas, st);
        case 64: return launch_tc<64, SPLIT, BF16, 0>(maps, p, zdim, max_ctas, st);
        case 128: return launch_tc<128, SPLIT, BF16, 0>(maps, p, zdim, max_ctas, st);
        case 144: return launch_tc<144, SPLIT, BF16, 0>(maps, p, zdim, max_ctas, st);
        default:
            if constexpr (SPLIT) { set_error("gemm_tc: split-fp16 tiles are at most 144 columns wide (got %d)", BN); return 1; }
            else {
                switch (BN) {
                    case 192: return launch_tc<192, false, BF16, 0>(maps, p, zdim, max_ctas, st);
                    default: return launch_tc<256, false, BF16, 0>(maps, p, zdim, max_ctas, st);
                }
            }
    }
}

int gemm_tc(const rb_gemm_args* a, cudaStream_t stream) {
    RB_REQUIRE(a->dtype_ab == RB_F16 || a->dtype_ab == RB_BF16 || a->dtype_ab == RB_F16S, "gemm_tc: operands must be fp16/bf16/split-fp16 (got %d)", a->dtype_ab);
    RB_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "gemm_tc: empty problem");
    const bool split = a->dtype_ab == RB_F16S;
    RB_REQUIRE(!split || (a->A_lo && a->B_lo), "gemm_tc: split-fp16 operands need A_lo and B_lo");
    RB_REQUIRE(a->dtype_c != RB_F16S || a->C_lo, "gemm_tc: split-fp16 output needs C_lo");
    TcParams p;
    p.M = a->M; p.N = a->N; p.K = a->K;
    p.batch1 = a->batch1 > 0 ? a->batch1 : 1;
    const int batch0 = a->batch0 > 0 ? a->batch0 : 1;
    p.ntaps = a->ntaps > 1 ? a->ntaps : 1;
    p.k_per_tap = a->K / p.ntaps;
    for (int i = 0; i < 9; ++i) p.tap_rows[i] = a->tap_rows[i];
    const bool bf16 = a->dtype_ab == RB_BF16;
    p.sc0 = a->sc0; p.sc1 = a->sc1; p.sr0 = a->sr0; p.sr1 = a->sr1; p.sna0 = a->sna0; p.snb0 = a->snb0;
    p.epi = make_epilogue(a);
    if (p.ntaps > 1) {
        RB_REQUIRE(a->K % p.ntaps == 0 && p.k_per_tap % TC_BK == 0, "gemm_tc: K/ntaps=%d must be a multiple of %d", p.k_per_tap, TC_BK);
        RB_REQUIRE(!a->trans_b && batch0 * p.batch1 == 1, "gemm_tc: taps need un-batched [N,K] weights");
    }
    const int zdim = batch0 * p.batch1;
    RB_REQUIRE(zdim <= 65535, "gemm_tc: batch too large");
    const int64_t a_rows = a->a_rows > 0 ? a->a_rows : a->M;
    // tile width: the narrowest that covers N up to 128; [N,K] weights wider than that take the width that wastes the fewest
    // columns (C = 144 / 569 / 1137 ...).  [K,N] operands load boxes of 64 columns (64 or 128 wide); split operands hold two
    // accumulators in registers, which caps them at 144: of 128 and 144 they take the one that pads fewer columns (ties: 128).
    int BN = a->N <= 32 && !a->trans_b ? 32 : (a->N <= 64 ? 64 : 128);
    if (!a->trans_b && a->N > 128) {
        if (split) BN = (a->N + 143) / 144 * 144 < (a->N + 127) / 128 * 128 ? 144 : 128;
        else if (a->N <= 144) BN = 144;
        else if (a->N <= 192) BN = 192;
        else {
            const int w192 = (a->N + 191) / 192 * 192 - a->N, w256 = (a->N + 255) / 256 * 256 - a->N;
            BN = (w192 + a->N / 20 < w256) ? 192 : 256;
        }
        // few tiles: keep 128-wide tiles so that more CTAs are in flight (below about two thirds of the SMs)
        if (((int64_t)((a->M + 127) / 128) * ((a->N + BN - 1) / BN) * zdim) < sm_count() * 2 / 3) BN = 128;
    }
    TcMaps maps;
    const uint64_t a_inner = p.ntaps > 1 ? p.k_per_tap : a->K;
    if (make_map(&maps.a, a->A, a->dtype_ab, a_inner, a_rows, a->lda, p.batch1, a->sa1, batch0, a->sa0, TC_BK, TC_BM)) return 1;
    if (split && make_map(&maps.a_lo, a->A_lo, a->dtype_ab, a_inner, a_rows, a->lda, p.batch1, a->sa1, batch0, a->sa0, TC_BK, TC_BM)) return 1;
    if (!a->trans_b) {
        if (make_map(&maps.b, a->B, a->dtype_ab, a->K, a->N, a->ldb, p.batch1, a->sb1, batch0, a->sb0, TC_BK, BN)) return 1;
        if (split && make_map(&maps.b_lo, a->B_lo, a->dtype_ab, a->K, a->N, a->ldb, p.batch1, a->sb1, batch0, a->sb0, TC_BK, BN)) return 1;
    } else {
        if (make_map(&maps.b, a->B, a->dtype_ab, a->N, a->K, a->ldb, p.batch1, a->sb1, batch0, a->sb0, 64, TC_BK)) return 1;
        if (split && make_map(&maps.b_lo, a->B_lo, a->dtype_ab, a->N, a->K, a->ldb, p.batch1, a->sb1, batch0, a->sb0, 64, TC_BK)) return 1;
    }
    if (!split) { maps.a_lo = maps.a; maps.b_lo = maps.b; }
    {
        // a plain (or zero-bordered) output with 16-byte aligned pitches and no residual operand gets the pad columns of its last
        // 16-byte granule zeroed, so that a later consumer reading whole granules never meets stale values
        const int es_c = dtype_size(a->dtype_c);
        const bool align_ok = ((uintptr_t)a->C) % 16 == 0 && (a->ldc * es_c) % 16 == 0 && (p.batch1 <= 1 || (a->sc1 * es_c) % 16 == 0) &&
                              (batch0 <= 1 || (a->sc0 * es_c) % 16 == 0) && (a->dtype_c != RB_F16S || ((uintptr_t)a->C_lo) % 16 == 0);
        const bool rowmap_ok = a->rowmap == RB_ROWMAP_NONE || a->rowmap == RB_ROWMAP_PAD_KEEP;
        const int gran = 16 / es_c;
        p.n_zero_to = align_ok && rowmap_ok && !a->R ? (a->N + gran - 1) / gran * gran : a->N;
    }
    if (split) return dispatch_tc<true, false>(BN, a->trans_b, maps, p, zdim, a->max_ctas, stream);
    return bf16 ? dispatch_tc<false, true>(BN, a->trans_b, maps, p, zdim, a->max_ctas, stream)
                : dispatch_tc<false, false>(BN, a->trans_b, maps, p, zdim, a->max_ctas, stream);
}

}  // namespace rb
