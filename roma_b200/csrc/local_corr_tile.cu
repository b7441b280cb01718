// Tile-cooperative ConvRefiner prologue for fp32 maps (matcher.py:132-168, local_correlation.py:77-142):
//   d = [x | grid_sample(y, flow) | disp_emb | local_corr]
// for a tile of TQX x TQY neighbouring pixels per CTA.  Where the flow is coherent (real image pairs: neighbouring
// pixels land on neighbouring pixels of the other image) the (2R+2)^2 integer neighbourhoods of the tile's pixels
// overlap almost entirely, so their union -- a box of (TQ + 2R + 1 + spread)^2 positions -- is staged ONCE per tile in
// shared memory, CK channels at a time through a two-stage cp.async ring (out-of-image positions are zero-filled by the
// copy itself = grid_sample's zero padding), instead of every pixel pulling its own 64..256 rows of f1 through L1/L2.
// One thread accumulates one row of one pixel's (2R+2)^2 dot products in registers; the lanes of a quarter-warp are the
// eight pixels of one tile row, whose window rows start in neighbouring columns of the box: with CK+4 floats per
// position and a box pitch that is a multiple of 8 positions their 16-byte shared loads fall into eight different
// bank groups (conflict-free; without the pitch rule a one-row difference between neighbours aliases them).  x and grid_sample(y) are produced from the
// same staged channels, so f0 and f1 are read exactly once per tile.  A tile whose box does not fit (incoherent flow,
// e.g. the seeded synthetic weights) writes tile_done = 0 and leaves its pixels to refiner_prologue_kernel
// (refiner.cu), which skips the pixels of finished tiles.
#include "refiner_common.cuh"
#include "tma.cuh"

namespace rb {

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int R>
struct LcTileSmem {
    using Cfg = LcTile<R>;
    static constexpr int TQ = Cfg::TQX * Cfg::TQY;
    static constexpr int S = 2 * R + 2;
    static constexpr int THREADS = TQ * S;                          // one thread per (pixel, window row)
    static constexpr int MIN_CTAS = R == 7 ? 2 : 3;
    static constexpr int ROWF = Cfg::CK + 4;                        // floats per staged position (16 B aligned, 4 mod 8 float4s)
    static constexpr int F1_FLOATS = Cfg::MAXPOS * ROWF;
    static constexpr int F0_FLOATS = TQ * ROWF;
    static constexpr int DT_PITCH = S * S + 1;
    static constexpr int BYTES = (2 * F1_FLOATS + 2 * F0_FLOATS) * 4;
    static_assert(TQ * DT_PITCH <= 2 * F1_FLOATS, "the D tables reuse the f1 stages");
    static_assert(THREADS % 32 == 0 && THREADS <= 256, "whole warps");
};

template <int R>
__global__ void __launch_bounds__(LcTileSmem<R>::THREADS, LcTileSmem<R>::MIN_CTAS)
refiner_prologue_tile_kernel(const PrologueParams p, unsigned char* __restrict__ tile_done) {
    using Cfg = LcTile<R>;
    using SM = LcTileSmem<R>;
    constexpr int TQX = Cfg::TQX, TQY = Cfg::TQY, TQ = SM::TQ, CK = Cfg::CK, ROWF = SM::ROWF, S = SM::S, NT = SM::THREADS;
    constexpr int C4 = CK / 4;                                      // 16-byte pieces per staged position
    static_assert(C4 == 4 && TQX == 8, "index arithmetic below");

    extern __shared__ __align__(16) float smem[];
    float* f1s = smem;                                              // [2][MAXPOS][ROWF]
    float* f0s = smem + 2 * SM::F1_FLOATS;                          // [2][TQ][ROWF]
    __shared__ int q_bx[TQ], q_by[TQ], q_off[TQ], q_pix[TQ];
    __shared__ float q_fx[TQ], q_fy[TQ];
    __shared__ int box[4];                                          // min bx, max bx, min by, max by
    __shared__ int plan[Cfg::MAXPOS];                               // per box position: element offset into the y image, -1 = zero fill, -2 = pad column

    rb::pdl_wait();
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int tiles_x = (p.w + TQX - 1) / TQX, tiles_y = (p.h + TQY - 1) / TQY;
    const int tile = blockIdx.x;
    const int item = tile / (tiles_x * tiles_y);
    const int trem = tile - item * tiles_x * tiles_y;
    const int ty0 = (trem / tiles_x) * TQY, tx0 = (trem % tiles_x) * TQX;
    const int64_t hw = (int64_t)p.h * p.w;
    const float* feat = (const float*)p.feat;
    const float* ximg = feat + (int64_t)item * hw * p.ldf;
    const float* yimg = feat + (int64_t)((item + p.y_shift) % p.n_img) * hw * p.ldf;

    if (tid == 0) { box[0] = INT_MAX; box[1] = INT_MIN; box[2] = INT_MAX; box[3] = INT_MIN; }
    __syncthreads();
    if (tid < TQ) {
        const int y = ty0 + tid / TQX, x = tx0 + tid % TQX;
        int pix = -1, bx = 0, by = 0;
        float fx = 0.f, fy = 0.f;
        if (y < p.h && x < p.w) {
            pix = (int)((int64_t)item * hw + (int64_t)y * p.w + x);
            fx = p.state[(int64_t)pix * 3 + 0]; fy = p.state[(int64_t)pix * 3 + 1];
            const float cx = ((fx + 1.f) * p.w - 1.f) * 0.5f, cy = ((fy + 1.f) * p.h - 1.f) * 0.5f;
            const float flx = floorf(cx), fly = floorf(cy);
            if (fabsf(flx) < 1e6f && fabsf(fly) < 1e6f) {
                bx = (int)flx - R; by = (int)fly - R;
                atomicMin(&box[0], bx); atomicMax(&box[1], bx); atomicMin(&box[2], by); atomicMax(&box[3], by);
            } else {                                                // far outside / not finite: the per-pixel kernel takes the tile
                atomicMin(&box[0], -(1 << 24)); atomicMax(&box[1], 1 << 24);
            }
        }
        q_pix[tid] = pix; q_bx[tid] = bx; q_by[tid] = by; q_fx[tid] = fx; q_fy[tid] = fy;
    }
    __syncthreads();
    const int bx0 = box[0], by0 = box[2];
    const int64_t uw64 = (int64_t)box[1] - bx0 + S, uh64 = (int64_t)box[3] - by0 + S;
    // pitch (in positions) of a box row, a multiple of 8: the bank group of a position is then its column mod 8 whatever its
    // row, and the eight pixels of a quarter-warp (one tile row) sit in eight neighbouring columns
    const int64_t pitch64 = (uw64 + 7) / 8 * 8;
    const bool coherent = uw64 > 0 && uh64 > 0 && uw64 <= Cfg::MAXPOS && uh64 <= Cfg::MAXPOS && pitch64 * uh64 <= Cfg::MAXPOS;
    if (!coherent) {
        if (tid == 0) tile_done[tile] = 0;
        return;
    }
    const int uw = (int)uw64, uh = (int)uh64, pitch = (int)pitch64, npos = pitch * uh;
    if (tid < TQ) q_off[tid] = q_pix[tid] >= 0 ? ((q_by[tid] - by0) * pitch + (q_bx[tid] - bx0)) * ROWF : 0;
    for (int pos = tid; pos < npos; pos += NT) {                    // staging plan, the same for every channel chunk
        const int j = pos / pitch, i = pos - j * pitch;
        const int gy = by0 + j, gx = bx0 + i;
        plan[pos] = i >= uw ? -2 : ((gy >= 0 && gy < p.h && gx >= 0 && gx < p.w) ? (int)(((int64_t)gy * p.w + gx) * p.ldf) : -1);
    }
    const int f0_q = tid / C4, f0_piece = tid % C4;
    const bool f0_thread = tid < TQ * C4;
    int f0_src = -1;
    if (f0_thread && q_pix[f0_q] >= 0) f0_src = (int)(((int64_t)q_pix[f0_q] - (int64_t)item * hw) * p.ldf) + f0_piece * 4;
    const uint32_t f1s_u32 = (uint32_t)__cvta_generic_to_shared(f1s), f0s_u32 = (uint32_t)__cvta_generic_to_shared(f0s);
    __syncthreads();                                                // q_off, plan

    auto stage = [&](int k, int buf) {
        const int c0 = k * CK;
        for (int idx = tid; idx < npos * C4; idx += NT) {
            const int pos = idx >> 2, piece = idx & 3;
            const int src = plan[pos];
            if (src != -2)
                cp_async16(f1s_u32 + (uint32_t)(buf * SM::F1_FLOATS + pos * ROWF + piece * 4) * 4u, yimg + (src >= 0 ? src + c0 + piece * 4 : 0), src >= 0 ? 16 : 0);
        }
        if (f0_thread) {
            const bool ok = f0_src >= 0;
            cp_async16(f0s_u32 + (uint32_t)(buf * SM::F0_FLOATS + f0_q * ROWF + f0_piece * 4) * 4u, ximg + (ok ? f0_src + c0 : 0), ok ? 16 : 0);
        }
        cp_async_commit();
    };

    // ---- roles in the compute phase: local correlation = (pixel cq, window row crow): S dot products in registers
    const int cq = tid % TQ, crow = tid / TQ;
    const int my_off = q_off[cq] + crow * pitch * ROWF;
    float acc[S];
#pragma unroll
    for (int n = 0; n < S; ++n) acc[n] = 0.f;
    // x copy and grid_sample(y, flow): pixel gq, 16-byte piece of the chunk
    const int gq = f0_q;
    const bool g_thread = f0_thread && q_pix[gq] >= 0;
    float w00 = 0.f, w01 = 0.f, w10 = 0.f, w11 = 0.f;
    int g_off = 0;
    float* g_drow = nullptr;
    if (g_thread) {
        const float fx = q_fx[gq], fy = q_fy[gq];
        const float ix = ((fx + 1.f) * p.w - 1.f) * 0.5f, iy = ((fy + 1.f) * p.h - 1.f) * 0.5f;
        const float x0f = floorf(ix), y0f = floorf(iy);
        const float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
        w00 = wx0 * wy0; w01 = wx1 * wy0; w10 = wx0 * wy1; w11 = wx1 * wy1;
        g_off = q_off[gq] + (R * pitch + R) * ROWF + f0_piece * 4;      // floor(ix), floor(iy) = window origin + R
        g_drow = (float*)p.d + (int64_t)q_pix[gq] * p.ldd + f0_piece * 4;
    }

    const int nchunks = p.cf / CK;
    stage(0, 0);
    for (int k = 0; k < nchunks; ++k) {
        const int buf = k & 1;
        if (k + 1 < nchunks) { stage(k + 1, buf ^ 1); cp_async_wait<1>(); }
        else cp_async_wait<0>();
        __syncthreads();
        const float* f1b = f1s + buf * SM::F1_FLOATS;
        const float* f0b = f0s + buf * SM::F0_FLOATS;
        {
            const float* base = f1b + my_off;
            // channel quads outermost: the S accumulators are independent chains, so consecutive instructions never wait on each other
#pragma unroll
            for (int c = 0; c < C4; ++c) {
                const float4 a = *reinterpret_cast<const float4*>(f0b + cq * ROWF + c * 4);
#pragma unroll
                for (int n = 0; n < S; ++n) {
                    const float4 b = *reinterpret_cast<const float4*>(base + n * ROWF + c * 4);
                    acc[n] = fmaf(a.x, b.x, acc[n]); acc[n] = fmaf(a.y, b.y, acc[n]); acc[n] = fmaf(a.z, b.z, acc[n]); acc[n] = fmaf(a.w, b.w, acc[n]);
                }
            }
        }
        // x and grid_sample(y, flow) for this chunk of channels (zero-filled positions stand for the zero padding)
        if (g_thread) {
            const int c0 = k * CK;
            *reinterpret_cast<float4*>(g_drow + c0) = *reinterpret_cast<const float4*>(f0b + gq * ROWF + f0_piece * 4);
            const float4 t00 = *reinterpret_cast<const float4*>(f1b + g_off);
            const float4 t01 = *reinterpret_cast<const float4*>(f1b + g_off + ROWF);
            const float4 t10 = *reinterpret_cast<const float4*>(f1b + g_off + pitch * ROWF);
            const float4 t11 = *reinterpret_cast<const float4*>(f1b + g_off + pitch * ROWF + ROWF);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            v.x += t00.x * w00; v.y += t00.y * w00; v.z += t00.z * w00; v.w += t00.w * w00;
            v.x += t01.x * w01; v.y += t01.y * w01; v.z += t01.z * w01; v.w += t01.w * w01;
            v.x += t10.x * w10; v.y += t10.y * w10; v.z += t10.z * w10; v.w += t10.w * w10;
            v.x += t11.x * w11; v.y += t11.y * w11; v.z += t11.z * w11; v.w += t11.w * w11;
            *reinterpret_cast<float4*>(g_drow + p.cf + c0) = v;
        }
        __syncthreads();                                            // the stage is refilled two iterations later
    }

    // ---- D tables -> window samples, displacement embedding
    float* dtab = f1s;                                              // [TQ][S*S + 1]
    const float scale = rsqrtf((float)p.cf);
#pragma unroll
    for (int n = 0; n < S; ++n) dtab[cq * SM::DT_PITCH + crow * S + n] = acc[n] * scale;
    if (tid == 0) tile_done[tile] = 1;
    __syncthreads();
    for (int q = wid; q < TQ; q += NT / 32) {
        const int pix = q_pix[q];
        if (pix < 0) continue;
        const float fx = q_fx[q], fy = q_fy[q];
        float* drow = (float*)p.d + (int64_t)pix * p.ldd;
        const int y = ty0 + q / TQX, x = tx0 + q % TQX;
        const float ddx = p.disp_scale * (fx - p.gx[x]), ddy = p.disp_scale * (fy - p.gy[y]);
        for (int e = lane; e < p.emb; e += 32) drow[2 * p.cf + e] = p.emb_w[2 * e] * ddx + p.emb_w[2 * e + 1] * ddy + p.emb_b[e];
        lc_blend_window<R, float>(dtab + q * SM::DT_PITCH, fx, fy, q_bx[q], q_by[q], p.h, p.w, p.winx, p.winy, drow + 2 * p.cf + p.emb, lane);
    }
}

// fp32 maps with 16-byte aligned rows and cf a multiple of the staged chunk; the caller has checked the rest
int refiner_prologue_tile(const PrologueParams& p, int radius, unsigned char* tile_done, cudaStream_t st) {
    RB_REQUIRE((int64_t)p.D * p.h * p.w < (1ll << 31) && (int64_t)p.h * p.w * p.ldf < (1ll << 31), "refiner_prologue (tile): map too large for 32-bit offsets");
    return with_value<2, 3, 7>(radius, "refiner_prologue (tile): radius", [&](auto r) {
        constexpr int R = decltype(r)::value;
        using SM = LcTileSmem<R>;
        if (ensure_smem<refiner_prologue_tile_kernel<R>>(SM::BYTES, "refiner_prologue (tile)")) return 1;
        const int tiles = p.D * ((p.h + LcTile<R>::TQY - 1) / LcTile<R>::TQY) * ((p.w + LcTile<R>::TQX - 1) / LcTile<R>::TQX);
        rb::launch_pdl(refiner_prologue_tile_kernel<R>, dim3((unsigned)tiles), dim3(SM::THREADS), (size_t)SM::BYTES, st, p, tile_done);
        return check_launch("refiner_prologue_tile");
    });
}

}  // namespace rb
