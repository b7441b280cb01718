// Coarse-to-fine refinement kernels (romatch/models/matcher.py:124-179, 395-527, 839-927;
// romatch/utils/local_correlation.py:77-142; romatch/utils/utils.py:300-322).
//
// Layout: every feature map is channels-last [img, h, w, C] with an explicit pitch; the flow and the
// certainty logit travel together as a 3-channel fp32 "state" map [D, h, w, 3] = (x, y, logit).
// All kernels here are gather / streaming kernels (HBM- or L2-bound); one warp per pixel with lanes over
// channels, so every global access is a contiguous run of the channel vector.
#include "refiner_common.cuh"
#include "tma.cuh"

namespace rb {

// --------------------------------------------------------------------------------------------------
// helpers
// --------------------------------------------------------------------------------------------------
template <typename T> struct Vec16;   // 16-byte vector of T
template <> struct Vec16<float> { static constexpr int N = 4; };
template <> struct Vec16<__half> { static constexpr int N = 8; };
template <> struct Vec16<__nv_bfloat16> { static constexpr int N = 8; };

template <typename T>
__device__ __forceinline__ void load_vec(const T* p, float* out) {
    constexpr int N = Vec16<T>::N;
    uint4 raw = *reinterpret_cast<const uint4*>(p);
    const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
    for (int i = 0; i < N; ++i) out[i] = to_f(e[i]);
}

// sum v[i] over the warp for all 32 i at once: afterwards lane l returns the total of v[l] (31 shuffles)
__device__ __forceinline__ float warp_transpose_reduce(float (&v)[32], int lane) {
#define RB_STAGE(OFF, HALF)                                                    \
    {                                                                          \
        bool up = lane & OFF;                                                  \
        _Pragma("unroll") for (int i = 0; i < HALF; ++i) {                     \
            float send = up ? v[i] : v[i + HALF];                              \
            float keep = up ? v[i + HALF] : v[i];                              \
            v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);             \
        }                                                                      \
    }
    RB_STAGE(16, 16) RB_STAGE(8, 8) RB_STAGE(4, 4) RB_STAGE(2, 2) RB_STAGE(1, 1)
#undef RB_STAGE
    return v[0];
}

// --------------------------------------------------------------------------------------------------
// local correlation for one pixel by one warp.
// D[j][i] = scale * <f0, f1[by+j, bx+i]> on the (2R+2)^2 integer neighbourhood (zero outside the image),
// then every window sample k is the bilinear blend of four D entries with the weights grid_sample would
// use for the coordinate flow + window[k] (all (2R+1)^2 samples sit on a unit pixel lattice, SURVEY §7.2).
// --------------------------------------------------------------------------------------------------
template <typename T, int R, typename TO>
__device__ __forceinline__ void local_corr_warp(const T* __restrict__ f0, const T* __restrict__ f1, int64_t ldf1, float fx, float fy,
                                                int h, int w, int c, float scale, const float* __restrict__ winx,
                                                const float* __restrict__ winy, float* __restrict__ dtab, TO* __restrict__ out, int lane,
                                                const float* __restrict__ table_row = nullptr) {
    constexpr int S = 2 * R + 2, P = S * S;
    constexpr int VN = Vec16<T>::N;
    constexpr int MAXCH = 512 / (32 * VN);      // channel chunks per lane (c <= 512)
    const float cx = ((fx + 1.f) * w - 1.f) * 0.5f, cy = ((fy + 1.f) * h - 1.f) * 0.5f;
    const int bx = (int)floorf(cx) - R, by = (int)floorf(cy) - R;

    if (table_row) {
        // the dot products of this pixel with EVERY position of the other map already exist (one tensor-core GEMM per direction,
        // the same contraction as the all-pairs GP kernel at this scale): D is a gather of (2R+2)^2 table entries
        for (int pl = lane; pl < P; pl += 32) {
            const int jl = pl / S, il = pl - jl * S;
            const int xl = bx + il, yl = by + jl;
            dtab[pl] = (xl >= 0 && xl < w && yl >= 0 && yl < h) ? table_row[yl * w + xl] : 0.f;
        }
        __syncwarp();
        lc_blend_window<R, TO>(dtab, fx, fy, bx, by, h, w, winx, winy, out, lane);
        __syncwarp();
        return;
    }
    float f0r[MAXCH][VN];
#pragma unroll
    for (int t = 0; t < MAXCH; ++t) {
        int c0 = (t * 32 + lane) * VN;
        if (c0 < c) load_vec<T>(f0 + c0, f0r[t]);
        else {
#pragma unroll
            for (int i = 0; i < VN; ++i) f0r[t][i] = 0.f;
        }
    }
    // Per group of 32 window positions the address / validity arithmetic is done ONCE, one position per lane, and
    // handed to the dot-product loop by shuffle and ballot; the loads themselves are unconditional (clamped address,
    // result masked) so that eight positions = up to 16 independent 16-byte loads are in flight per lane.  (ncu on
    // the first version, which branched per position: 16.8k instructions per pixel at R=7, 63 % of them ALU work
    // replicated in all lanes, one L2 round trip per position.)
    constexpr int QB = 8;
    const int nch = (c + 32 * VN - 1) / (32 * VN);            // 16-byte chunks per lane that carry channels (warp-uniform)
    for (int g = 0; g < (P + 31) / 32; ++g) {
        const int pl = g * 32 + lane;
        const int jl = pl / S, il = pl - jl * S;
        const int xl = bx + il, yl = by + jl;
        const bool okl = pl < P && xl >= 0 && xl < w && yl >= 0 && yl < h;
        const int offl = min(max(yl, 0), h - 1) * w + min(max(xl, 0), w - 1);
        const unsigned okmask = __ballot_sync(0xffffffffu, okl);
        float part[32];
#pragma unroll
        for (int qb = 0; qb < 32; qb += QB) {
            if (g * 32 + qb >= P) {                           // warp-uniform: nothing left in this group
#pragma unroll
                for (int q = 0; q < QB; ++q) part[qb + q] = 0.f;
                continue;
            }
            uint4 raw[QB][MAXCH];
#pragma unroll
            for (int q = 0; q < QB; ++q) {
                const int off = __shfl_sync(0xffffffffu, offl, qb + q);
                const T* src = f1 + (int64_t)off * ldf1 + lane * VN;
#pragma unroll
                for (int t = 0; t < MAXCH; ++t) {
                    raw[q][t] = make_uint4(0u, 0u, 0u, 0u);
                    if (t < nch && (t * 32 + lane) * VN < c) raw[q][t] = *reinterpret_cast<const uint4*>(src + t * 32 * VN);
                }
            }
#pragma unroll
            for (int q = 0; q < QB; ++q) {
                float s = 0.f;
#pragma unroll
                for (int t = 0; t < MAXCH; ++t) {
                    if (t < nch) {
                        const T* e = reinterpret_cast<const T*>(&raw[q][t]);
#pragma unroll
                        for (int k = 0; k < VN; ++k) s = fmaf(f0r[t][k], to_f(e[k]), s);
                    }
                }
                part[qb + q] = ((okmask >> (qb + q)) & 1u) ? s : 0.f;
            }
        }
        float tot = warp_transpose_reduce(part, lane);
        if (g * 32 + lane < P) dtab[g * 32 + lane] = tot * scale;
    }
    __syncwarp();
    lc_blend_window<R, TO>(dtab, fx, fy, bx, by, h, w, winx, winy, out, lane);
    __syncwarp();
}

// --------------------------------------------------------------------------------------------------
// ConvRefiner prologue: d = [x | grid_sample(y, flow) | disp_emb | local_corr]   (matcher.py:132-168)
// --------------------------------------------------------------------------------------------------

// thin maps (stride 1: 9 feature channels, 24 in total): one THREAD per pixel, the whole d row is assembled in
// registers and written with 16-byte stores (a warp per pixel would leave 3/4 of the lanes idle on 1.5 M pixels)
template <typename T>
__global__ void __launch_bounds__(256) refiner_prologue_small_kernel(const PrologueParams p) {
    rb::pdl_wait();
    constexpr int MAXC = 32;
    const int64_t pix = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t hw = (int64_t)p.h * p.w;
    if (pix >= p.D * hw) return;
    const int item = (int)(pix / hw);
    const int rem = (int)(pix - item * hw);
    const int y = rem / p.w, x = rem - y * p.w;
    const float fx = p.state[pix * 3 + 0], fy = p.state[pix * 3 + 1];
    const T* feat = (const T*)p.feat;
    const T* xrow = feat + ((int64_t)item * hw + rem) * p.ldf;
    const T* yimg = feat + (int64_t)((item + p.y_shift) % p.n_img) * hw * p.ldf;
    const int cf = p.cf;
    const float ix = ((fx + 1.f) * p.w - 1.f) * 0.5f, iy = ((fy + 1.f) * p.h - 1.f) * 0.5f;
    const float x0f = floorf(ix), y0f = floorf(iy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
    const bool vx0 = x0 >= 0 && x0 < p.w, vx1 = x0 + 1 >= 0 && x0 + 1 < p.w;
    const bool vy0 = y0 >= 0 && y0 < p.h, vy1 = y0 + 1 >= 0 && y0 + 1 < p.h;
    const T* p00 = yimg + ((int64_t)y0 * p.w + x0) * p.ldf;
    const T* p01 = p00 + p.ldf;
    const T* p10 = p00 + (int64_t)p.w * p.ldf;
    const T* p11 = p10 + p.ldf;
    T row[MAXC];
#pragma unroll
    for (int c = 0; c < MAXC; ++c) row[c] = from_f<T>(0.f);
    for (int c = 0; c < cf; ++c) {
        float v = 0.f;
        if (vy0 && vx0) v += to_f(p00[c]) * (wx0 * wy0);
        if (vy0 && vx1) v += to_f(p01[c]) * (wx1 * wy0);
        if (vy1 && vx0) v += to_f(p10[c]) * (wx0 * wy1);
        if (vy1 && vx1) v += to_f(p11[c]) * (wx1 * wy1);
#pragma unroll
        for (int k = 0; k < MAXC; ++k) {          // static indexing keeps `row` in registers
            if (k == c) row[k] = xrow[c];
            if (k == cf + c) row[k] = from_f<T>(v);
        }
    }
    const float ddx = p.disp_scale * (fx - p.gx[x]), ddy = p.disp_scale * (fy - p.gy[y]);
    for (int e = 0; e < p.emb; ++e) {
        const T v = from_f<T>(p.emb_w[2 * e] * ddx + p.emb_w[2 * e + 1] * ddy + p.emb_b[e]);
#pragma unroll
        for (int k = 0; k < MAXC; ++k)
            if (k == 2 * cf + e) row[k] = v;
    }
    T* drow = (T*)p.d + pix * p.ldd;
    constexpr int VN = Vec16<T>::N;
#pragma unroll
    for (int k = 0; k < MAXC; k += VN)
        if (k < p.ldd) *reinterpret_cast<uint4*>(drow + k) = *reinterpret_cast<uint4*>(&row[k]);
}

template <typename T, int R>
__global__ void __launch_bounds__(128) refiner_prologue_kernel(const PrologueParams p) {
    rb::pdl_wait();
    constexpr int S = 2 * R + 2;
    __shared__ float dtab_all[4][R > 0 ? S * S : 1];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t pix = (int64_t)blockIdx.x * 4 + wid;
    const int64_t hw = (int64_t)p.h * p.w;
    if (pix >= p.D * hw) return;
    const int item = (int)(pix / hw);
    const int rem = (int)(pix - item * hw);
    const int y = rem / p.w, x = rem - y * p.w;
    if constexpr (R > 0) {
        if (p.tile_done && p.tile_done[lc_tile_index<R>(item, y, x, p.h, p.w)]) return;     // written by refiner_prologue_tile_kernel
    }
    const float fx = p.state[pix * 3 + 0], fy = p.state[pix * 3 + 1];
    const T* feat = (const T*)p.feat;
    const T* xrow = feat + ((int64_t)item * hw + rem) * p.ldf;
    const T* yimg = feat + (int64_t)((item + p.y_shift) % p.n_img) * hw * p.ldf;
    T* drow = (T*)p.d + pix * p.ldd;
    const int cf = p.cf;

    // grid_sample(y, flow): bilinear, zeros padding, align_corners=False
    const float ix = ((fx + 1.f) * p.w - 1.f) * 0.5f, iy = ((fy + 1.f) * p.h - 1.f) * 0.5f;
    const float x0f = floorf(ix), y0f = floorf(iy);
    const int x0 = (int)x0f, y0 = (int)y0f;
    const float wx1 = ix - x0f, wx0 = (x0f + 1.f) - ix, wy1 = iy - y0f, wy0 = (y0f + 1.f) - iy;
    const bool vx0 = x0 >= 0 && x0 < p.w, vx1 = x0 + 1 >= 0 && x0 + 1 < p.w;
    const bool vy0 = y0 >= 0 && y0 < p.h, vy1 = y0 + 1 >= 0 && y0 + 1 < p.h;
    const T* p00 = yimg + ((int64_t)y0 * p.w + x0) * p.ldf;
    const T* p01 = p00 + p.ldf;
    const T* p10 = p00 + (int64_t)p.w * p.ldf;
    const T* p11 = p10 + p.ldf;
    constexpr int VN = Vec16<T>::N;
    if (cf % VN == 0 && p.vec_ok) {
        // 16-byte channel vectors: copy x, blend the four bilinear corners of y in fp32
        const float w00 = wx0 * wy0, w01 = wx1 * wy0, w10 = wx0 * wy1, w11 = wx1 * wy1;
        for (int c = lane * VN; c < cf; c += 32 * VN) {
            *reinterpret_cast<uint4*>(drow + c) = *reinterpret_cast<const uint4*>(xrow + c);
            float acc[VN], t[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) acc[e] = 0.f;
            if (vy0 && vx0) { load_vec<T>(p00 + c, t);
#pragma unroll
                for (int e = 0; e < VN; ++e) acc[e] += t[e] * w00; }
            if (vy0 && vx1) { load_vec<T>(p01 + c, t);
#pragma unroll
                for (int e = 0; e < VN; ++e) acc[e] += t[e] * w01; }
            if (vy1 && vx0) { load_vec<T>(p10 + c, t);
#pragma unroll
                for (int e = 0; e < VN; ++e) acc[e] += t[e] * w10; }
            if (vy1 && vx1) { load_vec<T>(p11 + c, t);
#pragma unroll
                for (int e = 0; e < VN; ++e) acc[e] += t[e] * w11; }
            T pk[VN];
#pragma unroll
            for (int e = 0; e < VN; ++e) pk[e] = from_f<T>(acc[e]);
            *reinterpret_cast<uint4*>(drow + cf + c) = *reinterpret_cast<uint4*>(pk);
        }
    } else {
        for (int c = lane; c < cf; c += 32) {
            drow[c] = xrow[c];
            float v = 0.f;
            if (vy0 && vx0) v += to_f(p00[c]) * (wx0 * wy0);
            if (vy0 && vx1) v += to_f(p01[c]) * (wx1 * wy0);
            if (vy1 && vx0) v += to_f(p10[c]) * (wx0 * wy1);
            if (vy1 && vx1) v += to_f(p11[c]) * (wx1 * wy1);
            drow[cf + c] = from_f<T>(v);
        }
    }
    // displacement embedding: 1x1 conv 2 -> emb on disp_scale * (flow - identity grid)   (matcher.py:135-148)
    const float ddx = p.disp_scale * (fx - p.gx[x]), ddy = p.disp_scale * (fy - p.gy[y]);
    for (int e = lane; e < p.emb; e += 32)
        drow[2 * cf + e] = from_f<T>(p.emb_w[2 * e] * ddx + p.emb_w[2 * e + 1] * ddy + p.emb_b[e]);
    if constexpr (R > 0)
        local_corr_warp<T, R, T>(xrow, yimg, p.ldf, fx, fy, p.h, p.w, cf, rsqrtf((float)cf), p.winx, p.winy, dtab_all[wid],
                                 drow + 2 * cf + p.emb, lane, p.corr_table ? p.corr_table + pix * p.ld_table : nullptr);
}

// stand-alone local correlation (the reference wheel's operator boundary, local_correlation.py:22-35)
struct LocalCorrParams {
    const void* f0; const void* f1; int64_t ldf0, ldf1, f0_img_stride, f1_img_stride;
    const float* flow; int64_t ldflow; void* out; int64_t ldo;
    int batch, h, w, c; float scale; int n_img, y_shift;
    const float* winx; const float* winy;
};
template <typename T, int R, typename TO>
__global__ void __launch_bounds__(128) local_corr_kernel(const LocalCorrParams p) {
    rb::pdl_wait();
    constexpr int S = 2 * R + 2;
    __shared__ float dtab_all[4][S * S];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t pix = (int64_t)blockIdx.x * 4 + wid;
    const int64_t hw = (int64_t)p.h * p.w;
    if (pix >= p.batch * hw) return;
    const int item = (int)(pix / hw);
    const int rem = (int)(pix - item * hw);
    const float fx = p.flow[pix * p.ldflow + 0], fy = p.flow[pix * p.ldflow + 1];
    const T* f0 = (const T*)p.f0 + item * p.f0_img_stride + (int64_t)rem * p.ldf0;
    const T* f1 = (const T*)p.f1 + (int64_t)((item + p.y_shift) % p.n_img) * p.f1_img_stride;
    local_corr_warp<T, R, TO>(f0, f1, p.ldf1, fx, fy, p.h, p.w, p.c, p.scale, p.winx, p.winy, dtab_all[wid],
                              (TO*)p.out + pix * p.ldo, lane);
}


// --------------------------------------------------------------------------------------------------
// Generic local correlation with the wheel's interface (romab200_local_corr_warp): one warp per (b, p); for every k the
// (up to) four corner rows of f1 are blended lane-wise over the channels and dotted with f0 — any warp, no lattice assumed.
// --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) local_corr_warp_kernel(const float* __restrict__ f0, const float* __restrict__ f1, int64_t ldf0, int64_t ldf1,
                                                              const float* __restrict__ warp, float* __restrict__ out, int B, int H, int W, int C, int K, int mode) {
    rb::pdl_wait();
    const int lane = threadIdx.x & 31;
    const int64_t pix = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int64_t hw = (int64_t)H * W;
    if (pix >= (int64_t)B * hw) return;
    const int b = (int)(pix / hw);
    const float* q = f0 + pix * ldf0;
    const float* img = f1 + (int64_t)b * hw * ldf1;
    for (int k = 0; k < K; ++k) {
        const float gx = warp[(pix * K + k) * 2], gy = warp[(pix * K + k) * 2 + 1];
        const float ix = ((gx + 1.f) * W - 1.f) * 0.5f, iy = ((gy + 1.f) * H - 1.f) * 0.5f;
        int xs[4], ys[4]; float ws[4]; int n = 0;
        if (mode == 1) {                                  // nearest: round half to even like ATen's grid_sampler
            xs[0] = (int)nearbyintf(ix); ys[0] = (int)nearbyintf(iy); ws[0] = 1.f; n = 1;
        } else {
            const float fx0 = floorf(ix), fy0 = floorf(iy);
            const int x0 = (int)fx0, y0 = (int)fy0;
            const float ax = ix - fx0, ay = iy - fy0;
            xs[0] = x0; ys[0] = y0; ws[0] = (1.f - ax) * (1.f - ay);
            xs[1] = x0 + 1; ys[1] = y0; ws[1] = ax * (1.f - ay);
            xs[2] = x0; ys[2] = y0 + 1; ws[2] = (1.f - ax) * ay;
            xs[3] = x0 + 1; ys[3] = y0 + 1; ws[3] = ax * ay;
            n = 4;
        }
        float acc = 0.f;
        for (int c = lane; c < C; c += 32) {
            float v = 0.f;
#pragma unroll
            for (int t = 0; t < 4; ++t)
                if (t < n && xs[t] >= 0 && xs[t] < W && ys[t] >= 0 && ys[t] < H) v = fmaf(ws[t], img[((int64_t)ys[t] * W + xs[t]) * ldf1 + c], v);
            acc = fmaf(q[c], v, acc);
        }
        acc = warp_sum(acc);
        if (lane == 0) out[pix * K + k] = acc;
    }
}

// --------------------------------------------------------------------------------------------------
// depthwise 5x5 + folded BN + ReLU, channels-last.  Block = 8 output rows x 16 output columns x 32 channels;
// the (8+4)x(16+4)x32 input tile is staged in shared memory as fp32; each thread owns one channel of one
// output row and slides along x with the 25 weights in registers (100 LDS + 400 FMA per 16 outputs).
// --------------------------------------------------------------------------------------------------
template <typename T, bool SPLIT = false>
__global__ void __launch_bounds__(256) dwconv5x5_relu_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t ldi, int64_t ldo,
                                                             const float* __restrict__ wgt, int64_t ldw, const float* __restrict__ bias,
                                                             int H, int W, int C, int tiles_x, __half* __restrict__ out_lo = nullptr) {
    rb::pdl_wait();
    constexpr int TH = 8, TW = 16, CH = 32;
    __shared__ float tile[TH + 4][TW + 4][CH];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
    const int c0 = blockIdx.y * CH, b = blockIdx.z;
    const int x0 = tx * TW, y0 = ty * TH;
    const int c = c0 + lane;
    const bool cok = c < C;
    const T* inb = in + (int64_t)b * H * W * ldi;
    for (int pidx = wid; pidx < (TH + 4) * (TW + 4); pidx += 8) {
        int py = pidx / (TW + 4), px = pidx % (TW + 4);
        int yy = y0 + py - 2, xx = x0 + px - 2;
        float v = 0.f;
        if (cok && yy >= 0 && yy < H && xx >= 0 && xx < W) v = to_f(inb[((int64_t)yy * W + xx) * ldi + c]);
        tile[py][px][lane] = v;
    }
    float wr[25];
#pragma unroll
    for (int t = 0; t < 25; ++t) wr[t] = cok ? wgt[(int64_t)t * ldw + c] : 0.f;
    const float bv = cok ? bias[c] : 0.f;
    __syncthreads();
    float acc[TW];
#pragma unroll
    for (int i = 0; i < TW; ++i) acc[i] = bv;
#pragma unroll
    for (int ky = 0; ky < 5; ++ky) {
#pragma unroll
        for (int px = 0; px < TW + 4; ++px) {
            float v = tile[wid + ky][px][lane];
#pragma unroll
            for (int kx = 0; kx < 5; ++kx) {
                int ox = px - kx;
                if (ox >= 0 && ox < TW) acc[ox] = fmaf(wr[ky * 5 + kx], v, acc[ox]);
            }
        }
    }
    const int yy = y0 + wid;
    if (!cok || yy >= H) return;
    if constexpr (SPLIT) {      // fp32 map in, RB_F16S pair out (the A operand of the split-fp16 pointwise GEMM)
        const int64_t o0 = ((int64_t)b * H * W + (int64_t)yy * W) * ldo + c;
        __half* oh = reinterpret_cast<__half*>(out);
#pragma unroll
        for (int i = 0; i < TW; ++i)
            if (x0 + i < W) split_f16s(fmaxf(acc[i], 0.f), oh[o0 + (int64_t)(x0 + i) * ldo], out_lo[o0 + (int64_t)(x0 + i) * ldo]);
    } else {
        T* ob = out + ((int64_t)b * H * W + (int64_t)yy * W) * ldo + c;
#pragma unroll
        for (int i = 0; i < TW; ++i)
            if (x0 + i < W) ob[(int64_t)(x0 + i) * ldo] = from_f<T>(fmaxf(acc[i], 0.f));
    }
}

// (the 16-bit maps take the TMA-fed persistent kernel in dwconv_tma.cu)

// --------------------------------------------------------------------------------------------------
// Fused ConvRefiner block for thin maps (C = 24 at stride 1): depthwise 5x5 + folded BN + ReLU + pointwise
// C x C + bias in ONE pass over the activation (read once, written once).  The stride-1 maps are the
// largest tensors of the path (1.5 M pixels at 864^2) and far too thin for a tensor-core tile, so this is a
// CUDA-core kernel: a 16x16 pixel tile (+2 halo) is staged in shared memory, the depthwise stage runs
// channel-pair x row strips with its 50 filter taps in registers, the pointwise stage runs one pixel per
// thread.  The pointwise weights travel as a KERNEL PARAMETER (2.4 KB): every use is an FFMA with a
// constant-bank operand, so the stage needs no shared-memory traffic and no weight registers.  (ncu on the
// previous version, which broadcast the weights from shared memory with LDS.128: LSU wavefronts at 77 % of
// peak, a third of them bank conflicts of the depthwise reads, FMA pipe 37 % busy.)
// --------------------------------------------------------------------------------------------------
template <int C>
struct SmallPw { float w[C][C]; float b[C]; };        // w[co][ci]

template <typename T, int C>
__global__ void __launch_bounds__(256) refiner_block_small_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t ld,
                                                                  const float* __restrict__ dw_w, int64_t ldw, const float* __restrict__ dw_b,
                                                                  const __grid_constant__ SmallPw<C> pw, int H, int W, int tiles_x) {
    rb::pdl_wait();
    constexpr int TS = 16, IN = TS + 4, CP = C / 2;
    constexpr int PS = C + 2;                 // input pixel stride in halves (odd number of 32-bit words)
    constexpr int RS = IN * PS + 16;          // input row stride in halves: 268 words = 12 mod 32, so the (channel pair, row) lanes
                                              // of a warp, 12 consecutive words per row, fall into 32 distinct banks
    constexpr int MS = C + 1;                 // mid pixel stride in floats
    __shared__ __align__(16) T tile[IN * RS];
    __shared__ float mid[TS * TS * MS];
    const int tid = threadIdx.x;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x, b = blockIdx.y;
    const int x0 = tx * TS, y0 = ty * TS;
    const T* inb = in + (int64_t)b * H * W * ld;
    {   // 16-byte global loads, all issued before the first shared store
        constexpr int VPP = C / 8, NV = IN * IN * VPP, PER = (NV + 255) / 256;
        uint4 vals[PER];
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int i = tid + k * 256;
            const int pix = i / VPP, v = i - pix * VPP;
            const int py = pix / IN, px = pix - py * IN;
            const int yy = y0 + py - 2, xx = x0 + px - 2;
            vals[k] = make_uint4(0u, 0u, 0u, 0u);
            if (i < NV && yy >= 0 && yy < H && xx >= 0 && xx < W)
                vals[k] = *reinterpret_cast<const uint4*>(inb + ((int64_t)yy * W + xx) * ld + 8 * v);
        }
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int i = tid + k * 256;
            if (i < NV) {
                const int pix = i / VPP, v = i - pix * VPP;
                const int py = pix / IN, px = pix - py * IN;
                uint32_t* dst = reinterpret_cast<uint32_t*>(&tile[py * RS + px * PS + 8 * v]);      // pixel stride 52 B: 4-byte aligned
                dst[0] = vals[k].x; dst[1] = vals[k].y; dst[2] = vals[k].z; dst[3] = vals[k].w;
            }
        }
    }
    // ---- depthwise: thread = (channel pair, output row); taps in registers, packed FFMA2
    const int cp = tid % CP, row = tid / CP;
    float2 wv[25];
    float2 bv = make_float2(0.f, 0.f);
    if (row < TS) {
#pragma unroll
        for (int t = 0; t < 25; ++t) wv[t] = make_float2(dw_w[(int64_t)t * ldw + 2 * cp], dw_w[(int64_t)t * ldw + 2 * cp + 1]);
        bv = make_float2(dw_b[2 * cp], dw_b[2 * cp + 1]);
    }
    __syncthreads();
    if (row < TS) {
        float2 acc[TS];
#pragma unroll
        for (int i = 0; i < TS; ++i) acc[i] = bv;
#pragma unroll
        for (int ky = 0; ky < 5; ++ky) {
#pragma unroll
            for (int px = 0; px < IN; ++px) {
                T pr[2];
                *reinterpret_cast<uint32_t*>(pr) = *reinterpret_cast<const uint32_t*>(&tile[(row + ky) * RS + px * PS + 2 * cp]);
                const float2 v = make_float2(to_f(pr[0]), to_f(pr[1]));
#pragma unroll
                for (int kx = 0; kx < 5; ++kx) {
                    const int ox = px - kx;
                    if (ox >= 0 && ox < TS) acc[ox] = rb::fma2(wv[ky * 5 + kx], v, acc[ox]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < TS; ++i) {
            // the unfused path stores this activation in the 16-bit compute dtype: round identically
            mid[(row * TS + i) * MS + 2 * cp] = to_f(from_f<T>(fmaxf(acc[i].x, 0.f)));
            mid[(row * TS + i) * MS + 2 * cp + 1] = to_f(from_f<T>(fmaxf(acc[i].y, 0.f)));
        }
    }
    __syncthreads();
    // ---- pointwise: thread = pixel; weights are constant-bank operands of the FFMAs
    const int py = tid / TS, px = tid - py * TS;
    const int yy = y0 + py, xx = x0 + px;
    if (yy >= H || xx >= W) return;
    float av[C];
#pragma unroll
    for (int ci = 0; ci < C; ++ci) av[ci] = mid[tid * MS + ci];
    T res[C];
#pragma unroll
    for (int co = 0; co < C; ++co) {
        float o = pw.b[co];
#pragma unroll
        for (int ci = 0; ci < C; ++ci) o = fmaf(pw.w[co][ci], av[ci], o);
        res[co] = from_f<T>(o);
    }
    T* op = out + ((int64_t)b * H * W + (int64_t)yy * W + xx) * ld;
#pragma unroll
    for (int v = 0; v < C / 8; ++v) *reinterpret_cast<uint4*>(op + 8 * v) = *reinterpret_cast<const uint4*>(&res[8 * v]);
}


// The same block for fp32 maps (parity mode): fp32 tile in shared memory, fp32 FFMA throughout, fp32 result — the arithmetic of
// the un-fused fp32 path (depthwise kernel + fp32 pointwise GEMM) in one pass over the activation.  Dynamic shared memory:
// input tile 20 rows x 504 words (pixel stride 24, row stride = 24 mod 32 words so that the 64-bit (channel pair, row) reads of a
// half-warp fall into 32 distinct banks) + the 16x16x25 intermediate.
template <int C>
struct SmallF32Cfg {
    static constexpr int TS = 16, IN = TS + 4, PS = C, RS = IN * PS + 24, MS = C + 1;
    static constexpr int SMEM = (IN * RS + TS * TS * MS) * 4;
};

template <int C>
__global__ void __launch_bounds__(256) refiner_block_small_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t ld,
                                                                      const float* __restrict__ dw_w, int64_t ldw, const float* __restrict__ dw_b,
                                                                      const __grid_constant__ SmallPw<C> pw, int H, int W, int tiles_x) {
    rb::pdl_wait();
    using Cfg = SmallF32Cfg<C>;
    constexpr int TS = Cfg::TS, IN = Cfg::IN, CP = C / 2, PS = Cfg::PS, RS = Cfg::RS, MS = Cfg::MS;
    extern __shared__ __align__(16) float sm_small[];
    float* tile = sm_small;                   // [IN][RS]
    float* mid = sm_small + IN * RS;          // [TS*TS][MS]
    const int tid = threadIdx.x;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x, b = blockIdx.y;
    const int x0 = tx * TS, y0 = ty * TS;
    const float* inb = in + (int64_t)b * H * W * ld;
    {   // 16-byte global loads, all issued before the first shared store
        constexpr int VPP = C / 4, NV = IN * IN * VPP, PER = (NV + 255) / 256;
        float4 vals[PER];
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int i = tid + k * 256;
            const int pix = i / VPP, v = i - pix * VPP;
            const int py = pix / IN, px = pix - py * IN;
            const int yy = y0 + py - 2, xx = x0 + px - 2;
            vals[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < NV && yy >= 0 && yy < H && xx >= 0 && xx < W)
                vals[k] = *reinterpret_cast<const float4*>(inb + ((int64_t)yy * W + xx) * ld + 4 * v);
        }
#pragma unroll
        for (int k = 0; k < PER; ++k) {
            const int i = tid + k * 256;
            if (i < NV) {
                const int pix = i / VPP, v = i - pix * VPP;
                const int py = pix / IN, px = pix - py * IN;
                *reinterpret_cast<float4*>(&tile[py * RS + px * PS + 4 * v]) = vals[k];      // RS, PS multiples of 4: 16-byte aligned
            }
        }
    }
    // ---- depthwise: thread = (channel pair, output row); taps in registers, packed FFMA2
    const int cp = tid % CP, row = tid / CP;
    float2 wv[25];
    float2 bv = make_float2(0.f, 0.f);
    if (row < TS) {
#pragma unroll
        for (int t = 0; t < 25; ++t) wv[t] = make_float2(dw_w[(int64_t)t * ldw + 2 * cp], dw_w[(int64_t)t * ldw + 2 * cp + 1]);
        bv = make_float2(dw_b[2 * cp], dw_b[2 * cp + 1]);
    }
    __syncthreads();
    if (row < TS) {
        float2 acc[TS];
#pragma unroll
        for (int i = 0; i < TS; ++i) acc[i] = bv;
#pragma unroll
        for (int ky = 0; ky < 5; ++ky) {
#pragma unroll
            for (int px = 0; px < IN; ++px) {
                const float2 v = *reinterpret_cast<const float2*>(&tile[(row + ky) * RS + px * PS + 2 * cp]);
#pragma unroll
                for (int kx = 0; kx < 5; ++kx) {
                    const int ox = px - kx;
                    if (ox >= 0 && ox < TS) acc[ox] = rb::fma2(wv[ky * 5 + kx], v, acc[ox]);
                }
            }
        }
#pragma unroll
        for (int i = 0; i < TS; ++i) {
            mid[(row * TS + i) * MS + 2 * cp] = fmaxf(acc[i].x, 0.f);
            mid[(row * TS + i) * MS + 2 * cp + 1] = fmaxf(acc[i].y, 0.f);
        }
    }
    __syncthreads();
    // ---- pointwise: thread = pixel; weights are constant-bank operands of the FFMAs
    const int py = tid / TS, px = tid - py * TS;
    const int yy = y0 + py, xx = x0 + px;
    if (yy >= H || xx >= W) return;
    float av[C];
#pragma unroll
    for (int ci = 0; ci < C; ++ci) av[ci] = mid[tid * MS + ci];
    float res[C];
#pragma unroll
    for (int co = 0; co < C; ++co) {
        float o = pw.b[co];
#pragma unroll
        for (int ci = 0; ci < C; ++ci) o = fmaf(pw.w[co][ci], av[ci], o);
        res[co] = o;
    }
    float* op = out + ((int64_t)b * H * W + (int64_t)yy * W + xx) * ld;
#pragma unroll
    for (int v = 0; v < C / 4; ++v) *reinterpret_cast<float4*>(op + 4 * v) = make_float4(res[4 * v], res[4 * v + 1], res[4 * v + 2], res[4 * v + 3]);
}

// --------------------------------------------------------------------------------------------------
// out_conv (C -> 3, fp32) + state update: one warp per pixel
// --------------------------------------------------------------------------------------------------
// LPP lanes cooperate on one pixel (32 for the wide maps, 8 / 4 for the thin ones so that no lane idles on 1.5 M pixels);
// every lane reads 16-byte channel vectors, partial dot products are combined with shuffles inside the lane group.
template <typename T, int LPP>
__global__ void __launch_bounds__(256) refiner_tail_kernel(const T* __restrict__ d, int64_t ldd, const float* __restrict__ wgt, int64_t ldw,
                                                           const float* __restrict__ bias, float* __restrict__ state, int64_t rows, int C,
                                                           float sx, float sy, float* __restrict__ delta_out) {
    rb::pdl_wait();
    constexpr int VN = Vec16<T>::N;
    const int sub = threadIdx.x % LPP;
    const int64_t row = ((int64_t)blockIdx.x * 256 + threadIdx.x) / LPP;
    const bool live = row < rows;
    const int cpad = (C + VN - 1) / VN * VN;              // weights and activations are zero-padded to the vector width
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    if (live) {
        const T* dr = d + row * ldd;
        for (int c = sub * VN; c < cpad; c += LPP * VN) {
            float v[VN];
            load_vec<T>(dr + c, v);
#pragma unroll
            for (int e = 0; e < VN; e += 4) {
                const float4 w0 = *reinterpret_cast<const float4*>(wgt + c + e);
                const float4 w1 = *reinterpret_cast<const float4*>(wgt + ldw + c + e);
                const float4 w2 = *reinterpret_cast<const float4*>(wgt + 2 * ldw + c + e);
                a0 += v[e] * w0.x + v[e + 1] * w0.y + v[e + 2] * w0.z + v[e + 3] * w0.w;
                a1 += v[e] * w1.x + v[e + 1] * w1.y + v[e + 2] * w1.z + v[e + 3] * w1.w;
                a2 += v[e] * w2.x + v[e + 1] * w2.y + v[e + 2] * w2.z + v[e + 3] * w2.w;
            }
        }
    }
#pragma unroll
    for (int o = LPP / 2; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    }
    if (live && sub == 0) {
        a0 += bias[0]; a1 += bias[1]; a2 += bias[2];
        if (delta_out) { delta_out[row * 3 + 0] = a0; delta_out[row * 3 + 1] = a1; delta_out[row * 3 + 2] = a2; }
        state[row * 3 + 0] += sx * a0;
        state[row * 3 + 1] += sy * a1;
        state[row * 3 + 2] += a2;
    }
}

// --------------------------------------------------------------------------------------------------
// bilinear resize (align_corners=False, no antialias) of a small-channel fp32 map
// src index: max(scale*(dst+0.5)-0.5, 0), scale = in/out (ATen area_pixel_compute_source_index)
// --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bilinear_src(int dst, int in_size, int out_size, int& i0, int& i1, float& l1) {
    float scale = (float)in_size / (float)out_size;
    float s = scale * (dst + 0.5f) - 0.5f;
    if (s < 0.f) s = 0.f;
    i0 = (int)s;
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    l1 = s - i0;
}

__global__ void bilinear_resize_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int hi, int wi, int ho, int wo, int C) {
    rb::pdl_wait();
    int64_t total = (int64_t)B * ho * wo * C;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(idx % C); int64_t p = idx / C;
        int xo = (int)(p % wo); int yo = (int)((p / wo) % ho); int b = (int)(p / ((int64_t)wo * ho));
        int y0, y1, x0, x1; float ly, lx;
        bilinear_src(yo, hi, ho, y0, y1, ly);
        bilinear_src(xo, wi, wo, x0, x1, lx);
        const float* s = in + (int64_t)b * hi * wi * C + c;
        float v00 = s[((int64_t)y0 * wi + x0) * C], v01 = s[((int64_t)y0 * wi + x1) * C];
        float v10 = s[((int64_t)y1 * wi + x0) * C], v11 = s[((int64_t)y1 * wi + x1) * C];
        float hy = 1.f - ly, hx = 1.f - lx;
        out[idx] = hy * (hx * v00 + lx * v01) + ly * (hx * v10 + lx * v11);
    }
}

// --------------------------------------------------------------------------------------------------
// cls_to_flow_refine (utils.py:300-322): one block per location
// --------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) cls_to_flow_kernel(const T* __restrict__ logits, float* __restrict__ state, int64_t ldl, int res) {
    rb::pdl_wait();
    __shared__ float smax[8]; __shared__ int sidx[8]; __shared__ float ssum[8];
    const int C = res * res;
    const int64_t row = blockIdx.x;
    const T* l = logits + row * ldl;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    float m = -INFINITY; int mi = 0x7fffffff;
    for (int c = tid; c < C; c += 256) { float v = to_f(l[c]); if (v > m) { m = v; mi = c; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        float om = __shfl_xor_sync(0xffffffffu, m, o); int oi = __shfl_xor_sync(0xffffffffu, mi, o);
        if (om > m || (om == m && oi < mi)) { m = om; mi = oi; }
    }
    if (lane == 0) { smax[wid] = m; sidx[wid] = mi; }
    __syncthreads();
    m = smax[0]; mi = sidx[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) if (smax[i] > m || (smax[i] == m && sidx[i] < mi)) { m = smax[i]; mi = sidx[i]; }
    float s = 0.f;
    for (int c = tid; c < C; c += 256) s += expf(to_f(l[c]) - m);
    s = warp_sum(s);
    if (lane == 0) ssum[wid] = s;
    __syncthreads();
    if (tid == 0) {
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) tot += ssum[i];
        int nb[5] = {mi - 1, mi, mi + 1, mi - res, mi + res};
        float fx = 0.f, fy = 0.f, ps = 0.f;
        const float step = 2.0f / res, first = -1.0f + 1.0f / res;
#pragma unroll
        for (int j = 0; j < 5; ++j) {
            int i = min(max(nb[j], 0), C - 1);
            float pj = expf(to_f(l[i]) - m) / tot;
            // anchor grid: linspace(-1+1/res, 1-1/res, res): x = c % res, y = c / res
            float ax = first + step * (i % res), ay = first + step * (i / res);
            fx += pj * ax; fy += pj * ay; ps += pj;
        }
        state[row * 3 + 0] = fx / ps;
        state[row * 3 + 1] = fy / ps;
        state[row * 3 + 2] = to_f(l[C]);
    }
}

// --------------------------------------------------------------------------------------------------
// match() epilogue (matcher.py:839-850, 891-927)
// --------------------------------------------------------------------------------------------------
__global__ void match_epilogue_kernel(const float* __restrict__ state, const float* __restrict__ coarse, int hc, int wc,
                                      float* __restrict__ warp, float* __restrict__ cert, int b, int H, int W, int symmetric,
                                      const float* __restrict__ gx, const float* __restrict__ gy) {
    rb::pdl_wait();
    const int D = symmetric ? 2 * b : b;
    int64_t total = (int64_t)D * H * W;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int x = (int)(idx % W); int y = (int)((idx / W) % H); int item = (int)(idx / ((int64_t)W * H));
        float fx = state[idx * 3 + 0], fy = state[idx * 3 + 1], logit = state[idx * 3 + 2];
        if (coarse) {
            int y0, y1, x0, x1; float ly, lx;
            bilinear_src(y, hc, H, y0, y1, ly);
            bilinear_src(x, wc, W, x0, x1, lx);
            const float* s = coarse + (int64_t)item * hc * wc * 3 + 2;      // certainty channel of the stride-16 state
            float v00 = s[((int64_t)y0 * wc + x0) * 3], v01 = s[((int64_t)y0 * wc + x1) * 3];
            float v10 = s[((int64_t)y1 * wc + x0) * 3], v11 = s[((int64_t)y1 * wc + x1) * 3];
            float low = (1.f - ly) * ((1.f - lx) * v00 + lx * v01) + ly * ((1.f - lx) * v10 + lx * v11);
            low = 0.5f * low * (low < 0.f ? 1.f : 0.f);
            logit -= low;
        }
        float c = 1.0f / (1.0f + expf(-logit));
        if (fabsf(fx) > 1.f || fabsf(fy) > 1.f) c = 0.f;
        fx = fminf(fmaxf(fx, -1.f), 1.f); fy = fminf(fmaxf(fy, -1.f), 1.f);
        const int Wout = symmetric ? 2 * W : W;
        const bool second = symmetric && item >= b;
        const int ob = second ? item - b : item;
        const int64_t o = ((int64_t)ob * H + y) * Wout + (second ? W + x : x);
        float4 wv = second ? make_float4(fx, fy, gx[x], gy[y]) : make_float4(gx[x], gy[y], fx, fy);
        *reinterpret_cast<float4*>(warp + o * 4) = wv;
        cert[o] = c;
    }
}

}  // namespace rb

using namespace rb;

// ROMAB200_LC_TILE=0 keeps every pixel on the per-pixel kernel (A/B measurements)
static inline bool lc_tile_enabled() { static const bool on = [] { const char* e = getenv("ROMAB200_LC_TILE"); return !e || atoi(e) != 0; }(); return on; }

extern "C" int romab200_refiner_prologue(const rb_refiner_prologue_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->cf > 0 && a->cf <= 512, "refiner_prologue: cf=%d", a->cf);
    RB_REQUIRE(a->ldd >= 2 * a->cf + a->emb + (2 * a->radius + 1) * (2 * a->radius + 1) * (a->radius > 0), "refiner_prologue: ldd too small");
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "refiner_prologue", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int es = sizeof(T);
        if (a->radius > 0) {
            RB_REQUIRE(a->cf % (16 / es) == 0 && a->ldf % (16 / es) == 0 && ((uintptr_t)a->feat) % 16 == 0,
                       "refiner_prologue: local correlation needs 16-byte aligned channel vectors (cf=%d ldf=%lld)", a->cf, (long long)a->ldf);
            RB_REQUIRE(a->win_x && a->win_y, "refiner_prologue: window offsets missing");
        }
        PrologueParams p;
        p.feat = a->feat; p.ldf = a->ldf; p.n_img = a->n_img; p.y_shift = a->y_shift; p.state = a->state; p.d = a->d; p.ldd = a->ldd;
        p.D = a->D; p.h = a->h; p.w = a->w; p.cf = a->cf; p.emb = a->emb; p.emb_w = a->emb_weight; p.emb_b = a->emb_bias;
        p.disp_scale = a->disp_scale; p.gx = a->grid_x; p.gy = a->grid_y; p.winx = a->win_x; p.winy = a->win_y;
        p.vec_ok = (a->ldf * es) % 16 == 0 && (a->ldd * es) % 16 == 0 && ((uintptr_t)a->feat) % 16 == 0 && ((uintptr_t)a->d) % 16 == 0;
        p.tile_done = nullptr;
        p.corr_table = a->corr_table; p.ld_table = a->ld_corr_table;
        RB_REQUIRE(!a->corr_table || (a->radius > 0 && a->ld_corr_table >= (int64_t)a->h * a->w), "refiner_prologue: corr_table needs a local correlation and ld >= h*w");
        int64_t pixels = (int64_t)a->D * a->h * a->w;
        if (a->radius > 0 && std::is_same_v<T, float> && a->tile_done && !a->corr_table && p.vec_ok && a->cf % 16 == 0 && lc_tile_enabled()) {
            const int tqy = a->radius == 7 ? LcTile<7>::TQY : LcTile<3>::TQY, tqx = LcTile<3>::TQX;
            const int64_t tiles = (int64_t)a->D * ((a->h + tqy - 1) / tqy) * ((a->w + tqx - 1) / tqx);
            RB_REQUIRE(a->radius == 2 || a->radius == 3 || a->radius == 7, "refiner_prologue: radius %d unsupported", a->radius);
            RB_REQUIRE(a->tile_done_len >= tiles, "refiner_prologue: tile_done holds %d bytes, %lld tiles", a->tile_done_len, (long long)tiles);
            if (int rc = refiner_prologue_tile(p, a->radius, (unsigned char*)a->tile_done, st)) return rc;
            p.tile_done = (const unsigned char*)a->tile_done;
        }
        if (a->radius == 0 && 2 * a->cf + a->emb <= 32 && a->ldd <= 32 && p.vec_ok) {
            rb::launch_pdl(refiner_prologue_small_kernel<T>, dim3((unsigned)((pixels + 255) / 256)), dim3(256), 0, st, p);      // thin stride-1 maps: one thread per pixel
            return check_launch("refiner_prologue_small");
        }
        return with_value<0, 2, 3, 7>(a->radius, "refiner_prologue: radius", [&](auto r) {
            rb::launch_pdl(refiner_prologue_kernel<T, decltype(r)::value>, dim3((unsigned)((pixels + 3) / 4)), dim3(128), 0, st, p);
            return check_launch("refiner_prologue");
        });
    });
}

extern "C" int romab200_local_corr(const rb_local_corr_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->c > 0 && a->c <= 512, "local_corr: c=%d (max 512)", a->c);
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype_f, "local_corr", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int vn = 16 / sizeof(T);
        RB_REQUIRE(a->c % vn == 0 && a->ldf0 % vn == 0 && a->ldf1 % vn == 0 && a->f0_img_stride % vn == 0 && a->f1_img_stride % vn == 0 &&
                   ((uintptr_t)a->f0) % 16 == 0 && ((uintptr_t)a->f1) % 16 == 0, "local_corr: channel vectors must be 16-byte aligned");
        RB_REQUIRE(a->dtype_out == RB_F32 || a->dtype_out == a->dtype_f, "local_corr: output dtype must be fp32 or the feature dtype");
        LocalCorrParams p;
        p.f0 = a->f0; p.f1 = a->f1; p.ldf0 = a->ldf0; p.ldf1 = a->ldf1; p.f0_img_stride = a->f0_img_stride; p.f1_img_stride = a->f1_img_stride;
        p.flow = a->flow; p.ldflow = a->ldflow; p.out = a->out; p.ldo = a->ldo; p.batch = a->batch; p.h = a->h; p.w = a->w; p.c = a->c;
        p.scale = a->scale; p.n_img = a->n_img > 0 ? a->n_img : a->batch; p.y_shift = a->y_shift; p.winx = a->win_x; p.winy = a->win_y;
        const int64_t pixels = (int64_t)a->batch * a->h * a->w;
        return with_value<2, 3, 7>(a->radius, "local_corr: radius", [&](auto r) {
            constexpr int R = decltype(r)::value;
            rb::launch_pdl(a->dtype_out == RB_F32 ? local_corr_kernel<T, R, float> : local_corr_kernel<T, R, T>, dim3((unsigned)((pixels + 3) / 4)), dim3(128), 0, st, p);
            return check_launch("local_corr");
        });
    });
}

extern "C" int romab200_local_corr_warp(const rb_local_corr_warp_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->f0 && a->f1 && a->warp && a->out && a->batch > 0 && a->h > 0 && a->w > 0 && a->c > 0 && a->k > 0, "local_corr_warp: bad arguments");
    RB_REQUIRE(a->mode == 0 || a->mode == 1, "local_corr_warp: mode must be 0 (bilinear) or 1 (nearest)");
    RB_REQUIRE(a->ldf0 >= a->c && a->ldf1 >= a->c, "local_corr_warp: pitches smaller than the channel count");
    const int64_t pixels = (int64_t)a->batch * a->h * a->w;
    RB_REQUIRE((pixels + 7) / 8 < (1ll << 31), "local_corr_warp: grid too large");
    rb::launch_pdl(local_corr_warp_kernel, dim3((unsigned)((pixels + 7) / 8)), dim3(256), 0, st, a->f0, a->f1, a->ldf0, a->ldf1, a->warp, a->out, a->batch, a->h, a->w,
                   a->c, a->k, a->mode);
    return check_launch("local_corr_warp");
}

extern "C" int romab200_dwconv5x5_relu(const rb_dwconv_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int tiles_x = (a->w + 15) / 16, tiles_y = (a->h + 7) / 8;
    dim3 grid(tiles_x * tiles_y, (a->c + 31) / 32, a->batch);
    RB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "dwconv: grid too large");
    const int cpad = (a->c + 7) & ~7;
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "dwconv5x5_relu", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr bool f32 = std::is_same_v<T, float>;
        if (!f32 && a->ldi % 8 == 0 && a->ldo % 2 == 0 && a->ldi >= cpad && a->ldo >= cpad && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 4 == 0)
            return dwconv_tma(a, st);
        if (f32 && a->out_lo && a->ldi % 4 == 0 && a->ldo % 2 == 0 && a->ldi >= cpad && a->ldo >= cpad &&
            ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 4 == 0 && ((uintptr_t)a->out_lo) % 4 == 0)
            return dwconv_tma(a, st);           // parity mode: fp32 map -> RB_F16S pair, TMA-fed persistent kernel
        RB_REQUIRE(!a->out_lo || f32, "dwconv: the RB_F16S output (out_lo) is for fp32 maps");
        auto kernel = dwconv5x5_relu_kernel<T, false>;
        if constexpr (f32) if (a->out_lo) kernel = dwconv5x5_relu_kernel<float, true>;
        rb::launch_pdl(kernel, grid, dim3(256), 0, st, (const T*)a->in, (T*)a->out, a->ldi, a->ldo, a->weight, a->ldw, a->bias, a->h, a->w, a->c, tiles_x, (__half*)a->out_lo);
        return check_launch("dwconv5x5_relu");
    });
}

extern "C" int romab200_refiner_block_small(const rb_refiner_block_small_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->c == 24, "refiner_block_small: only C = 24 is instantiated (got %d)", a->c);
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "refiner_block_small", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr bool f32 = std::is_same_v<T, float>;
        RB_REQUIRE(a->ld % (16 / sizeof(T)) == 0 && ((uintptr_t)a->in) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0 && a->in != a->out, "refiner_block_small: bad layout");
        int tiles_x = (a->w + 15) / 16, tiles_y = (a->h + 15) / 16;
        dim3 grid(tiles_x * tiles_y, a->batch);
        RB_REQUIRE(grid.y <= 65535, "refiner_block_small: batch too large");
        RB_REQUIRE(a->pw_weight_host && a->pw_bias_host, "refiner_block_small: the pointwise weights must be given as HOST arrays (they are passed as kernel parameters)");
        SmallPw<24> pw;
        for (int co = 0; co < 24; ++co) {
            for (int ci = 0; ci < 24; ++ci) pw.w[co][ci] = a->pw_weight_host[co * 24 + ci];
            pw.b[co] = a->pw_bias_host[co];
        }
        auto kernel = [] { if constexpr (f32) return refiner_block_small_f32_kernel<24>; else return refiner_block_small_kernel<T, 24>; }();
        constexpr int smem = f32 ? SmallF32Cfg<24>::SMEM : 0;      // the fp32 kernel stages its tile in dynamic shared memory
        if constexpr (f32) if (ensure_smem<refiner_block_small_f32_kernel<24>>(smem, "refiner_block_small")) return 1;
        rb::launch_pdl(kernel, grid, dim3(256), smem, st, (const T*)a->in, (T*)a->out, a->ld, a->dw_weight, a->ldw, a->dw_bias, pw, a->h, a->w, tiles_x);
        return check_launch("refiner_block_small");
    });
}

extern "C" int romab200_refiner_tail(const rb_refiner_tail_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "refiner_tail", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int vn = 16 / sizeof(T);
        const int cpad = (a->c + vn - 1) / vn * vn;
        RB_REQUIRE(a->ldd >= cpad && a->ldw >= cpad && a->ldd % vn == 0 && a->ldw % 4 == 0 && ((uintptr_t)a->d) % 16 == 0 &&
                   ((uintptr_t)a->weight) % 16 == 0, "refiner_tail: rows must be zero-padded to whole 16-byte vectors (c=%d ldd=%lld ldw=%lld)",
                   a->c, (long long)a->ldd, (long long)a->ldw);
        const int lpp = a->c <= 32 ? 4 : (a->c <= 256 ? 8 : 32);
        return with_value<4, 8, 32>(lpp, "refiner_tail: lanes per pixel", [&](auto l) {
            rb::launch_pdl(refiner_tail_kernel<T, decltype(l)::value>, dim3((unsigned)((a->rows * lpp + 255) / 256)), dim3(256), 0, st, (const T*)a->d, a->ldd, a->weight,
                           a->ldw, a->bias, a->state, a->rows, a->c, a->scale_x, a->scale_y, a->delta_out);
            return check_launch("refiner_tail");
        });
    });
}

extern "C" int romab200_bilinear_resize(const rb_resize_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int64_t total = (int64_t)a->batch * a->ho * a->wo * a->c;
    RB_REQUIRE(total > 0, "bilinear_resize: empty");
    rb::launch_pdl(bilinear_resize_kernel, dim3(grid1d(total, 256, 132 * 64)), dim3(256), 0, st, a->in, a->out, a->batch, a->hi, a->wi, a->ho, a->wo, a->c);
    return check_launch("bilinear_resize");
}

extern "C" int romab200_cls_to_flow_refine(const rb_cls_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->rows < (1ll << 31) && a->ldl > (int64_t)a->res * a->res, "cls_to_flow_refine: bad shape");
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "cls_to_flow_refine", [&](auto t) {
        using T = typename decltype(t)::type;
        rb::launch_pdl(cls_to_flow_kernel<T>, dim3((unsigned)a->rows), dim3(256), 0, st, (const T*)a->logits, a->state, a->ldl, a->res);
        return check_launch("cls_to_flow_refine");
    });
}

extern "C" int romab200_match_epilogue(const rb_match_epilogue_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int D = a->symmetric ? 2 * a->b : a->b;
    int64_t total = (int64_t)D * a->H * a->W;
    RB_REQUIRE(total > 0 && a->grid_x && a->grid_y, "match_epilogue: bad arguments");
    rb::launch_pdl(match_epilogue_kernel, dim3(grid1d(total, 256, 132 * 64)), dim3(256), 0, st, a->state, a->coarse_state, a->hc, a->wc, a->warp, a->cert, a->b, a->H, a->W,
                                                              a->symmetric, a->grid_x, a->grid_y);
    return check_launch("match_epilogue");
}
