// sample(): Gaussian kernel density of the 4-D match coordinates (romatch/utils/kde.py:4-12) as a tiled
// all-pairs reduction that never materialises the N x N matrix (the reference builds a 40000^2 fp16
// matrix = 3.2 GB).  half != 0 reproduces the reference's fp16 arithmetic step by step (see below); the row
// sum accumulates in fp32 and is rounded to fp16 at the end, as torch's half `sum` does.
#include "common.cuh"

namespace rb {

__device__ __forceinline__ float rh(float v) { return __half2float(__float2half_rn(v)); }

// half mode follows torch.cdist's matmul formulation for fp16 inputs (the path the reference takes):
//   d2 = fp16( fp32-accumulated  [-2x | ||x||^2 | 1] . [y | 1 | ||y||^2] ) clamped at 0,
// then exp(-d2 / (2 std^2)) in fp32, fp32 row sum rounded to fp16 (see the comment in the loop for what is skipped).
// Grid: (row blocks of 256, j-splits).  One thread owns TWO rows (i and i + 128: every staged point is loaded once for both) and
// the j range of its split; with splits > 1 the fp32 partial sums go to workspace[split][n] and kde_finish_kernel adds them in a
// fixed order (deterministic), so that the 40000-point problem of sample() is 1256 CTAs instead of 313 (2.1 per SM: 30 % idle).
// Batched calls put the items on gridDim.z: item z reads x + z * 4n and writes out + z * out_item; each item runs the single-item schedule.
__global__ void __launch_bounds__(128) kde_kernel(const float* __restrict__ x, float* __restrict__ out, int n, float two_var, int half, int j_per_split, int final_half,
                                                  int64_t out_item) {
    rb::pdl_wait();
    x += (int64_t)blockIdx.z * 4 * n;
    out += (int64_t)blockIdx.z * out_item;
    __shared__ float4 pts[512];
    __shared__ float nrm[512];
    const int i0 = blockIdx.x * 256 + threadIdx.x, i1 = i0 + 128;
    float4 xa = make_float4(0.f, 0.f, 0.f, 0.f), xb = xa;
    if (i0 < n) xa = reinterpret_cast<const float4*>(x)[i0];
    if (i1 < n) xb = reinterpret_cast<const float4*>(x)[i1];
    float na = 0.f, nb = 0.f;
    if (half) {
        xa.x = rh(xa.x); xa.y = rh(xa.y); xa.z = rh(xa.z); xa.w = rh(xa.w);
        xb.x = rh(xb.x); xb.y = rh(xb.y); xb.z = rh(xb.z); xb.w = rh(xb.w);
        na = rh(rh(xa.x * xa.x) + rh(xa.y * xa.y) + rh(xa.z * xa.z) + rh(xa.w * xa.w));
        nb = rh(rh(xb.x * xb.x) + rh(xb.y * xb.y) + rh(xb.z * xb.z) + rh(xb.w * xb.w));
    }
    const float ax = -2.f * xa.x, ay = -2.f * xa.y, az = -2.f * xa.z, aw = -2.f * xa.w;
    const float bx = -2.f * xb.x, by = -2.f * xb.y, bz = -2.f * xb.z, bw = -2.f * xb.w;
    float acc_a = 0.f, acc_b = 0.f;
    const int j_begin = blockIdx.y * j_per_split, j_end = min(n, j_begin + j_per_split);
    for (int j0 = j_begin; j0 < j_end; j0 += 512) {
        for (int t = threadIdx.x; t < 512; t += 128) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            float nv = half ? INFINITY : 0.f;
            if (j0 + t < j_end) {
                nv = 0.f;
                v = reinterpret_cast<const float4*>(x)[j0 + t];
                if (half) {
                    v.x = rh(v.x); v.y = rh(v.y); v.z = rh(v.z); v.w = rh(v.w);
                    nv = rh(rh(v.x * v.x) + rh(v.y * v.y) + rh(v.z * v.z) + rh(v.w * v.w));
                }
            }
            pts[t] = v; nrm[t] = nv;
        }
        __syncthreads();
        int lim = min(512, j_end - j0);
        if (half) {
            // fp32 dot product (the matmul), d2 rounded to fp16 and clamped (that quantisation is the one fp16 effect that matters: a
            // d2 ulp moves exp(-50 d2) by up to 10 %), then exp in fp32.  The reference's sqrt -> square round trip (cdist, then **2)
            // and the fp16 rounding of each exp are skipped: together they move a density by at most one fp16 ulp (measured against
            // the oracle: max 1e-3, mean 1e-4 relative) and cost two of the three MUFU operations per pair.
            // padding entries (j >= j_end) hold x = 0, norm = +inf  ->  d2 = inf  ->  exp(-inf) = 0
            const __half2 zero2 = __float2half2_rn(0.f);
            const float nscale = -1.4426950408889634f / two_var;       // exp(-d2 / two_var) = exp2(d2 * nscale)
            float acc_a2 = 0.f, acc_b2 = 0.f;
#pragma unroll 4
            for (int t = 0; t < 512; t += 2) {
                if (t >= lim) break;
                const float4 v0 = pts[t], v1 = pts[t + 1];
                const float n0 = nrm[t], n1 = nrm[t + 1];
                float s0 = ax * v0.x, s1 = ax * v1.x, u0 = bx * v0.x, u1 = bx * v1.x;
                s0 = fmaf(ay, v0.y, s0); s1 = fmaf(ay, v1.y, s1); u0 = fmaf(by, v0.y, u0); u1 = fmaf(by, v1.y, u1);
                s0 = fmaf(az, v0.z, s0); s1 = fmaf(az, v1.z, s1); u0 = fmaf(bz, v0.z, u0); u1 = fmaf(bz, v1.z, u1);
                s0 = fmaf(aw, v0.w, s0); s1 = fmaf(aw, v1.w, s1); u0 = fmaf(bw, v0.w, u0); u1 = fmaf(bw, v1.w, u1);
                s0 = (s0 + na) + n0; s1 = (s1 + na) + n1; u0 = (u0 + nb) + n0; u1 = (u1 + nb) + n1;
                const float2 d2 = __half22float2(__hmax2(__floats2half2_rn(s0, s1), zero2));
                const float2 e2 = __half22float2(__hmax2(__floats2half2_rn(u0, u1), zero2));
                acc_a += exp2f(d2.x * nscale); acc_a2 += exp2f(d2.y * nscale);
                acc_b += exp2f(e2.x * nscale); acc_b2 += exp2f(e2.y * nscale);
            }
            acc_a += acc_a2; acc_b += acc_b2;
        } else {
            for (int t = 0; t < lim; ++t) {
                float4 v = pts[t];
                float dx = xa.x - v.x, dy = xa.y - v.y, dz = xa.z - v.z, dw = xa.w - v.w;
                acc_a += expf(-(dx * dx + dy * dy + dz * dz + dw * dw) / two_var);
                dx = xb.x - v.x; dy = xb.y - v.y; dz = xb.z - v.z; dw = xb.w - v.w;
                acc_b += expf(-(dx * dx + dy * dy + dz * dz + dw * dw) / two_var);
            }
        }
        __syncthreads();
    }
    float* dst = out + (int64_t)blockIdx.y * n;
    if (i0 < n) dst[i0] = final_half ? rh(acc_a) : acc_a;
    if (i1 < n) dst[i1] = final_half ? rh(acc_b) : acc_b;
}

__global__ void __launch_bounds__(256) kde_finish_kernel(const float* __restrict__ partial, float* __restrict__ density, int n, int splits, int half) {
    rb::pdl_wait();
    partial += (int64_t)blockIdx.z * splits * n;
    density += (int64_t)blockIdx.z * n;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += partial[(int64_t)s * n + i];
    density[i] = half ? rh(acc) : acc;
}

// sum v[i] over the warp for all 32 i at once: afterwards lane l holds the total of v[l] (31 shuffles)
__device__ __forceinline__ float kde_transpose_reduce(float (&v)[32], int lane) {
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

// Symmetric schedule of the half mode: exp(-d2(i, j)) = exp(-d2(j, i)) (the fp16-rounded d2 differs between the two orders only when the
// fp32 sum sits within one fp32 ulp of an fp16 rounding boundary: ~1e-4 of the pairs, each worth <= 10 % of one of thousands of terms), so
// only the block pairs (I, J >= I) of 256 x 256 points are evaluated: block I's CTA adds every value to the row sum of i AND, for J > I, to
// the column sum of j.  Column sums: 32 j at a time are summed over the warp's 64 rows with one transpose-reduce (2 instructions per j and
// thread instead of a 10-instruction butterfly), over the four warps through shared memory, and stored per (I, j): the finishing kernel adds
// row partials (per split) and column partials (per I < block(i)) in a fixed order.  Grid (row blocks, splits): split s owns the J blocks
// [s * bps, (s + 1) * bps); it writes zeros when none of them is >= I.  6.75 instead of 12 instructions per credited pair.
__global__ void __launch_bounds__(128) kde_sym_kernel(const float* __restrict__ x, float* __restrict__ ws_row, float* __restrict__ ws_col, int n, float two_var,
                                                      int blocks_per_split, int nblocks, int64_t ws_item) {
    rb::pdl_wait();
    x += (int64_t)blockIdx.z * 4 * n;
    ws_row += (int64_t)blockIdx.z * ws_item;
    ws_col += (int64_t)blockIdx.z * ws_item;
    __shared__ float4 pts[256];
    __shared__ float nrm[256];
    __shared__ float colsum[4][256];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int I = blockIdx.x;
    const int i0 = I * 256 + tid, i1 = i0 + 128;
    float4 xa = make_float4(0.f, 0.f, 0.f, 0.f), xb = xa;
    float na = INFINITY, nb = INFINITY;                    // rows beyond n: d2 = inf -> exp = 0 (they must not reach the column sums)
    if (i0 < n) {
        xa = reinterpret_cast<const float4*>(x)[i0];
        xa.x = rh(xa.x); xa.y = rh(xa.y); xa.z = rh(xa.z); xa.w = rh(xa.w);
        na = rh(rh(xa.x * xa.x) + rh(xa.y * xa.y) + rh(xa.z * xa.z) + rh(xa.w * xa.w));
    }
    if (i1 < n) {
        xb = reinterpret_cast<const float4*>(x)[i1];
        xb.x = rh(xb.x); xb.y = rh(xb.y); xb.z = rh(xb.z); xb.w = rh(xb.w);
        nb = rh(rh(xb.x * xb.x) + rh(xb.y * xb.y) + rh(xb.z * xb.z) + rh(xb.w * xb.w));
    }
    const float ax = -2.f * xa.x, ay = -2.f * xa.y, az = -2.f * xa.z, aw = -2.f * xa.w;
    const float bx = -2.f * xb.x, by = -2.f * xb.y, bz = -2.f * xb.z, bw = -2.f * xb.w;
    const __half2 zero2 = __float2half2_rn(0.f);
    const float nscale = -1.4426950408889634f / two_var;   // exp(-d2 / two_var) = exp2(d2 * nscale)
    float acc_a = 0.f, acc_b = 0.f;
    const int j_first = max(blockIdx.y * blocks_per_split, I), j_last = min(nblocks, (blockIdx.y + 1) * blocks_per_split);
    for (int J = j_first; J < j_last; ++J) {
        for (int t = tid; t < 256; t += 128) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            float nv = INFINITY;                           // padding: d2 = inf -> exp = 0
            const int j = J * 256 + t;
            if (j < n) {
                v = reinterpret_cast<const float4*>(x)[j];
                v.x = rh(v.x); v.y = rh(v.y); v.z = rh(v.z); v.w = rh(v.w);
                nv = rh(rh(v.x * v.x) + rh(v.y * v.y) + rh(v.z * v.z) + rh(v.w * v.w));
            }
            pts[t] = v; nrm[t] = nv;
        }
        __syncthreads();
        const bool offdiag = J > I;                        // CTA-uniform
#pragma unroll 1
        for (int jb = 0; jb < 256; jb += 32) {
            float c[32];
#pragma unroll
            for (int t = 0; t < 32; t += 2) {
                const float4 v0 = pts[jb + t], v1 = pts[jb + t + 1];
                const float n0 = nrm[jb + t], n1 = nrm[jb + t + 1];
                float s0 = ax * v0.x, s1 = ax * v1.x, u0 = bx * v0.x, u1 = bx * v1.x;
                s0 = fmaf(ay, v0.y, s0); s1 = fmaf(ay, v1.y, s1); u0 = fmaf(by, v0.y, u0); u1 = fmaf(by, v1.y, u1);
                s0 = fmaf(az, v0.z, s0); s1 = fmaf(az, v1.z, s1); u0 = fmaf(bz, v0.z, u0); u1 = fmaf(bz, v1.z, u1);
                s0 = fmaf(aw, v0.w, s0); s1 = fmaf(aw, v1.w, s1); u0 = fmaf(bw, v0.w, u0); u1 = fmaf(bw, v1.w, u1);
                s0 = (s0 + na) + n0; s1 = (s1 + na) + n1; u0 = (u0 + nb) + n0; u1 = (u1 + nb) + n1;
                const float2 d2 = __half22float2(__hmax2(__floats2half2_rn(s0, s1), zero2));
                const float2 e2 = __half22float2(__hmax2(__floats2half2_rn(u0, u1), zero2));
                const float ea0 = exp2f(d2.x * nscale), ea1 = exp2f(d2.y * nscale), eb0 = exp2f(e2.x * nscale), eb1 = exp2f(e2.y * nscale);
                acc_a += ea0 + ea1; acc_b += eb0 + eb1;
                c[t] = ea0 + eb0; c[t + 1] = ea1 + eb1;
            }
            if (offdiag) {
                const float tot = kde_transpose_reduce(c, lane);   // lane l: sum over this warp's 64 rows for j = jb + l
                colsum[wid][jb + lane] = tot;
            }
        }
        __syncthreads();
        if (offdiag) {
            for (int t = tid; t < 256; t += 128) {
                const int j = J * 256 + t;
                if (j < n) ws_col[(int64_t)I * n + j] = (colsum[0][t] + colsum[1][t]) + (colsum[2][t] + colsum[3][t]);
            }
        }
        __syncthreads();
    }
    float* dst = ws_row + (int64_t)blockIdx.y * n;
    if (i0 < n) dst[i0] = acc_a;
    if (i1 < n) dst[i1] = acc_b;
}

__global__ void __launch_bounds__(256) kde_sym_finish_kernel(const float* __restrict__ ws_row, const float* __restrict__ ws_col, float* __restrict__ density, int n, int splits,
                                                             int64_t ws_item) {
    rb::pdl_wait();
    ws_row += (int64_t)blockIdx.z * ws_item;
    ws_col += (int64_t)blockIdx.z * ws_item;
    density += (int64_t)blockIdx.z * n;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    float acc = 0.f;
    for (int s = 0; s < splits; ++s) acc += ws_row[(int64_t)s * n + i];
    const int blk = i >> 8;
    for (int I = 0; I < blk; ++I) acc += ws_col[(int64_t)I * n + i];      // every block before mine evaluated my column
    density[i] = rh(acc);
}

}  // namespace rb

extern "C" int romab200_kde_density(const rb_kde_args* a, void* stream) {
    using namespace rb;
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->n > 0 && ((uintptr_t)a->x) % 16 == 0, "kde_density: n=%d or unaligned input", a->n);
    RB_REQUIRE(a->batch >= 0 && a->batch <= 65535, "kde_density: batch %d outside [0, 65535]", a->batch);
    const int batch = a->batch > 0 ? a->batch : 1;
    float two_var = (float)(2.0 * (double)a->std * (double)a->std);
    if (a->symmetric && a->half && a->workspace) {
        // upper-triangle schedule: workspace = (splits + ceil(n / 256)) * n floats
        const int nblocks = (a->n + 255) / 256;
        int splits = a->splits > 1 ? a->splits : 1;
        if (splits > nblocks) splits = nblocks;
        const int bps = (nblocks + splits - 1) / splits;
        splits = (nblocks + bps - 1) / bps;
        const int64_t ws_item = (int64_t)(splits + nblocks) * a->n;
        RB_REQUIRE(a->workspace_floats >= batch * ws_item, "kde_density: the symmetric schedule needs batch * (splits + ceil(n/256)) * n = %lld workspace floats, got %lld",
                   (long long)(batch * ws_item), (long long)a->workspace_floats);
        float* ws_row = a->workspace;
        float* ws_col = a->workspace + (int64_t)splits * a->n;
        rb::launch_pdl(kde_sym_kernel, dim3(nblocks, splits, batch), dim3(128), 0, st, a->x, ws_row, ws_col, a->n, two_var, bps, nblocks, ws_item);
        if (int rc = check_launch("kde_density(sym)")) return rc;
        rb::launch_pdl(kde_sym_finish_kernel, dim3((a->n + 255) / 256, 1, batch), dim3(256), 0, st, (const float*)ws_row, (const float*)ws_col, a->density, a->n,
                       splits, ws_item);
        return check_launch("kde_finish(sym)");
    }
    const int chunks = (a->n + 511) / 512;
    int splits = a->workspace && a->splits > 1 ? a->splits : 1;
    if (splits > chunks) splits = chunks;
    const int per = (chunks + splits - 1) / splits * 512;
    splits = (a->n + per - 1) / per;                                 // no empty split
    const dim3 grid((a->n + 255) / 256, splits, batch);
    if (splits == 1) {
        rb::launch_pdl(kde_kernel, grid, dim3(128), 0, st, a->x, a->density, a->n, two_var, a->half, per, a->half, (int64_t)a->n);
        return check_launch("kde_density");
    }
    RB_REQUIRE(batch == 1 || a->workspace_floats >= (int64_t)batch * splits * a->n, "kde_density: %d items of %d splits need %lld workspace floats, got %lld", batch,
               splits, (long long)batch * splits * a->n, (long long)a->workspace_floats);
    rb::launch_pdl(kde_kernel, grid, dim3(128), 0, st, a->x, a->workspace, a->n, two_var, a->half, per, 0, (int64_t)splits * a->n);
    if (int rc = check_launch("kde_density")) return rc;
    rb::launch_pdl(kde_finish_kernel, dim3((a->n + 255) / 256, 1, batch), dim3(256), 0, st, (const float*)a->workspace, a->density, a->n, splits, a->half);
    return check_launch("kde_finish");
}
