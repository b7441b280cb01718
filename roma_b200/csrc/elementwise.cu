// Row-wise / element-wise kernels: LayerNorm, softmax, row norms, casts, fp16 hi/lo split,
// DINOv2 tokenisation, batched transpose.  All HBM-bound; one warp (or block) per row, 16-byte
// vector accesses where the pitch allows.
#include "common.cuh"

namespace rb {

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, two-pass (mean, then centred variance) in fp32 like ATen's CPU kernel.
// ------------------------------------------------------------------------------------------------
template <typename TI, typename TO>
__global__ void layernorm_kernel(const TI* __restrict__ x, TO* __restrict__ y, const float* __restrict__ g,
                                 const float* __restrict__ b, int64_t rows, int cols, int64_t ldx, int64_t ldy, float eps) {
    rb::pdl_wait();
    int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    int lane = threadIdx.x & 31;
    const TI* xr = x + row * ldx;
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s += to_f(xr[c]);
    float mean = warp_sum(s) / cols;
    float v = 0.f;
    for (int c = lane; c < cols; c += 32) { float d = to_f(xr[c]) - mean; v += d * d; }
    float rstd = rsqrtf(warp_sum(v) / cols + eps);
    TO* yr = y + row * ldy;
    for (int c = lane; c < cols; c += 32) yr[c] = from_f<TO>((to_f(xr[c]) - mean) * rstd * g[c] + b[c]);
}

// the same with an RB_F16S (split fp16 pair) result
__global__ void layernorm_split_kernel(const float* __restrict__ x, __half* __restrict__ yh, __half* __restrict__ yl, const float* __restrict__ g,
                                       const float* __restrict__ b, int64_t rows, int cols, int64_t ldx, int64_t ldy, float eps) {
    rb::pdl_wait();
    int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    int lane = threadIdx.x & 31;
    const float* xr = x + row * ldx;
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s += xr[c];
    float mean = warp_sum(s) / cols;
    float v = 0.f;
    for (int c = lane; c < cols; c += 32) { float d = xr[c] - mean; v += d * d; }
    float rstd = rsqrtf(warp_sum(v) / cols + eps);
    for (int c = lane; c < cols; c += 32) split_f16s((xr[c] - mean) * rstd * g[c] + b[c], yh[row * ldy + c], yl[row * ldy + c]);
}

// Row-in-registers variant for fp32 rows of NV * 128 columns (the ViT and decoder width 1024: NV = 8): the row is read
// once with 16-byte loads (the generic kernel reads it three times with 4-byte loads and ran at a third of the HBM
// rate), mean and centred variance are formed from the registers, the result is written with 8/16-byte stores.
template <typename TO, int NV, bool SPLIT = false>
__global__ void __launch_bounds__(128) layernorm_vec_kernel(const float* __restrict__ x, TO* __restrict__ y, const float* __restrict__ g,
                                                            const float* __restrict__ b, int64_t rows, int64_t ldx, int64_t ldy, float eps,
                                                            TO* __restrict__ y_lo = nullptr) {
    rb::pdl_wait();
    const int64_t row = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int lane = threadIdx.x & 31;
    constexpr int cols = NV * 128;
    const float4* xr = reinterpret_cast<const float4*>(x + row * ldx);
    float4 v[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) v[k] = xr[k * 32 + lane];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) s += (v[k].x + v[k].y) + (v[k].z + v[k].w);
    const float mean = warp_sum(s) / cols;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        v[k].x -= mean; v[k].y -= mean; v[k].z -= mean; v[k].w -= mean;
        q += (v[k].x * v[k].x + v[k].y * v[k].y) + (v[k].z * v[k].z + v[k].w * v[k].w);
    }
    const float rstd = rsqrtf(warp_sum(q) / cols + eps);
    TO* yr = y + row * ldy;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
        const int c = (k * 32 + lane) * 4;
        const float4 gg = *reinterpret_cast<const float4*>(g + c), bb = *reinterpret_cast<const float4*>(b + c);
        const float o0 = v[k].x * rstd * gg.x + bb.x, o1 = v[k].y * rstd * gg.y + bb.y, o2 = v[k].z * rstd * gg.z + bb.z, o3 = v[k].w * rstd * gg.w + bb.w;
        if constexpr (SPLIT) {
            __half hi[4], lo[4];
            split_f16s(o0, hi[0], lo[0]); split_f16s(o1, hi[1], lo[1]); split_f16s(o2, hi[2], lo[2]); split_f16s(o3, hi[3], lo[3]);
            *reinterpret_cast<uint2*>(yr + c) = *reinterpret_cast<uint2*>(hi);
            *reinterpret_cast<uint2*>(y_lo + row * ldy + c) = *reinterpret_cast<uint2*>(lo);
        } else if constexpr (sizeof(TO) == 4) {
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(yr) + c) = make_float4(o0, o1, o2, o3);
        } else {
            TO pk[4] = {from_f<TO>(o0), from_f<TO>(o1), from_f<TO>(o2), from_f<TO>(o3)};
            *reinterpret_cast<uint2*>(yr + c) = *reinterpret_cast<uint2*>(pk);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// softmax over rows (attention scores), in place: one block of 256 threads per row.  With `oh` (fp32 scores only) the result
// goes to an RB_F16S pair [rows, ldo] instead, for rows too long for softmax_rows_split_kernel.
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void softmax_rows_kernel(T* __restrict__ s, int64_t rows, int cols, int64_t lds, float scale, __half* __restrict__ oh,
                                    __half* __restrict__ ol, int64_t ldo) {
    rb::pdl_wait();
    __shared__ float red[8];
    int64_t row = blockIdx.x;
    T* sr = s + row * lds;
    int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    float m = -INFINITY;
    for (int c = tid; c < cols; c += 256) m = fmaxf(m, to_f(sr[c]) * scale);
    m = warp_max(m);
    if (lane == 0) red[wid] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) m = fmaxf(m, red[i]);
    __syncthreads();
    float sum = 0.f;
    for (int c = tid; c < cols; c += 256) sum += expf(to_f(sr[c]) * scale - m);
    sum = warp_sum(sum);
    if (lane == 0) red[wid] = sum;
    __syncthreads();
    sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sum += red[i];
    float inv = 1.0f / sum;
    if (oh) {
        // the pad columns of the last 4-element group receive 0, as from the warp kernel
        for (int c = tid; c < (cols + 3) / 4 * 4; c += 256)
            split_f16s(c < cols ? expf(to_f(sr[c]) * scale - m) * inv : 0.f, oh[row * ldo + c], ol[row * ldo + c]);
        return;
    }
    for (int c = tid; c < cols; c += 256) sr[c] = from_f<T>(expf(to_f(sr[c]) * scale - m) * inv);
}

// warp-per-row softmax for rows of at most 2048 elements (attention: 1600/1601): the row is read once with
// 16-byte loads, kept in registers, and written once.
template <typename T>
__global__ void __launch_bounds__(256) softmax_rows_warp_kernel(T* __restrict__ s, int64_t rows, int cols, int64_t lds, float scale) {
    rb::pdl_wait();
    constexpr int VN = 16 / sizeof(T);
    constexpr int ITERS = 2048 / (32 * VN);
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    T* sr = s + row * lds;
    float v[ITERS][VN];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
        const int c0 = (i * 32 + lane) * VN;
        if (c0 < cols) {
            uint4 raw = *reinterpret_cast<const uint4*>(sr + c0);
            const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
            for (int j = 0; j < VN; ++j) {
                v[i][j] = (c0 + j < cols) ? to_f(e[j]) * scale : -INFINITY;
                m = fmaxf(m, v[i][j]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < VN; ++j) v[i][j] = -INFINITY;
        }
    }
    m = warp_max(m);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; ++i)
#pragma unroll
        for (int j = 0; j < VN; ++j) { v[i][j] = expf(v[i][j] - m); sum += v[i][j]; }
    const float inv = 1.0f / warp_sum(sum);
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
        const int c0 = (i * 32 + lane) * VN;
        if (c0 < cols) {
            uint4 raw;
            T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
            for (int j = 0; j < VN; ++j) e[j] = from_f<T>(v[i][j] * inv);      // pad columns (>= cols) receive 0
            *reinterpret_cast<uint4*>(sr + c0) = raw;
        }
    }
}

// fp32 scores -> softmax written as an RB_F16S pair (the A operand of the split-fp16 PV product); not in place
__global__ void __launch_bounds__(256) softmax_rows_split_kernel(const float* __restrict__ s, __half* __restrict__ oh, __half* __restrict__ ol,
                                                                 int64_t rows, int cols, int64_t lds, int64_t ldo, float scale) {
    rb::pdl_wait();
    constexpr int VN = 4, ITERS = 2048 / (32 * VN);
    const int lane = threadIdx.x & 31;
    const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float* sr = s + row * lds;
    float v[ITERS][VN];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
        const int c0 = (i * 32 + lane) * VN;
        if (c0 < cols) {
            const float4 raw = *reinterpret_cast<const float4*>(sr + c0);
            const float e[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
            for (int j = 0; j < VN; ++j) {
                v[i][j] = (c0 + j < cols) ? e[j] * scale : -INFINITY;
                m = fmaxf(m, v[i][j]);
            }
        } else {
#pragma unroll
            for (int j = 0; j < VN; ++j) v[i][j] = -INFINITY;
        }
    }
    m = warp_max(m);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < ITERS; ++i)
#pragma unroll
        for (int j = 0; j < VN; ++j) { v[i][j] = expf(v[i][j] - m); sum += v[i][j]; }
    const float inv = 1.0f / warp_sum(sum);
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
        const int c0 = (i * 32 + lane) * VN;
        if (c0 < cols) {
            __half hi[4], lo[4];
#pragma unroll
            for (int j = 0; j < VN; ++j) split_f16s(v[i][j] * inv, hi[j], lo[j]);          // pad columns (>= cols) receive 0
            *reinterpret_cast<uint2*>(oh + row * ldo + c0) = *reinterpret_cast<uint2*>(hi);
            *reinterpret_cast<uint2*>(ol + row * ldo + c0) = *reinterpret_cast<uint2*>(lo);
        }
    }
}

template <typename T>
__global__ void row_norms_kernel(const T* __restrict__ x, float* __restrict__ out, int64_t rows, int cols, int64_t ldx) {
    rb::pdl_wait();
    int64_t row = (int64_t)blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (row >= rows) return;
    int lane = threadIdx.x & 31;
    const T* xr = x + row * ldx;
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) { float v = to_f(xr[c]); s += v * v; }
    s = warp_sum(s);
    if (lane == 0) out[row] = sqrtf(s);
}

__global__ void copy2d_kernel(const void* __restrict__ src, void* __restrict__ dst, int64_t rows, int cols, int64_t lds,
                              int64_t ldd, int ds, int dd, const float* __restrict__ row_scale, int recip) {
    rb::pdl_wait();
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t total = rows * cols;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx / cols; int c = (int)(idx - r * cols);
        float v = load_any(src, r * lds + c, ds);
        if (row_scale) v = recip ? v / row_scale[r] : v * row_scale[r];
        store_any(dst, r * ldd + c, dd, v);
    }
}

// dst row dst_index[i] = src row src_index[i] (NULL: i), blockIdx.y = i; 16-byte words, grid-stride along the row
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const int32_t* __restrict__ src_index,
                                                          const int32_t* __restrict__ dst_index, int64_t words, int64_t ld_src, int64_t ld_dst,
                                                          int src_rows, int dst_rows) {
    rb::pdl_wait();
    const int i = blockIdx.y;
    const int s = src_index ? src_index[i] : i, d = dst_index ? dst_index[i] : i;
    if (s < 0 || s >= src_rows || d < 0 || d >= dst_rows) return;
    const uint4* sr = src + (int64_t)s * ld_src;
    uint4* dr = dst + (int64_t)d * ld_dst;
    for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < words; k += (int64_t)gridDim.x * blockDim.x) dr[k] = sr[k];
}

// x / norm -> fp16 hi and lo parts laid out [hi|lo|hi] (A operand) or [hi|hi|lo] (B operand)
__global__ void split_f16x3_kernel(const float* __restrict__ x, __half* __restrict__ dst, int64_t rows, int cols,
                                   int64_t ldx, int64_t ldd, const float* __restrict__ norm, int layout_b) {
    rb::pdl_wait();
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int64_t total = rows * cols;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int64_t r = idx / cols; int c = (int)(idx - r * cols);
        float v = x[r * ldx + c];
        if (norm) v = v / norm[r];
        __half hi = __float2half_rn(v);
        __half lo = __float2half_rn(v - __half2float(hi));
        __half* d = dst + r * ldd;
        d[c] = hi;
        d[cols + c] = layout_b ? hi : lo;
        d[2 * cols + c] = layout_b ? lo : hi;
    }
}

// fp32 -> RB_F16S planes, 4 elements per thread (16-byte load, two 8-byte stores); pitches are multiples of 4 elements
__global__ void __launch_bounds__(256) split_f16s_vec_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo,
                                                             int64_t rows, int cols4, int cols, int64_t ldx, int64_t ldd,
                                                             const float* __restrict__ norm) {
    rb::pdl_wait();
    const int64_t total = rows * cols4;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / cols4; const int c = (int)(idx - r * cols4) * 4;
        float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
        if (norm) { const float n = norm[r]; v.x /= n; v.y /= n; v.z /= n; v.w /= n; }
        // the pitch pads beyond `cols` (at most 3 elements here) are written too: the GEMM never reads past K (TMA zero fill)
        __half h[4], l[4];
        split_f16s(v.x, h[0], l[0]); split_f16s(v.y, h[1], l[1]); split_f16s(v.z, h[2], l[2]); split_f16s(v.w, h[3], l[3]);
        *reinterpret_cast<uint2*>(hi + r * ldd + c) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(lo + r * ldd + c) = *reinterpret_cast<uint2*>(l);
    }
}
// batched variant (blockIdx.y = matrix): used by the tensor-core GP solve for its strided panels.  Columns [0, cols) only: a last
// group of fewer than 4 columns (the GP's last diagonal block at n % 4 != 0) is read and written element by element, so that
// nothing beyond `cols` is read (the source pad may hold anything) or written.
__global__ void __launch_bounds__(256) split_f16s_batched_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int64_t rows, int cols4,
                                                                 int cols, int64_t ldx, int64_t ldd, int64_t sx, int64_t sd) {
    rb::pdl_wait();
    x += blockIdx.y * sx; hi += blockIdx.y * sd; lo += blockIdx.y * sd;
    const int64_t total = rows * cols4;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / cols4; const int c = (int)(idx - r * cols4) * 4;
        if (c + 4 > cols) {
            for (int j = c; j < cols; ++j) split_f16s(x[r * ldx + j], hi[r * ldd + j], lo[r * ldd + j]);
            continue;
        }
        const float4 v = *reinterpret_cast<const float4*>(x + r * ldx + c);
        __half h[4], l[4];
        split_f16s(v.x, h[0], l[0]); split_f16s(v.y, h[1], l[1]); split_f16s(v.z, h[2], l[2]); split_f16s(v.w, h[3], l[3]);
        *reinterpret_cast<uint2*>(hi + r * ldd + c) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(lo + r * ldd + c) = *reinterpret_cast<uint2*>(l);
    }
}

__global__ void split_f16s_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int64_t rows, int cols,
                                  int64_t ldx, int64_t ldd, const float* __restrict__ norm) {
    rb::pdl_wait();
    const int64_t total = rows * cols;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = idx / cols; const int c = (int)(idx - r * cols);
        float v = x[r * ldx + c];
        if (norm) v = v / norm[r];
        split_f16s(v, hi[r * ldd + c], lo[r * ldd + c]);
    }
}

// im2col of PxP non-overlapping patches: out[(b*hp+py)*wp+px][c*P*P + ky*P + kx] = img[b][c][py*P+ky][px*P+kx]
// (same (c,ky,kx) order as Conv2d weight.flatten(1), patch_embed.py:69-82)
template <typename TO>
__global__ void im2col_patch_kernel(const float* __restrict__ img, TO* __restrict__ out, int B, int H, int W, int P, int64_t ldo) {
    rb::pdl_wait();
    int hp = H / P, wp = W / P, kk = 3 * P * P;
    int64_t total = (int64_t)B * hp * wp * kk;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int k = (int)(idx % kk); int64_t row = idx / kk;
        int px = (int)(row % wp); int py = (int)((row / wp) % hp); int b = (int)(row / ((int64_t)wp * hp));
        int c = k / (P * P), r = k % (P * P), ky = r / P, kx = r % P;
        float v = img[(((int64_t)b * 3 + c) * H + (py * P + ky)) * W + (px * P + kx)];
        out[row * ldo + k] = from_f<TO>(v);
    }
}

__global__ void assemble_tokens_kernel(const float* __restrict__ patch, const float* __restrict__ cls,
                                       const float* __restrict__ pos, float* __restrict__ tok, int B, int np, int dim) {
    rb::pdl_wait();
    int64_t total = (int64_t)B * (np + 1) * dim;
    int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(idx % dim); int64_t r = idx / dim;
        int t = (int)(r % (np + 1)); int b = (int)(r / (np + 1));
        float v = t == 0 ? cls[c] : patch[((int64_t)b * np + (t - 1)) * dim + c];
        tok[idx] = v + pos[(int64_t)t * dim + c];
    }
}

// batched transpose through a 32x33 shared tile
template <typename T>
__global__ void transpose_kernel(const T* __restrict__ src, T* __restrict__ dst, int rows, int cols, int64_t lds, int64_t ldd,
                                 int batch1, int64_t ss0, int64_t ss1, int64_t sd0, int64_t sd1) {
    rb::pdl_wait();
    __shared__ T tile[32][33];
    int z = blockIdx.z, z0 = z / batch1, z1 = z % batch1;
    const T* s = src + z0 * ss0 + z1 * ss1;
    T* d = dst + z0 * sd0 + z1 * sd1;
    int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int r = r0 + i, c = c0 + threadIdx.x;
        if (r < rows && c < cols) tile[i][threadIdx.x] = s[(int64_t)r * lds + c];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        int c = c0 + i, r = r0 + threadIdx.x;
        if (r < rows && c < cols) d[(int64_t)c * ldd + r] = tile[threadIdx.x][i];
    }
}

// fp32 [batch][rows, cols] (pitch ldx, matrix stride sx) -> RB_F16S planes [batch][rows, ldd] (matrix stride sd); 16-byte aligned rows
int split_f16s_batched(const float* x, void* hi, void* lo, int64_t rows, int cols, int64_t ldx, int64_t ldd, int batch, int64_t sx, int64_t sd, cudaStream_t st) {
    RB_REQUIRE(ldx % 4 == 0 && ldd % 4 == 0 && sx % 4 == 0 && sd % 4 == 0 && ((uintptr_t)x) % 16 == 0 && ((uintptr_t)hi) % 8 == 0 && ((uintptr_t)lo) % 8 == 0,
               "split_f16s_batched: alignment");
    RB_REQUIRE(batch > 0 && batch <= 65535 && rows > 0 && cols > 0 && cols <= ldx && cols <= ldd, "split_f16s_batched: bad shape");
    const int cols4 = (cols + 3) / 4;
    dim3 grid(grid1d(rows * cols4, 256, 132 * 8), batch);
    rb::launch_pdl(split_f16s_batched_kernel, grid, dim3(256), 0, st, x, (__half*)hi, (__half*)lo, rows, cols4, cols, ldx, ldd, sx, sd);
    return check_launch("split_f16s_batched");
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_layernorm(const rb_layernorm_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->cols > 0, "layernorm: empty input");
    RB_REQUIRE(a->dtype_y != RB_F16S || (a->y_lo && a->dtype_x == RB_F32), "layernorm: RB_F16S output needs y_lo and fp32 input");
    if (a->dtype_y == RB_F16S && !(a->cols == 1024 && a->ldx % 4 == 0 && a->ldy % 4 == 0 && ((uintptr_t)a->x) % 16 == 0 &&
                                   ((uintptr_t)a->y) % 8 == 0 && ((uintptr_t)a->y_lo) % 8 == 0 && ((uintptr_t)a->gamma) % 16 == 0 && ((uintptr_t)a->beta) % 16 == 0)) {
        dim3 grid((unsigned)((a->rows + 7) / 8));
        rb::launch_pdl(layernorm_split_kernel, grid, dim3(256), 0, st, (const float*)a->x, (__half*)a->y, (__half*)a->y_lo, a->gamma, a->beta, a->rows, a->cols, a->ldx, a->ldy, a->eps);
        return check_launch("layernorm");
    }
    if (a->dtype_y == RB_F16S) {
        dim3 gridv((unsigned)((a->rows + 3) / 4));
        rb::launch_pdl(layernorm_vec_kernel<__half, 8, true>, gridv, dim3(128), 0, st, (const float*)a->x, (__half*)a->y, a->gamma, a->beta, a->rows, a->ldx, a->ldy, a->eps, (__half*)a->y_lo);
        return check_launch("layernorm");
    }
    if (check_dtype<float>(a->dtype_x, "layernorm")) return 1;
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype_y, "layernorm", [&](auto t) {
        using TO = typename decltype(t)::type;
        if (a->cols == 1024 && a->ldx % 4 == 0 && (a->ldy * (int)sizeof(TO)) % 16 == 0 && ((uintptr_t)a->x) % 16 == 0 &&
            ((uintptr_t)a->y) % 16 == 0 && ((uintptr_t)a->gamma) % 16 == 0 && ((uintptr_t)a->beta) % 16 == 0)
            rb::launch_pdl(layernorm_vec_kernel<TO, 8, false>, dim3((unsigned)((a->rows + 3) / 4)), dim3(128), 0, st, (const float*)a->x, (TO*)a->y, a->gamma, a->beta,
                           a->rows, a->ldx, a->ldy, a->eps, (TO*)nullptr);
        else
            rb::launch_pdl(layernorm_kernel<float, TO>, dim3((unsigned)((a->rows + 7) / 8)), dim3(256), 0, st, (const float*)a->x, (TO*)a->y, a->gamma, a->beta,
                           a->rows, a->cols, a->ldx, a->ldy, a->eps);
        return check_launch("layernorm");
    });
}

extern "C" int romab200_softmax_rows(const rb_softmax_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->cols > 0 && a->rows < (1ll << 31), "softmax: bad shape");
    if (a->out_hi) {
        RB_REQUIRE(a->dtype == RB_F32 && a->out_lo && a->lds % 4 == 0 && a->ldo % 4 == 0 && (a->cols + 3) / 4 * 4 <= a->ldo &&
                   (a->cols + 3) / 4 * 4 <= a->lds && ((uintptr_t)a->s) % 16 == 0 && ((uintptr_t)a->out_hi) % 8 == 0 && ((uintptr_t)a->out_lo) % 8 == 0,
                   "softmax: split output needs fp32 scores and 4-element aligned pitches");
        if (a->cols <= 2048)
            rb::launch_pdl(softmax_rows_split_kernel, dim3((unsigned)((a->rows + 7) / 8)), dim3(256), 0, st, (const float*)a->s, (__half*)a->out_hi, (__half*)a->out_lo,
                           a->rows, a->cols, a->lds, a->ldo, a->scale);
        else
            rb::launch_pdl(softmax_rows_kernel<float>, dim3((unsigned)a->rows), dim3(256), 0, st, (float*)a->s, a->rows, a->cols, a->lds, a->scale,
                           (__half*)a->out_hi, (__half*)a->out_lo, a->ldo);
        return check_launch("softmax_rows");
    }
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "softmax_rows", [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int vn = 16 / sizeof(T);
        // warp per row when the rows are padded to whole 16-byte vectors (the pad columns are rewritten with zeros), else block per row
        const bool warp = a->cols <= 2048 && (a->lds * (int)sizeof(T)) % 16 == 0 && ((uintptr_t)a->s) % 16 == 0 && (a->cols + vn - 1) / vn * vn <= a->lds;
        if (warp)
            rb::launch_pdl(softmax_rows_warp_kernel<T>, dim3((unsigned)((a->rows + 7) / 8)), dim3(256), 0, st, (T*)a->s, a->rows, a->cols, a->lds, a->scale);
        else
            rb::launch_pdl(softmax_rows_kernel<T>, dim3((unsigned)a->rows), dim3(256), 0, st, (T*)a->s, a->rows, a->cols, a->lds, a->scale,
                           (__half*)nullptr, (__half*)nullptr, (int64_t)0);
        return check_launch("softmax_rows");
    });
}

extern "C" int romab200_row_norms(const rb_rownorm_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->cols > 0, "row_norms: empty input");
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "row_norms", [&](auto t) {
        using T = typename decltype(t)::type;
        rb::launch_pdl(row_norms_kernel<T>, dim3((unsigned)((a->rows + 7) / 8)), dim3(256), 0, st, (const T*)a->x, a->out, a->rows, a->cols, a->ldx);
        return check_launch("row_norms");
    });
}

extern "C" int romab200_copy2d(const rb_copy2d_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->cols > 0, "copy2d: empty input");
    if (check_dtype<float, __half, __nv_bfloat16>(a->dtype_src, "copy2d") || check_dtype<float, __half, __nv_bfloat16>(a->dtype_dst, "copy2d")) return 1;
    rb::launch_pdl(copy2d_kernel, dim3(grid1d(a->rows * a->cols, 256, 132 * 32)), dim3(256), 0, st, a->src, a->dst, a->rows, a->cols, a->lds, a->ldd,
                                                                   a->dtype_src, a->dtype_dst, a->row_scale, a->row_scale_reciprocal);
    return check_launch("copy2d");
}

extern "C" int romab200_gather_rows(const rb_gather_rows_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->src && a->dst && a->count > 0 && a->count <= 65535 && a->row_bytes > 0 && a->src_rows > 0 && a->dst_rows > 0,
               "gather_rows: bad shape");
    RB_REQUIRE(a->row_bytes % 16 == 0 && a->ld_src % 16 == 0 && a->ld_dst % 16 == 0 && a->ld_src >= a->row_bytes && a->ld_dst >= a->row_bytes &&
               ((uintptr_t)a->src) % 16 == 0 && ((uintptr_t)a->dst) % 16 == 0, "gather_rows: rows, pitches and pointers must be 16-byte multiples");
    const int64_t words = a->row_bytes / 16;
    dim3 grid(grid1d(words, 256, 132 * 8 / a->count + 1), a->count);
    rb::launch_pdl(gather_rows_kernel, grid, dim3(256), 0, st, (const uint4*)a->src, (uint4*)a->dst, a->src_index, a->dst_index, words,
                   a->ld_src / 16, a->ld_dst / 16, a->src_rows, a->dst_rows);
    return check_launch("gather_rows");
}

extern "C" int romab200_split_f16x3(const rb_split_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->rows > 0 && a->cols > 0 && a->ldd >= 3 * a->cols, "split_f16x3: bad shape");
    rb::launch_pdl(split_f16x3_kernel, dim3(grid1d(a->rows * a->cols, 256, 132 * 32)), dim3(256), 0, st, a->x, (__half*)a->dst, a->rows, a->cols, a->ldx, a->ldd,
                                                                        a->row_norm, a->layout_b);
    return check_launch("split_f16x3");
}

extern "C" int romab200_split_f16s(const rb_split_pair_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->x && a->hi && a->lo && a->rows > 0 && a->cols > 0 && a->ldd >= a->cols, "split_f16s: bad arguments");
    const int cols4 = (a->cols + 3) / 4;
    if (a->ldx % 4 == 0 && a->ldd % 4 == 0 && (int64_t)cols4 * 4 <= a->ldx && (int64_t)cols4 * 4 <= a->ldd && ((uintptr_t)a->x) % 16 == 0 &&
        ((uintptr_t)a->hi) % 8 == 0 && ((uintptr_t)a->lo) % 8 == 0) {
        rb::launch_pdl(split_f16s_vec_kernel, dim3(grid1d(a->rows * cols4, 256, 132 * 32)), dim3(256), 0, st, a->x, (__half*)a->hi, (__half*)a->lo, a->rows, cols4,
                       a->cols, a->ldx, a->ldd, a->row_norm);
    } else {
        rb::launch_pdl(split_f16s_kernel, dim3(grid1d(a->rows * a->cols, 256, 132 * 32)), dim3(256), 0, st, a->x, (__half*)a->hi, (__half*)a->lo, a->rows, a->cols,
                       a->ldx, a->ldd, a->row_norm);
    }
    return check_launch("split_f16s");
}

extern "C" int romab200_im2col_patch(const rb_im2col_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->height % a->patch == 0 && a->width % a->patch == 0, "im2col: %dx%d not a multiple of patch %d", a->height, a->width, a->patch);
    int64_t total = (int64_t)a->batch * (a->height / a->patch) * (a->width / a->patch) * 3 * a->patch * a->patch;
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype_out, "im2col_patch", [&](auto t) {
        using TO = typename decltype(t)::type;
        rb::launch_pdl(im2col_patch_kernel<TO>, dim3(grid1d(total, 256, 132 * 32)), dim3(256), 0, st, a->image, (TO*)a->out, a->batch, a->height, a->width, a->patch, a->ldo);
        return check_launch("im2col_patch");
    });
}

extern "C" int romab200_assemble_tokens(const rb_tokens_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int64_t total = (int64_t)a->batch * (a->npatch + 1) * a->dim;
    rb::launch_pdl(assemble_tokens_kernel, dim3(grid1d(total, 256, 132 * 32)), dim3(256), 0, st, a->patch, a->cls, a->pos, a->tokens, a->batch, a->npatch, a->dim);
    return check_launch("assemble_tokens");
}

extern "C" int romab200_transpose(const rb_transpose_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    int b0 = a->batch0 > 0 ? a->batch0 : 1, b1 = a->batch1 > 0 ? a->batch1 : 1;
    dim3 grid((a->cols + 31) / 32, (a->rows + 31) / 32, b0 * b1), block(32, 8);
    RB_REQUIRE(grid.y <= 65535 && grid.z <= 65535, "transpose: grid too large");
    return with_dtype<float, __half, __nv_bfloat16>(a->dtype, "transpose", [&](auto t) {
        // a transpose only moves bits: the 16-bit types share one kernel
        using T = std::conditional_t<sizeof(typename decltype(t)::type) == 4, float, uint16_t>;
        rb::launch_pdl(transpose_kernel<T>, grid, block, 0, st, (const T*)a->src, (T*)a->dst, a->rows, a->cols, a->lds, a->ldd, b1, a->ss0, a->ss1, a->sd0, a->sd1);
        return check_launch("transpose");
    });
}
