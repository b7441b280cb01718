// TinyRoMa (romatch/models/tiny.py) kernels: XFeat backbone pieces, the fused correlation / argmax / soft-argmax embedding,
// the warp-and-concat prologue of the matcher heads and the match() epilogue.  fp32 on the CUDA cores, like the reference.
#include "common.cuh"
#include <math.h>

namespace {

inline unsigned blocks_for(int64_t total, int block) {
    int64_t g = (total + block - 1) / block;
    return (unsigned)(g < 65535 * 16 ? g : 65535 * 16);
}

// --------------------------------------------------------------------------------------------------
// direct convolution: each thread owns 4 consecutive output channels (one float4 of the weight row) of CONV_P pixels;
// the TC threads of a pixel row share their input loads (broadcast), the weights stream through L1.
// --------------------------------------------------------------------------------------------------
constexpr int CONV_P = 8;

template <int K, bool VEC>
__global__ void __launch_bounds__(256, 2) tiny_conv_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ weight,
                                                        const float* __restrict__ bias, const float* __restrict__ col_scale,
                                                        const float* __restrict__ R, int64_t ldi, int64_t ldo, int64_t ldw, int64_t ldr,
                                                        int B, int hi, int wi, int ho, int wo, int cin, int cout, int stride, int relu, int tc) {
    rb::pdl_wait();
    const int q = threadIdx.x % tc, r = threadIdx.x / tc, rows = blockDim.x / tc;
    const int n0 = (blockIdx.y * tc + q) * 4;
    if (n0 >= ldw) return;
    const int64_t npix = (int64_t)B * ho * wo;
    const int64_t base = (int64_t)blockIdx.x * rows * CONV_P + r;
    int pb[CONV_P], py[CONV_P], px[CONV_P];
#pragma unroll
    for (int k = 0; k < CONV_P; ++k) {
        int64_t p = base + (int64_t)k * rows;
        if (p >= npix) { pb[k] = -1; py[k] = px[k] = 0; continue; }
        px[k] = (int)(p % wo); int64_t t = p / wo; py[k] = (int)(t % ho); pb[k] = (int)(t / ho);
    }
    float acc[CONV_P][4];
#pragma unroll
    for (int k = 0; k < CONV_P; ++k) acc[k][0] = acc[k][1] = acc[k][2] = acc[k][3] = 0.f;
    constexpr int PAD = K / 2;
    for (int tap = 0; tap < K * K; ++tap) {
        const int ky = tap / K, kx = tap % K;
        const float* src[CONV_P];
#pragma unroll
        for (int k = 0; k < CONV_P; ++k) {
            int yi = py[k] * stride + ky - PAD, xi = px[k] * stride + kx - PAD;
            bool ok = pb[k] >= 0 && yi >= 0 && yi < hi && xi >= 0 && xi < wi;
            src[k] = ok ? in + (((int64_t)pb[k] * hi + yi) * wi + xi) * ldi : nullptr;
        }
        const float* wt = weight + (int64_t)tap * cin * ldw + n0;
        if (VEC) {
            for (int c = 0; c < cin; c += 4) {
                float4 w0 = __ldg((const float4*)(wt + (int64_t)(c + 0) * ldw));
                float4 w1 = __ldg((const float4*)(wt + (int64_t)(c + 1) * ldw));
                float4 w2 = __ldg((const float4*)(wt + (int64_t)(c + 2) * ldw));
                float4 w3 = __ldg((const float4*)(wt + (int64_t)(c + 3) * ldw));
#pragma unroll
                for (int k = 0; k < CONV_P; ++k) {
                    float4 v = src[k] ? __ldg((const float4*)(src[k] + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
                    acc[k][0] = fmaf(v.x, w0.x, acc[k][0]); acc[k][1] = fmaf(v.x, w0.y, acc[k][1]);
                    acc[k][2] = fmaf(v.x, w0.z, acc[k][2]); acc[k][3] = fmaf(v.x, w0.w, acc[k][3]);
                    acc[k][0] = fmaf(v.y, w1.x, acc[k][0]); acc[k][1] = fmaf(v.y, w1.y, acc[k][1]);
                    acc[k][2] = fmaf(v.y, w1.z, acc[k][2]); acc[k][3] = fmaf(v.y, w1.w, acc[k][3]);
                    acc[k][0] = fmaf(v.z, w2.x, acc[k][0]); acc[k][1] = fmaf(v.z, w2.y, acc[k][1]);
                    acc[k][2] = fmaf(v.z, w2.z, acc[k][2]); acc[k][3] = fmaf(v.z, w2.w, acc[k][3]);
                    acc[k][0] = fmaf(v.w, w3.x, acc[k][0]); acc[k][1] = fmaf(v.w, w3.y, acc[k][1]);
                    acc[k][2] = fmaf(v.w, w3.z, acc[k][2]); acc[k][3] = fmaf(v.w, w3.w, acc[k][3]);
                }
            }
        } else {
            for (int c = 0; c < cin; ++c) {
                float4 w0 = __ldg((const float4*)(wt + (int64_t)c * ldw));
#pragma unroll
                for (int k = 0; k < CONV_P; ++k) {
                    float v = src[k] ? __ldg(src[k] + c) : 0.f;
                    acc[k][0] = fmaf(v, w0.x, acc[k][0]); acc[k][1] = fmaf(v, w0.y, acc[k][1]);
                    acc[k][2] = fmaf(v, w0.z, acc[k][2]); acc[k][3] = fmaf(v, w0.w, acc[k][3]);
                }
            }
        }
    }
#pragma unroll
    for (int k = 0; k < CONV_P; ++k) {
        if (pb[k] < 0) continue;
        const int64_t p = ((int64_t)pb[k] * ho + py[k]) * wo + px[k];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + j;
            if (n >= cout) break;
            float v = acc[k][j];
            if (bias) v += bias[n];
            if (relu) v = fmaxf(v, 0.f);
            if (col_scale) v *= col_scale[n];
            if (R) v += R[p * ldr + n];
            out[p * ldo + n] = v;
        }
    }
}

// --------------------------------------------------------------------------------------------------
// channel mean + optional InstanceNorm2d(1): one CTA per image, statistics in double
// --------------------------------------------------------------------------------------------------
__device__ double block_sum_d(double v, double* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    double s = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
    return s;
}

__global__ void __launch_bounds__(1024) tiny_gray_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int64_t hw, int norm, float eps) {
    rb::pdl_wait();
    __shared__ double red[32];
    const float* src = in + (int64_t)blockIdx.x * C * hw;
    float* dst = out + (int64_t)blockIdx.x * hw;
    double s = 0.0;
    for (int64_t p = threadIdx.x; p < hw; p += blockDim.x) {
        float g = 0.f;
        for (int c = 0; c < C; ++c) g += src[(int64_t)c * hw + p];
        g /= (float)C;
        dst[p] = g;
        s += g;
    }
    if (!norm) return;
    const double mean = block_sum_d(s, red) / (double)hw;
    double v = 0.0;
    for (int64_t p = threadIdx.x; p < hw; p += blockDim.x) {      // each thread re-reads what it wrote
        double d = (double)dst[p] - mean;
        v += d * d;
    }
    const double var = block_sum_d(v, red) / (double)hw;
    const float m = (float)mean, inv = (float)(1.0 / sqrt(var + (double)eps));
    for (int64_t p = threadIdx.x; p < hw; p += blockDim.x) dst[p] = (dst[p] - m) * inv;
}

__global__ void tiny_avgpool4_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int hi, int wi, int C) {
    rb::pdl_wait();
    const int ho = hi / 4, wo = wi / 4;
    const int64_t total = (int64_t)B * ho * wo * C;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        int c = (int)(idx % C); int64_t p = idx / C;
        int x = (int)(p % wo); int64_t t = p / wo; int y = (int)(t % ho); int b = (int)(t / ho);
        const float* s = in + (((int64_t)b * hi + 4 * y) * wi + 4 * x) * C + c;
        float acc = 0.f;
        for (int dy = 0; dy < 4; ++dy)
            for (int dx = 0; dx < 4; ++dx) acc += s[((int64_t)dy * wi + dx) * C];
        out[idx] = acc / 16.f;
    }
}

__global__ void tiny_add3_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c, float* __restrict__ out, int64_t n) {
    rb::pdl_wait();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) out[i] = (a[i] + b[i]) + c[i];
}

// --------------------------------------------------------------------------------------------------
// fused correlation + argmax + soft-argmax.  CTA = 64 query pixels x 4 groups of 64 threads; a query's 64-d feature lives in
// registers, image 1 streams through shared memory in tiles of 64 pixels, group g scores pixels g*16 .. g*16+15 of every tile
// (all lanes of a warp read the same row: broadcast).  Every thread keeps (first-index argmax, online-softmax max / sum / 2-column
// weighted sum) of its share; the four partial states are merged in shared memory at the end.
// --------------------------------------------------------------------------------------------------
constexpr int PE_C = 64, PE_I = 64, PE_G = 4, PE_TJ = 64;

struct SoftState { float m, l, ax, ay; };

__device__ __forceinline__ void soft_push(SoftState& st, float s, float gx, float gy) {
    if (s > st.m) {
        float a = expf(st.m - s);
        st.l = fmaf(st.l, a, 1.f); st.ax = fmaf(st.ax, a, gx); st.ay = fmaf(st.ay, a, gy); st.m = s;
    } else {
        float e = expf(s - st.m);
        st.l += e; st.ax = fmaf(e, gx, st.ax); st.ay = fmaf(e, gy, st.ay);
    }
}

__device__ __forceinline__ void soft_merge(SoftState& st, const SoftState& o) {
    float M = fmaxf(st.m, o.m);
    if (M == -INFINITY) return;
    float a = expf(st.m - M), b = expf(o.m - M);
    st.l = st.l * a + o.l * b; st.ax = st.ax * a + o.ax * b; st.ay = st.ay * a + o.ay * b; st.m = M;
}

__global__ void __launch_bounds__(PE_I * PE_G) tiny_pos_embed_kernel(const float* __restrict__ f0, const float* __restrict__ f1, float* __restrict__ state,
                                                                     int n0, int h1, int w1, float scale, int exact,
                                                                     const float* __restrict__ gx, const float* __restrict__ gy,
                                                                     const float* __restrict__ glx, const float* __restrict__ gly) {
    rb::pdl_wait();
    __shared__ __align__(16) float sf1[PE_TJ][PE_C];
    __shared__ SoftState s_soft[PE_G][PE_I];
    __shared__ float s_bv[PE_G][PE_I];
    __shared__ int s_bi[PE_G][PE_I];
    const int tid = threadIdx.x, il = tid % PE_I, g = tid / PE_I;
    const int b = blockIdx.y;
    const int i = blockIdx.x * PE_I + il;
    const int n1 = h1 * w1;
    float4 q[PE_C / 4];
    const float4* f0r = (const float4*)(f0 + ((int64_t)b * n0 + (i < n0 ? i : 0)) * PE_C);
#pragma unroll
    for (int c = 0; c < PE_C / 4; ++c) q[c] = f0r[c];
    const float4* f1b = (const float4*)(f1 + (int64_t)b * n1 * PE_C);
    SoftState st = {-INFINITY, 0.f, 0.f, 0.f};
    float bv = -INFINITY; int bi = 0;
    for (int j0 = 0; j0 < n1; j0 += PE_TJ) {
        __syncthreads();
#pragma unroll
        for (int k = 0; k < PE_TJ * PE_C / 4 / (PE_I * PE_G); ++k) {
            int idx = tid + k * PE_I * PE_G, jj = idx / (PE_C / 4), cc = idx % (PE_C / 4);
            float4 v = j0 + jj < n1 ? f1b[(int64_t)(j0 + jj) * (PE_C / 4) + cc] : make_float4(0.f, 0.f, 0.f, 0.f);
            *(float4*)&sf1[jj][cc * 4] = v;
        }
        __syncthreads();
        for (int t = 0; t < PE_TJ / PE_G; ++t) {
            const int jj = g * (PE_TJ / PE_G) + t, j = j0 + jj;
            if (j >= n1) break;
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < PE_C / 4; ++c) {
                float4 f = *(const float4*)&sf1[jj][c * 4];
                acc = fmaf(f.x, q[c].x, acc); acc = fmaf(f.y, q[c].y, acc);
                acc = fmaf(f.z, q[c].z, acc); acc = fmaf(f.w, q[c].w, acc);
            }
            const float s = acc / scale;
            const int yj = j / w1, xj = j - yj * w1;
            if (exact) {
                soft_push(st, s, gx[xj], gy[yj]);
            } else {
                if (s > bv) { bv = s; bi = j; }
                if (((yj | xj) & 3) == 0) soft_push(st, s, glx[xj >> 2], gly[yj >> 2]);
            }
        }
    }
    s_soft[g][il] = st; s_bv[g][il] = bv; s_bi[g][il] = bi;
    __syncthreads();
    if (g != 0 || i >= n0) return;
    for (int o = 1; o < PE_G; ++o) {
        soft_merge(st, s_soft[o][il]);
        float v = s_bv[o][il]; int k = s_bi[o][il];
        if (v > bv || (v == bv && k < bi)) { bv = v; bi = k; }
    }
    float px, py;
    if (exact) {
        px = st.ax / st.l; py = st.ay / st.l;
    } else {
        const float e = (float)bi;                 // the reference concatenates the argmax index itself as the extra logit
        const float M = fmaxf(st.m, e);
        const float a = expf(st.m - M), eb = expf(e - M);
        const float L = st.l * a + eb;
        px = (st.ax * a + eb * gx[bi % w1]) / L;
        py = (st.ay * a + eb * gy[bi / w1]) / L;
    }
    float* o = state + ((int64_t)b * n0 + i) * 3;
    o[0] = px; o[1] = py; o[2] = 0.f;
}

// --------------------------------------------------------------------------------------------------
// [f0 | grid_sample(f1, flow) | flow]: one thread per output element
// --------------------------------------------------------------------------------------------------
__global__ void tiny_warp_concat_kernel(const float* __restrict__ f0, const float* __restrict__ f1, const float* __restrict__ state, float* __restrict__ out,
                                        int64_t ldf0, int64_t ldf1, int64_t lds, int64_t ldo, int B, int h0, int w0, int h1, int w1, int C) {
    rb::pdl_wait();
    const int CT = 2 * C + 2;
    const int64_t total = (int64_t)B * h0 * w0 * CT;
    for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
        const int ch = (int)(idx % CT); const int64_t p = idx / CT;
        const int b = (int)(p / ((int64_t)h0 * w0));
        float v;
        if (ch < C) {
            v = f0[p * ldf0 + ch];
        } else if (ch >= 2 * C) {
            v = state[p * lds + (ch - 2 * C)];
        } else {
            const int c = ch - C;
            // grid_sample, bilinear, zeros, align_corners=False: x = (gx + 1) * W / 2 - 0.5
            const float x = (state[p * lds + 0] + 1.f) * (0.5f * w1) - 0.5f;
            const float y = (state[p * lds + 1] + 1.f) * (0.5f * h1) - 0.5f;
            const float xf = floorf(x), yf = floorf(y);
            const float wx = x - xf, wy = y - yf;
            const int x0 = (int)xf, y0 = (int)yf;
            const float* src = f1 + (int64_t)b * h1 * w1 * ldf1 + c;
            auto at = [&](int yy, int xx) -> float {
                return (yy >= 0 && yy < h1 && xx >= 0 && xx < w1) ? src[((int64_t)yy * w1 + xx) * ldf1] : 0.f;
            };
            v = at(y0, x0) * ((1.f - wy) * (1.f - wx)) + at(y0, x0 + 1) * ((1.f - wy) * wx) +
                at(y0 + 1, x0) * (wy * (1.f - wx)) + at(y0 + 1, x0 + 1) * (wy * wx);
        }
        out[p * ldo + ch] = v;
    }
}

__global__ void tiny_match_epilogue_kernel(const float* __restrict__ state, float* __restrict__ warp, float* __restrict__ cert, int B, int H, int W,
                                           const float* __restrict__ gx, const float* __restrict__ gy) {
    rb::pdl_wait();
    const int64_t total = (int64_t)B * H * W;
    for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (int64_t)gridDim.x * blockDim.x) {
        const int x = (int)(p % W), y = (int)((p / W) % H);
        const float* s = state + p * 3;
        *(float4*)(warp + p * 4) = make_float4(gx[x], gy[y], s[0], s[1]);
        cert[p] = 1.f / (1.f + expf(-s[2]));
    }
}

}  // namespace

extern "C" int romab200_tiny_conv(const rb_tiny_conv_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a && a->in && a->out && a->weight, "tiny_conv: null operand");
    RB_REQUIRE(a->ksize == 1 || a->ksize == 3, "tiny_conv: kernel size %d (1 or 3 supported)", a->ksize);
    RB_REQUIRE(a->stride == 1 || a->stride == 2, "tiny_conv: stride %d (1 or 2 supported)", a->stride);
    RB_REQUIRE(a->batch > 0 && a->cin > 0 && a->cout > 0 && a->ldw % 4 == 0 && a->ldw >= a->cout && a->ldi >= a->cin && a->ldo >= a->cout &&
               ((uintptr_t)a->weight) % 16 == 0, "tiny_conv: bad geometry (cin=%d cout=%d ldw=%lld)", a->cin, a->cout, (long long)a->ldw);
    RB_REQUIRE(a->ho == (a->hi - 1) / a->stride + 1 && a->wo == (a->wi - 1) / a->stride + 1, "tiny_conv: output size %dx%d does not match %dx%d / %d",
               a->ho, a->wo, a->hi, a->wi, a->stride);
    int quads = (int)(a->ldw / 4), tc = 1;
    while (tc < quads && tc < 64) tc *= 2;
    const int rows = 256 / tc;
    const int64_t npix = (int64_t)a->batch * a->ho * a->wo;
    dim3 grid((unsigned)((npix + rows * CONV_P - 1) / (rows * CONV_P)), (unsigned)((quads + tc - 1) / tc));
    const bool vec = a->cin % 4 == 0 && a->ldi % 4 == 0 && ((uintptr_t)a->in) % 16 == 0;
#define CONV(K, V) rb::launch_pdl(tiny_conv_kernel<K, V>, grid, dim3(256), 0, st, a->in, a->out, a->weight, a->bias, a->col_scale, a->R, a->ldi, a->ldo, \
                                  a->ldw, a->ldr, a->batch, a->hi, a->wi, a->ho, a->wo, a->cin, a->cout, a->stride, a->relu, tc)
    if (a->ksize == 3) { if (vec) CONV(3, true); else CONV(3, false); }
    else { if (vec) CONV(1, true); else CONV(1, false); }
#undef CONV
    return rb::check_launch("tiny_conv");
}

extern "C" int romab200_tiny_gray(const rb_tiny_gray_args* a, void* stream) {
    RB_REQUIRE(a && a->in && a->out && a->batch > 0 && a->channels > 0 && a->h > 0 && a->w > 0, "tiny_gray: bad arguments");
    rb::launch_pdl(tiny_gray_kernel, dim3(a->batch), dim3(1024), 0, (cudaStream_t)stream, a->in, a->out, a->channels, (int64_t)a->h * a->w,
                   a->instance_norm, a->eps);
    return rb::check_launch("tiny_gray");
}

extern "C" int romab200_tiny_avgpool4(const rb_tiny_avgpool_args* a, void* stream) {
    const int64_t total = (int64_t)a->batch * (a->hi / 4) * (a->wi / 4) * a->c;
    RB_REQUIRE(a && a->in && a->out && total > 0, "tiny_avgpool4: bad arguments");
    rb::launch_pdl(tiny_avgpool4_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, a->in, a->out, a->batch, a->hi, a->wi, a->c);
    return rb::check_launch("tiny_avgpool4");
}

extern "C" int romab200_tiny_add3(const rb_tiny_add3_args* a, void* stream) {
    RB_REQUIRE(a && a->a && a->b && a->c && a->out && a->n > 0, "tiny_add3: bad arguments");
    rb::launch_pdl(tiny_add3_kernel, dim3(blocks_for(a->n, 256)), dim3(256), 0, (cudaStream_t)stream, a->a, a->b, a->c, a->out, a->n);
    return rb::check_launch("tiny_add3");
}

extern "C" int romab200_tiny_pos_embed(const rb_tiny_pos_embed_args* a, void* stream) {
    RB_REQUIRE(a && a->f0 && a->f1 && a->state && a->grid_x && a->grid_y, "tiny_pos_embed: null operand");
    RB_REQUIRE(a->c == PE_C, "tiny_pos_embed: feature dim %d (64 supported)", a->c);
    RB_REQUIRE(a->exact || (a->grid_lr_x && a->grid_lr_y), "tiny_pos_embed: grid_lr needed unless exact");
    RB_REQUIRE(a->batch > 0 && a->h0 > 0 && a->w0 > 0 && a->h1 >= 4 && a->w1 >= 4 && a->h1 % 4 == 0 && a->w1 % 4 == 0,
               "tiny_pos_embed: bad sizes %dx%d / %dx%d", a->h0, a->w0, a->h1, a->w1);
    RB_REQUIRE(((uintptr_t)a->f0) % 16 == 0 && ((uintptr_t)a->f1) % 16 == 0, "tiny_pos_embed: features must be 16-byte aligned");
    const int n0 = a->h0 * a->w0;
    rb::launch_pdl(tiny_pos_embed_kernel, dim3((unsigned)((n0 + PE_I - 1) / PE_I), (unsigned)a->batch), dim3(PE_I * PE_G), 0, (cudaStream_t)stream,
                   a->f0, a->f1, a->state, n0, a->h1, a->w1, a->scale, a->exact, a->grid_x, a->grid_y, a->grid_lr_x, a->grid_lr_y);
    return rb::check_launch("tiny_pos_embed");
}

extern "C" int romab200_tiny_warp_concat(const rb_tiny_warp_concat_args* a, void* stream) {
    RB_REQUIRE(a && a->f0 && a->f1 && a->state && a->out && a->ldo >= 2 * a->c + 2 && a->lds >= 2, "tiny_warp_concat: bad arguments");
    const int64_t total = (int64_t)a->batch * a->h0 * a->w0 * (2 * a->c + 2);
    RB_REQUIRE(total > 0, "tiny_warp_concat: empty");
    rb::launch_pdl(tiny_warp_concat_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, a->f0, a->f1, a->state, a->out,
                   a->ldf0, a->ldf1, a->lds, a->ldo, a->batch, a->h0, a->w0, a->h1, a->w1, a->c);
    return rb::check_launch("tiny_warp_concat");
}

extern "C" int romab200_tiny_match_epilogue(const rb_tiny_epilogue_args* a, void* stream) {
    const int64_t total = (int64_t)a->batch * a->h * a->w;
    RB_REQUIRE(a && a->state && a->warp && a->cert && a->grid_x && a->grid_y && total > 0 && ((uintptr_t)a->warp) % 16 == 0,
               "tiny_match_epilogue: bad arguments");
    rb::launch_pdl(tiny_match_epilogue_kernel, dim3(blocks_for(total, 256)), dim3(256), 0, (cudaStream_t)stream, a->state, a->warp, a->cert,
                   a->batch, a->h, a->w, a->grid_x, a->grid_y);
    return rb::check_launch("tiny_match_epilogue");
}
