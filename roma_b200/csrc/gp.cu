// GP posterior solve (romatch/models/matcher.py:301-309): batched fp32 Cholesky of K_yy + sigma*I
// and the two triangular solves with the Fourier basis as right-hand sides, without leaving the GPU
// and without cuSOLVER.
//
// Blocked right-looking factorisation on an augmented workspace
//      W = [ K_yy + sigma I ]   n rows
//          [      F^T       ]   nrhs rows
// Applying the panel solve and trailing update to the F^T rows as well turns them into (L^-1 F)^T, so the
// forward substitution is free.  The backward substitution then runs row-wise on those rows
// (X^T L = Y^T), again block by block, and leaves alpha^T = X^T in place: exactly the [N,K] operand
// layout that mu = K_xy @ alpha needs.  Three schedules of the same algorithm (rb_gp_solve_args.algo):
//   2 (the engine's default)  128-wide blocks: chol_block128_kernel factors the diagonal block in shared memory and
//                             forms its inverse, every other step is a K = 128 GEMM (13 dependent steps for n = 1600)
//   0                         32-wide panels as a chain of small kernels (chol_diag / chol_panel / trsm_back + GEMMs)
//   1                         one cooperative persistent kernel with device-wide barriers
// All O(n^3) work is in the trailing updates, which are romab200 fp32 GEMMs (lower triangle only).
#include "tma.cuh"

namespace rb {

constexpr int NB = 32;

// one warp factors the (bs x bs, bs <= 32) diagonal block held one row per lane; result (lower) to smem L
__device__ void factor_diag_block(const float* __restrict__ Wd, int64_t ldw, int bs, float (*L)[NB + 1], float* Wout) {
    const int lane = threadIdx.x & 31;
    float r[NB];
#pragma unroll
    for (int c = 0; c < NB; ++c) {
        float v = 0.f;
        if (lane < bs && c < bs && c <= lane) v = __ldcg(Wd + (int64_t)lane * ldw + c);
        if (c == lane && lane >= bs) v = 1.f;      // identity padding
        r[c] = v;
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        float djj = __shfl_sync(0xffffffffu, r[j], j);
        float d = sqrtf(djj);
        float lij = 0.f;
        if (lane == j) { r[j] = d; }
        else if (lane > j) { lij = r[j] / d; r[j] = lij; }
#pragma unroll
        for (int c = j + 1; c < NB; ++c) {
            float lcj = __shfl_sync(0xffffffffu, lij, c);
            if (c <= lane) r[c] = fmaf(-lij, lcj, r[c]);
        }
    }
#pragma unroll
    for (int c = 0; c < NB; ++c) {
        L[lane][c] = (c <= lane) ? r[c] : 0.f;
        if (Wout && lane < bs && c < bs && c <= lane) Wout[(int64_t)lane * ldw + c] = r[c];
    }
}

// one warp per problem: factor the diagonal block in place
__global__ void __launch_bounds__(32) chol_diag_kernel(float* __restrict__ W, int64_t ldw, int64_t stride, int k, int bs) {
    rb::pdl_wait();
    __shared__ float L[NB][NB + 1];
    float* Wd = W + (int64_t)blockIdx.x * stride + (int64_t)k * ldw + k;
    factor_diag_block(Wd, ldw, bs, L, Wd);
}

__device__ __forceinline__ void load_diag_block(const float* __restrict__ Wd, int64_t ldw, int bs, float (*L)[NB + 1]) {
    for (int idx = threadIdx.x; idx < NB * NB; idx += blockDim.x) {
        int i = idx / NB, c = idx % NB;
        float v = 0.f;
        if (i < bs && c < bs && c <= i) v = Wd[(int64_t)i * ldw + c];
        if (i == c && i >= bs) v = 1.f;        // identity padding of a partial block
        L[i][c] = v;
    }
}

// grid: (row_blocks, batch); block 128 threads: one thread per row below the (already factored) diagonal
// block solves x * L^T = a with the 32-step recurrence held in registers.
__global__ void __launch_bounds__(128) chol_panel_kernel(float* __restrict__ W, int64_t ldw, int64_t stride, int k, int bs, int total_rows) {
    rb::pdl_wait();
    __shared__ float L[NB][NB + 1];
    float* Wb = W + (int64_t)blockIdx.y * stride;
    load_diag_block(Wb + (int64_t)k * ldw + k, ldw, bs, L);
    __syncthreads();
    int row = k + bs + blockIdx.x * 128 + threadIdx.x;
    if (row >= total_rows) return;
    float* ar = Wb + (int64_t)row * ldw + k;
    float a[NB];
#pragma unroll
    for (int c = 0; c < NB; ++c) a[c] = c < bs ? ar[c] : 0.f;
#pragma unroll
    for (int j = 0; j < NB; ++j) {
        float x = a[j] / L[j][j];
        a[j] = x;
#pragma unroll
        for (int c = j + 1; c < NB; ++c) a[c] = fmaf(-x, L[c][j], a[c]);
    }
#pragma unroll
    for (int c = 0; c < NB; ++c)
        if (c < bs) ar[c] = a[c];
}

// backward substitution panel: rows of the RHS block solve x * L_kk = y (L_kk lower, bs x bs)
__global__ void __launch_bounds__(128) trsm_back_kernel(float* __restrict__ W, int64_t ldw, int64_t stride, int k, int bs, int n, int nrhs) {
    rb::pdl_wait();
    __shared__ float L[NB][NB + 1];
    float* Wb = W + (int64_t)blockIdx.y * stride;
    load_diag_block(Wb + (int64_t)k * ldw + k, ldw, bs, L);
    __syncthreads();
    int r = blockIdx.x * 128 + threadIdx.x;
    if (r >= nrhs) return;
    float* yr = Wb + (int64_t)(n + r) * ldw + k;
    float y[NB];
#pragma unroll
    for (int c = 0; c < NB; ++c) y[c] = c < bs ? yr[c] : 0.f;
#pragma unroll
    for (int j = NB - 1; j >= 0; --j) {
        float x = y[j] / L[j][j];
        y[j] = x;
#pragma unroll
        for (int c = 0; c < j; ++c) y[c] = fmaf(-x, L[j][c], y[c]);
    }
#pragma unroll
    for (int c = 0; c < NB; ++c)
        if (c < bs) yr[c] = y[c];
}

// --------------------------------------------------------------------------------------------------
// Persistent single-launch variant: the whole factorisation + both substitutions in ONE cooperative kernel.
// The multi-kernel version above spends its time in ~250 dependent launches of a few microseconds each; here all
// CTAs stay resident and step through the same phases separated by a device-wide barrier (one atomic counter,
// release/acquire fences).  Per 32-wide panel: phase A = every CTA that owns panel rows re-factors the 32x32
// diagonal block in shared memory (one warp, shuffles) and solves its 64 rows; phase B = 64x64 tiles of the
// rank-32 trailing update spread over all CTAs.  Diagonal factors go to a side buffer (`diag`) so that nobody
// overwrites a block other CTAs are still reading.
// --------------------------------------------------------------------------------------------------
struct GpPersistParams {
    float* W; float* diag; unsigned int* counter;
    int n, nrhs, batch;
    int64_t ldw, stride;
};

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int& target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += gridDim.x;
        __threadfence();                              // release: this CTA's writes are visible device-wide
        atomicAdd(counter, 1u);
        unsigned int seen;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(counter) : "memory");
        } while (seen < target);
        __threadfence();                              // acquire + L1 invalidate for the loads that follow
    }
    __syncthreads();
}

constexpr int GP_THREADS = 128;     // lean CTAs: the kernel is latency-bound and should leave the SMs to concurrent GEMM CTAs

__global__ void __launch_bounds__(GP_THREADS) gp_solve_persistent_kernel(const GpPersistParams p) {
    __shared__ float L[NB][NB + 1];
    __shared__ float Pi[64][NB + 1];
    __shared__ float Pj[64][NB + 1];
    const int tid = threadIdx.x;
    const int n = p.n, total = p.n + p.nrhs;
    const int nblk = (n + NB - 1) / NB;
    unsigned int target = 0;

    // ================= factorisation + forward substitution =================
    for (int kb = 0; kb < nblk; ++kb) {
        const int k = kb * NB, bs = min(NB, n - k);
        const int below = total - (k + bs);
        const int nchunks = (below + 63) / 64;
        // ---- phase A
        int loaded_e = -1;
        for (int item = blockIdx.x; item < p.batch * nchunks; item += gridDim.x) {
            const int e = item / nchunks, c = item - e * nchunks;
            float* Wb = p.W + (int64_t)e * p.stride;
            if (e != loaded_e) {
                __syncthreads();
                if (tid < 32) factor_diag_block(Wb + (int64_t)k * p.ldw + k, p.ldw, bs, L, nullptr);
                __syncthreads();
                loaded_e = e;
            }
            if (c == 0) {                                   // publish L_kk for the backward pass
                float* dst = p.diag + ((int64_t)e * nblk + kb) * NB * NB;
                for (int i = tid; i < NB * NB; i += GP_THREADS) dst[i] = L[i / NB][i % NB];
            }
            const int row = k + bs + c * 64 + tid;
            if (tid < 64 && row < total) {
                float* ar = Wb + (int64_t)row * p.ldw + k;
                float a[NB];
#pragma unroll
                for (int q = 0; q < NB; ++q) a[q] = q < bs ? __ldcg(ar + q) : 0.f;
#pragma unroll
                for (int j = 0; j < NB; ++j) {
                    float x = a[j] / L[j][j];
                    a[j] = x;
#pragma unroll
                    for (int q = j + 1; q < NB; ++q) a[q] = fmaf(-x, L[q][j], a[q]);
                }
#pragma unroll
                for (int q = 0; q < NB; ++q)
                    if (q < bs) ar[q] = a[q];
            }
        }
        grid_barrier(p.counter, target);
        // ---- phase B: C[i, j] -= sum_p P[i, p] P[j, p] on rows/cols beyond the panel
        const int r0 = k + bs;
        const int nt = n - r0;                              // trailing columns
        if (nt > 0) {
            const int tiles_i = (total - r0 + 63) / 64, tiles_j = (nt + 63) / 64;
            for (int item = blockIdx.x; item < p.batch * tiles_i * tiles_j; item += gridDim.x) {
                const int e = item / (tiles_i * tiles_j), t = item - e * (tiles_i * tiles_j);
                const int ti = t / tiles_j, tj = t - ti * tiles_j;
                const int i0 = r0 + ti * 64, j0 = r0 + tj * 64;
                if (i0 + 63 < n && j0 > i0 + 63) continue;  // whole tile strictly above the diagonal of the SPD part: never read
                float* Wb = p.W + (int64_t)e * p.stride;
                __syncthreads();
                for (int idx = tid; idx < 64 * NB; idx += GP_THREADS) {
                    const int r = idx / NB, q = idx - r * NB;
                    Pi[r][q] = (i0 + r < total && q < bs) ? __ldcg(Wb + (int64_t)(i0 + r) * p.ldw + k + q) : 0.f;
                    Pj[r][q] = (j0 + r < n && q < bs) ? __ldcg(Wb + (int64_t)(j0 + r) * p.ldw + k + q) : 0.f;
                }
                __syncthreads();
                const int tr = (tid / 16) * 8, tc = (tid % 16) * 4;
                float acc[8][4];
#pragma unroll
                for (int a = 0; a < 8; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
#pragma unroll
                for (int q = 0; q < NB; ++q) {
                    float av[8], bv[4];
#pragma unroll
                    for (int a = 0; a < 8; ++a) av[a] = Pi[tr + a][q];
#pragma unroll
                    for (int a = 0; a < 4; ++a) bv[a] = Pj[tc + a][q];
#pragma unroll
                    for (int a = 0; a < 8; ++a)
#pragma unroll
                        for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
                }
#pragma unroll
                for (int a = 0; a < 8; ++a) {
                    const int r = i0 + tr + a;
                    if (r >= total) continue;
                    float* cp = Wb + (int64_t)r * p.ldw + j0 + tc;
                    if (j0 + tc + 3 < n) {
                        float4 v = __ldcg(reinterpret_cast<const float4*>(cp));
                        v.x -= acc[a][0]; v.y -= acc[a][1]; v.z -= acc[a][2]; v.w -= acc[a][3];
                        *reinterpret_cast<float4*>(cp) = v;
                    } else {
#pragma unroll
                        for (int b = 0; b < 4; ++b)
                            if (j0 + tc + b < n) cp[b] = __ldcg(cp + b) - acc[a][b];
                    }
                }
            }
            grid_barrier(p.counter, target);
        }
    }
    // ================= backward substitution on the RHS rows: X^T L = Y^T =================
    for (int kb = nblk - 1; kb >= 0; --kb) {
        const int k = kb * NB, bs = min(NB, n - k);
        const int nchunks = (p.nrhs + 63) / 64;
        int loaded_e = -1;
        for (int item = blockIdx.x; item < p.batch * nchunks; item += gridDim.x) {
            const int e = item / nchunks, c = item - e * nchunks;
            float* Wb = p.W + (int64_t)e * p.stride;
            if (e != loaded_e) {
                __syncthreads();
                const float* src = p.diag + ((int64_t)e * nblk + kb) * NB * NB;
                for (int i = tid; i < NB * NB; i += GP_THREADS) L[i / NB][i % NB] = __ldcg(src + i);
                __syncthreads();
                loaded_e = e;
            }
            const int r = c * 64 + tid;
            if (tid < 64 && r < p.nrhs) {
                float* yr = Wb + (int64_t)(n + r) * p.ldw + k;
                float y[NB];
#pragma unroll
                for (int q = 0; q < NB; ++q) y[q] = q < bs ? __ldcg(yr + q) : 0.f;
#pragma unroll
                for (int j = NB - 1; j >= 0; --j) {
                    float x = y[j] / L[j][j];
                    y[j] = x;
#pragma unroll
                    for (int q = 0; q < j; ++q) y[q] = fmaf(-x, L[j][q], y[q]);
                }
#pragma unroll
                for (int q = 0; q < NB; ++q)
                    if (q < bs) yr[q] = y[q];
            }
        }
        if (k == 0) break;
        grid_barrier(p.counter, target);
        // Y[:, 0:k] -= X[:, k:k+bs] . L[k:k+bs, 0:k]
        const int tiles_i = (p.nrhs + 63) / 64, tiles_j = (k + 63) / 64;
        for (int item = blockIdx.x; item < p.batch * tiles_i * tiles_j; item += gridDim.x) {
            const int e = item / (tiles_i * tiles_j), t = item - e * (tiles_i * tiles_j);
            const int ti = t / tiles_j, tj = t - ti * tiles_j;
            const int i0 = ti * 64, j0 = tj * 64;
            float* Wb = p.W + (int64_t)e * p.stride;
            __syncthreads();
            for (int idx = tid; idx < 64 * NB; idx += GP_THREADS) {
                const int r = idx / NB, q = idx - r * NB;
                Pi[r][q] = (i0 + r < p.nrhs && q < bs) ? __ldcg(Wb + (int64_t)(n + i0 + r) * p.ldw + k + q) : 0.f;
            }
            for (int idx = tid; idx < NB * 64; idx += GP_THREADS) {           // L rows k..k+bs, columns j0..j0+63 -> Pj[col][p]
                const int q = idx / 64, cidx = idx - q * 64;
                Pj[cidx][q] = (q < bs && j0 + cidx < k) ? __ldcg(Wb + (int64_t)(k + q) * p.ldw + j0 + cidx) : 0.f;
            }
            __syncthreads();
            const int tr = (tid / 16) * 8, tc = (tid % 16) * 4;
            float acc[8][4];
#pragma unroll
            for (int a = 0; a < 8; ++a)
#pragma unroll
                for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;
#pragma unroll
            for (int q = 0; q < NB; ++q) {
                float av[8], bv[4];
#pragma unroll
                for (int a = 0; a < 8; ++a) av[a] = Pi[tr + a][q];
#pragma unroll
                for (int a = 0; a < 4; ++a) bv[a] = Pj[tc + a][q];
#pragma unroll
                for (int a = 0; a < 8; ++a)
#pragma unroll
                    for (int b = 0; b < 4; ++b) acc[a][b] = fmaf(av[a], bv[b], acc[a][b]);
            }
#pragma unroll
            for (int a = 0; a < 8; ++a) {
                const int r = i0 + tr + a;
                if (r >= p.nrhs) continue;
                float* cp = Wb + (int64_t)(n + r) * p.ldw + j0 + tc;
                if (j0 + tc + 3 < k) {
                    float4 v = __ldcg(reinterpret_cast<const float4*>(cp));
                    v.x -= acc[a][0]; v.y -= acc[a][1]; v.z -= acc[a][2]; v.w -= acc[a][3];
                    *reinterpret_cast<float4*>(cp) = v;
                } else {
#pragma unroll
                    for (int b = 0; b < 4; ++b)
                        if (j0 + tc + b < k) cp[b] = __ldcg(cp + b) - acc[a][b];
                }
            }
        }
        grid_barrier(p.counter, target);
    }
}

static int sub_gemm(const float* A, int64_t lda, const float* B, int64_t ldb, int trans_b, float* C, int64_t ldc, int M, int N, int K,
                    int batch, int64_t stride, cudaStream_t st, int lower_only = 0) {
    rb_gemm_args g = {};
    g.A = A; g.B = B; g.C = C; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
    g.dtype_ab = RB_F32; g.dtype_c = RB_F32; g.trans_b = trans_b;
    g.batch0 = batch; g.batch1 = 1; g.sa0 = stride; g.sb0 = stride; g.sc0 = stride; g.sr0 = stride;
    g.ntaps = 1; g.alpha = -1.0f; g.R = C; g.ldr = ldc; g.dtype_r = RB_F32;
    return gemm_simt(&g, st, lower_only);
}


// --------------------------------------------------------------------------------------------------
// 128-wide blocked variant (algo 2): the dependent chain shrinks from n/32 = 50 to n/128 = 13 steps and every O(n^2)
// piece becomes a K = 128 GEMM.  One CTA per problem factors the 128x128 diagonal block entirely in shared memory
// (four 32-wide sub-panels) and also forms its explicit inverse, so that the panel solve  P = A21 L11^-T  and the
// backward block solve  X = Y L11^-1  are plain GEMMs against the inverse (diagonal blocks of K + sigma*I are well
// conditioned: cond(L11) <= ~30).
// --------------------------------------------------------------------------------------------------
constexpr int BB = 128, BBP = BB + 1;

constexpr int CB_THREADS = 512;
constexpr int CB_BUF = 40;                 // floats per broadcast buffer: 32 column entries, 1/pivot, 1/sqrt(pivot), pad
constexpr int VP = BB + 4;                 // row pitch of L^-1 in shared memory: rows stay 16-byte aligned for float4 access
constexpr int CB_SMEM_FLOATS = BB * BBP + 3 + BB * VP + 32 * BB + 2 * CB_BUF + BB;
#ifdef RB_CB_CLK
__device__ long long g_cb_clk[32];
#define CBCLK(i) if (threadIdx.x == 0 && blockIdx.x == 0) g_cb_clk[i] = clock64();
#else
#define CBCLK(i)
#endif

// 1/sqrt(p) of a pivot.  This sits on the serial chain of the whole factorisation, hence MUFU.RSQ and one Newton step
// (full fp32 accuracy; pivots of K + sigma*I are far from the denormal range) instead of a division and a square root.
__device__ __forceinline__ float rsqrt_newton(float p) {
    float r;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(p));
    return r * fmaf(-0.5f * p * r, r, 1.5f);
}

// One CTA factors the 128x128 diagonal block in shared memory and forms the inverse of the factor.
//   factorisation: four 32-column sub-panels.  Sub-panel: one thread per row keeps its 32 entries in registers; for step
//     j the 32 threads of the diagonal rows publish their column-j entry (double-buffered, one named barrier per step,
//     column j+1 is published before the rest of step j's updates so that the barrier wait overlaps them), everybody
//     applies a[c] -= a[j]/p * col[c] and scales a[j] by 1/sqrt(p).  Trailing update inside the block: 4x4 register
//     tiles over the lower triangle, operands read as float4 from a transposed copy of the sub-panel.
//   inverse: 32x32 diagonal blocks by forward substitution in registers, then block row by block row
//     V[bi][0:bi] = -V[bi][bi] (L[bi][0:bi] V[0:bi][0:bi])  as two register-tiled products.
// History: a fully unrolled first version had 20k instructions and was instruction-fetch bound (664 us per block); a
// column-at-a-time version with per-element predicates took 105 us; shared-memory wavefronts (one per cycle per SM)
// and in-order issue behind dependent loads are what the current structure is built around.
__global__ void __launch_bounds__(CB_THREADS) chol_block128_kernel(float* __restrict__ W, float* __restrict__ inv_ws, int64_t ldw, int64_t stride,
                                                                   int64_t ws_stride, int k, int kb, int bs) {
    rb::pdl_wait();
    extern __shared__ __align__(16) float sm128[];
    float* S = sm128;                                  // [128][129] the block, then its factor L (lower)
    float* V = sm128 + ((BB * BBP + 3) & ~3);          // [128][132] L^-1
    float* PT = V + BB * VP;                           // [32][128]  transposed sub-panel; later the scratch X of the inverse
    float* buf = PT + 32 * BB;                         // [2][CB_BUF]
    float* Dinv = buf + 2 * CB_BUF;                    // [128] 1 / L_ii
    const int tid = threadIdx.x;
    float* Wd = W + (int64_t)blockIdx.x * stride + (int64_t)k * ldw + k;
    CBCLK(0)
    {
        float v[16];
#pragma unroll 1
        for (int base = 0; base < BB * BB; base += 16 * CB_THREADS) {
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const int idx = base + u * CB_THREADS + tid, i = idx >> 7, c = idx & 127;
                v[u] = (i < bs && c < bs && c <= i) ? __ldcg(Wd + (int64_t)i * ldw + c) : ((i == c && i >= bs) ? 1.f : 0.f);
            }
#pragma unroll
            for (int u = 0; u < 16; ++u) {
                const int idx = base + u * CB_THREADS + tid, i = idx >> 7, c = idx & 127;
                S[i * BBP + c] = v[u];
            }
        }
        for (int idx = tid; idx < BB * VP / 4; idx += CB_THREADS) reinterpret_cast<float4*>(V)[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    __syncthreads();
    CBCLK(1)
    for (int j0 = 0; j0 < BB; j0 += 32) {
        const int nrows = BB - j0;                           // rows of this sub-panel = threads taking part (multiple of 32)
        if (tid < nrows) {
            const int row = j0 + tid;
            float a[32];
#pragma unroll
            for (int c = 0; c < 32; ++c) a[c] = S[row * BBP + j0 + c];
            // Producer/consumer barriers: the diagonal rows (warp 0) publish column j+1 and bar.arrive on FULL[(j+1)&1]
            // as soon as they have it; the other warps bar.sync on it one step later.  FREE[x] goes the other way
            // (readers of buffer x are done) so that warp 0 never overwrites a buffer still being read.  Inside warp 0 the
            // pivot scale travels by shuffle, which keeps shared-memory round trips off the serial chain
            // (shuffle -> 2 mul -> fma -> rsqrt + Newton -> next shuffle).
            const bool w0 = tid < 32;
            float rcur = 0.f;
            if (w0) {
                rcur = rsqrt_newton(a[0]);
                buf[tid] = a[0];
                if (tid == 0) { buf[32] = rcur * rcur; buf[33] = rcur; Dinv[j0] = rcur; }
                bar_arrive(1, nrows);
            }
#pragma unroll
            for (int j = 0; j < 32; ++j) {
                const float* bj = buf + (j & 1) * CB_BUF;
                float* bn = buf + ((j + 1) & 1) * CB_BUF;
                if (w0) __syncwarp(); else bar_named(1 + (j & 1), nrows);
                float4 cv[8];
#pragma unroll
                for (int c4 = (j + 1) / 4; c4 < 8; ++c4) cv[c4] = *reinterpret_cast<const float4*>(bj + 4 * c4);
                float ip, isq;
                if (w0) { isq = __shfl_sync(0xffffffffu, rcur, j); ip = isq * isq; }
                else { ip = bj[32]; isq = bj[33]; }
                const float t = a[j] * ip;
                const bool upd = tid > j;
                if (tid >= j) a[j] *= isq;                    // owner: p / sqrt(p) = sqrt(p)
                if (j < 31) {
                    if (w0) {
                        const float4 c1 = cv[(j + 1) / 4];
                        const float cj1 = ((j + 1) & 3) == 0 ? c1.x : ((j + 1) & 3) == 1 ? c1.y : ((j + 1) & 3) == 2 ? c1.z : c1.w;
                        if (upd) a[j + 1] = fmaf(-t, cj1, a[j + 1]);
                        rcur = rsqrt_newton(a[j + 1]);        // every lane, meaningful in lane j+1 (no divergence)
                        if (j >= 1) bar_named(3 + ((j + 1) & 1), nrows);
                        bn[tid] = a[j + 1];
                        if (tid == j + 1) { bn[32] = rcur * rcur; bn[33] = rcur; Dinv[j0 + j + 1] = rcur; }
                        bar_arrive(1 + ((j + 1) & 1), nrows);
                    }
                    if (upd) {
#pragma unroll
                        for (int c4 = (j + 1) / 4; c4 < 8; ++c4) {
                            const int lo = w0 ? j + 2 : j + 1;        // warp 0 has applied column j+1 already
                            if (4 * c4 + 0 >= j + 1 && 4 * c4 + 0 >= lo) a[4 * c4 + 0] = fmaf(-t, cv[c4].x, a[4 * c4 + 0]);
                            if (4 * c4 + 1 >= j + 1 && 4 * c4 + 1 >= lo) a[4 * c4 + 1] = fmaf(-t, cv[c4].y, a[4 * c4 + 1]);
                            if (4 * c4 + 2 >= j + 1 && 4 * c4 + 2 >= lo) a[4 * c4 + 2] = fmaf(-t, cv[c4].z, a[4 * c4 + 2]);
                            if (4 * c4 + 3 >= j + 1 && 4 * c4 + 3 >= lo) a[4 * c4 + 3] = fmaf(-t, cv[c4].w, a[4 * c4 + 3]);
                        }
                    }
                    if (!w0 && j < 30) bar_arrive(3 + (j & 1), nrows);
                }
            }
#pragma unroll
            for (int c = 0; c < 32; ++c) {
                if (tid >= 32 || c <= tid) S[row * BBP + j0 + c] = a[c];
                PT[c * BB + row] = a[c];
            }
        }
        __syncthreads();
        CBCLK(2 + (j0 >> 5) * 2)
        // trailing update of the block: C[i][c] -= sum_p L[i][j0+p] L[c][j0+p] over lower-triangular 4x4 tiles
        const int r0 = j0 + 32, nt = (BB - r0) >> 2, ntiles = nt * (nt + 1) / 2;
        if (tid < ntiles) {
            int ti = (int)((sqrtf(8.f * tid + 1.f) - 1.f) * 0.5f);
            while (ti * (ti + 1) / 2 > tid) --ti;
            while ((ti + 1) * (ti + 2) / 2 <= tid) ++ti;
            const int tj = tid - ti * (ti + 1) / 2;
            const int i0 = r0 + 4 * ti, c0 = r0 + 4 * tj;
            float acc[4][4];
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;
#pragma unroll 8
            for (int p = 0; p < 32; ++p) {
                const float4 av = *reinterpret_cast<const float4*>(PT + p * BB + i0);
                const float4 bv = *reinterpret_cast<const float4*>(PT + p * BB + c0);
                const float aa[4] = {av.x, av.y, av.z, av.w}, bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
                for (int x = 0; x < 4; ++x)
#pragma unroll
                    for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(aa[x], bb[y], acc[x][y]);
            }
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) S[(i0 + x) * BBP + c0 + y] -= acc[x][y];
        }
        __syncthreads();
        CBCLK(3 + (j0 >> 5) * 2)
    }
    // ---- inverse, diagonal 32x32 blocks: thread = (block, column), forward substitution with the column in registers
    if (tid < BB) {
        const int o = tid & ~31, jj = tid & 31;
        float x[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            const float* Lr = S + (o + i) * BBP + o;
            float s0 = i == jj ? 1.f : 0.f, s1 = 0.f;
#pragma unroll
            for (int p = 0; p < i; ++p) {
                if (p & 1) s1 = fmaf(-Lr[p], x[p], s1);
                else s0 = fmaf(-Lr[p], x[p], s0);
            }
            x[i] = i >= jj ? (s0 + s1) * Dinv[o + i] : 0.f;
            V[(o + i) * VP + o + jj] = x[i];
        }
    }
    __syncthreads();
    CBCLK(10)
    // ---- inverse, off-diagonal: block row bi,  X = L[bi][0:bi] V[0:bi][0:bi]  then  V[bi][0:bi] = -V[bi][bi] X
    for (int bi = 1; bi < 4; ++bi) {
        const int ctiles = 8 * bi, ntile = 8 * ctiles;         // 4x4 tiles: 8 tile rows x 8*bi tile columns
        const int ct = tid % ctiles, rt = tid / ctiles, c0 = 4 * ct, rr = 32 * bi + 4 * rt;
        if (tid < ntile) {
            float acc[4][4];
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;
#pragma unroll 4
            for (int p = c0 & ~31; p < 32 * bi; ++p) {          // V[p][c] = 0 above the diagonal block of column c
                const float4 bv = *reinterpret_cast<const float4*>(V + p * VP + c0);
                const float aa[4] = {S[rr * BBP + p], S[(rr + 1) * BBP + p], S[(rr + 2) * BBP + p], S[(rr + 3) * BBP + p]};
                const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
                for (int x = 0; x < 4; ++x)
#pragma unroll
                    for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(aa[x], bb[y], acc[x][y]);
            }
#pragma unroll
            for (int x = 0; x < 4; ++x) *reinterpret_cast<float4*>(PT + (4 * rt + x) * BB + c0) = make_float4(acc[x][0], acc[x][1], acc[x][2], acc[x][3]);
        }
        __syncthreads();
        if (tid < ntile) {
            float acc[4][4];
#pragma unroll
            for (int x = 0; x < 4; ++x)
#pragma unroll
                for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;
            const float* Vd = V + rr * VP + 32 * bi;            // rows of the diagonal block V[bi][bi] (lower triangular)
#pragma unroll 4
            for (int q = 0; q < 4 * rt + 4; ++q) {
                const float4 bv = *reinterpret_cast<const float4*>(PT + q * BB + c0);
                const float aa[4] = {Vd[q], Vd[VP + q], Vd[2 * VP + q], Vd[3 * VP + q]};
                const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
                for (int x = 0; x < 4; ++x)
#pragma unroll
                    for (int y = 0; y < 4; ++y) acc[x][y] = fmaf(aa[x], bb[y], acc[x][y]);
            }
#pragma unroll
            for (int x = 0; x < 4; ++x) *reinterpret_cast<float4*>(V + (rr + x) * VP + c0) = make_float4(-acc[x][0], -acc[x][1], -acc[x][2], -acc[x][3]);
        }
        __syncthreads();
    }
    CBCLK(11)
    // ---- write back: L in place (lower triangle), L^-1 to the workspace as a dense [128][128] block
    float* Vout = inv_ws + (int64_t)blockIdx.x * ws_stride + (int64_t)kb * BB * BB;
    for (int idx = tid; idx < BB * BB; idx += CB_THREADS) {
        const int i = idx >> 7, c = idx & 127;
        if (i < bs && c < bs && c <= i) Wd[(int64_t)i * ldw + c] = S[i * BBP + c];
        Vout[idx] = V[i * VP + c];
    }
    CBCLK(12)
}

struct Split2 { __half* hi; __half* lo; };

static int plain_gemm(const float* A, int64_t lda, const float* B, int64_t ldb, int trans_b, float* C, int64_t ldc, int M, int N, int K,
                      int batch, int64_t sa, int64_t sb, int64_t sc, cudaStream_t st) {
    rb_gemm_args g = {};
    g.A = A; g.B = B; g.C = C; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
    g.dtype_ab = RB_F32; g.dtype_c = RB_F32; g.trans_b = trans_b;
    g.batch0 = batch; g.batch1 = 1; g.sa0 = sa; g.sb0 = sb; g.sc0 = sc;
    g.ntaps = 1; g.alpha = 1.0f;
    return gemm_simt(&g, st);
}

static int gp_solve_block128(const rb_gp_solve_args* a, cudaStream_t st) {
    const int n = a->n, total = a->n + a->nrhs, nblk = (n + BB - 1) / BB;
    const int64_t ws_stride = (int64_t)nblk * BB * BB;
    float* W = a->W;
    float* ws = (float*)a->workspace;
    const size_t smem = (size_t)CB_SMEM_FLOATS * sizeof(float);
    if (ensure_smem<chol_block128_kernel>((int)smem, "gp_solve")) return 1;
    for (int kb = 0; kb < nblk; ++kb) {
        const int k = kb * BB, bs = n - k < BB ? n - k : BB;
        rb::launch_pdl(chol_block128_kernel, dim3(a->batch), dim3(CB_THREADS), smem, st, W, ws, a->ldw, a->stride, ws_stride, k, kb, bs);
        if (check_launch("chol_block128")) return 1;
        const int below = total - (k + bs);
        if (below > 0) {
            float* P = W + (int64_t)(k + bs) * a->ldw + k;                 // A21 (and the F^T rows)  ->  P = A21 L11^-T, in place
            if (plain_gemm(P, a->ldw, ws + (int64_t)kb * BB * BB, BB, 0, P, a->ldw, below, bs, bs, a->batch, a->stride, ws_stride, a->stride, st)) return 1;
            const int nt = n - (k + bs);
            if (nt > 0) {
                float* Tm = W + (int64_t)(k + bs) * a->ldw + (k + bs);
                if (sub_gemm(P, a->ldw, P, a->ldw, 0, Tm, a->ldw, below, nt, bs, a->batch, a->stride, st, 1)) return 1;
            }
        }
    }
    for (int kb = nblk - 1; kb >= 0; --kb) {
        const int k = kb * BB, bs = n - k < BB ? n - k : BB;
        float* Y = W + (int64_t)n * a->ldw + k;                            // RHS block  ->  X = Y L11^-1, in place
        if (plain_gemm(Y, a->ldw, ws + (int64_t)kb * BB * BB, BB, 1, Y, a->ldw, a->nrhs, bs, bs, a->batch, a->stride, ws_stride, a->stride, st)) return 1;
        if (k > 0) {
            float* Lr = W + (int64_t)k * a->ldw;
            float* Y0 = W + (int64_t)n * a->ldw;
            if (sub_gemm(Y, a->ldw, Lr, a->ldw, 1, Y0, a->ldw, a->nrhs, k, bs, a->batch, a->stride, st)) return 1;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// algo 3: the schedule of algo 2 with every O(n^2 * 128) product on the tensor cores.  The panels are converted to RB_F16S pairs
// (split_f16s_batched) and contracted by the split-fp16 tcgen05 GEMM (fp32-class: K = 128 means 8 accumulator updates); the
// symmetric trailing update and the back-substitution update are in-place fp32 reduce-adds of the TMA-store epilogue.  Nothing
// aliases any more: the GEMMs read the scratch pairs and write the fp32 workspace.
//   workspace = [batch * nblk * 128 * 128 fp32 block inverses | scratch pairs], see gp_tc_workspace_bytes().
// ---------------------------------------------------------------------------------------------------------------------------
static int64_t gp_tc_scratch_halves(int n, int nrhs, int64_t ldw) {       // fp16 elements per problem and plane
    const int64_t fwd = (int64_t)(n + nrhs) * BB + BB * BB;               // panel rows + inverse block
    const int64_t bwd = (int64_t)nrhs * BB + BB * BB + BB * ldw;          // Y block + inverse block + L rows
    return fwd > bwd ? fwd : bwd;
}

static int tc_gemm(const Split2& A, int64_t lda, const Split2& B, int64_t ldb, int trans_b, float* C, int64_t ldc, int M, int N, int K, int batch,
                   int64_t sa, int64_t sb, int64_t sc, float alpha, bool accumulate, cudaStream_t st) {
    rb_gemm_args g = {};
    g.A = A.hi; g.A_lo = A.lo; g.B = B.hi; g.B_lo = B.lo; g.C = C; g.M = M; g.N = N; g.K = K; g.lda = lda; g.ldb = ldb; g.ldc = ldc;
    g.dtype_ab = RB_F16S; g.dtype_c = RB_F32; g.trans_b = trans_b;
    g.batch0 = batch; g.batch1 = 1; g.sa0 = sa; g.sb0 = sb; g.sc0 = sc;
    g.ntaps = 1; g.alpha = alpha;
    if (accumulate) { g.R = C; g.ldr = ldc; g.dtype_r = RB_F32; g.sr0 = sc; }
    return gemm_tc(&g, st);
}

static int gp_solve_tc(const rb_gp_solve_args* a, cudaStream_t st) {
    const int n = a->n, total = a->n + a->nrhs, nblk = (n + BB - 1) / BB;
    const int64_t ws_stride = (int64_t)nblk * BB * BB;
    float* W = a->W;
    float* ws = (float*)a->workspace;
    const int64_t sh = gp_tc_scratch_halves(n, a->nrhs, a->ldw);          // plane stride between problems
    __half* s_hi = reinterpret_cast<__half*>(ws + (int64_t)a->batch * ws_stride);
    __half* s_lo = s_hi + (int64_t)a->batch * sh;
    const size_t smem = (size_t)CB_SMEM_FLOATS * sizeof(float);
    if (ensure_smem<chol_block128_kernel>((int)smem, "gp_solve")) return 1;
    for (int kb = 0; kb < nblk; ++kb) {
        const int k = kb * BB, bs = n - k < BB ? n - k : BB;
        rb::launch_pdl(chol_block128_kernel, dim3(a->batch), dim3(CB_THREADS), smem, st, W, ws, a->ldw, a->stride, ws_stride, k, kb, bs);
        if (check_launch("chol_block128")) return 1;
        const int below = total - (k + bs);
        if (below <= 0) continue;
        float* P = W + (int64_t)(k + bs) * a->ldw + k;                   // A21 (and the F^T rows)  ->  P = A21 L11^-T
        const Split2 sP{s_hi, s_lo}, sInv{s_hi + (int64_t)total * BB, s_lo + (int64_t)total * BB};
        if (split_f16s_batched(P, sP.hi, sP.lo, below, bs, a->ldw, BB, a->batch, a->stride, sh, st)) return 1;
        if (split_f16s_batched(ws + (int64_t)kb * BB * BB, sInv.hi, sInv.lo, bs, bs, BB, BB, a->batch, ws_stride, sh, st)) return 1;
        if (tc_gemm(sP, BB, sInv, BB, 0, P, a->ldw, below, bs, bs, a->batch, sh, sh, a->stride, 1.0f, false, st)) return 1;
        const int nt = n - (k + bs);
        if (nt > 0) {
            if (split_f16s_batched(P, sP.hi, sP.lo, below, bs, a->ldw, BB, a->batch, a->stride, sh, st)) return 1;
            float* Tm = W + (int64_t)(k + bs) * a->ldw + (k + bs);        // trailing matrix (+ F^T rows) -= P P^T  (first nt rows of P as B)
            if (tc_gemm(sP, BB, sP, BB, 0, Tm, a->ldw, below, nt, bs, a->batch, sh, sh, a->stride, -1.0f, true, st)) return 1;
        }
    }
    for (int kb = nblk - 1; kb >= 0; --kb) {
        const int k = kb * BB, bs = n - k < BB ? n - k : BB;
        float* Y = W + (int64_t)n * a->ldw + k;                            // RHS block  ->  X = Y L11^-1
        const Split2 sY{s_hi, s_lo}, sInv{s_hi + (int64_t)a->nrhs * BB, s_lo + (int64_t)a->nrhs * BB};
        const Split2 sL{sInv.hi + BB * BB, sInv.lo + BB * BB};
        if (split_f16s_batched(Y, sY.hi, sY.lo, a->nrhs, bs, a->ldw, BB, a->batch, a->stride, sh, st)) return 1;
        if (split_f16s_batched(ws + (int64_t)kb * BB * BB, sInv.hi, sInv.lo, bs, bs, BB, BB, a->batch, ws_stride, sh, st)) return 1;
        if (tc_gemm(sY, BB, sInv, BB, 1, Y, a->ldw, a->nrhs, bs, bs, a->batch, sh, sh, a->stride, 1.0f, false, st)) return 1;
        if (k > 0) {
            float* Lr = W + (int64_t)k * a->ldw;                           // L[k:k+bs, 0:k] as the [K, N] operand
            float* Y0 = W + (int64_t)n * a->ldw;
            if (split_f16s_batched(Y, sY.hi, sY.lo, a->nrhs, bs, a->ldw, BB, a->batch, a->stride, sh, st)) return 1;
            if (split_f16s_batched(Lr, sL.hi, sL.lo, bs, k, a->ldw, a->ldw, a->batch, a->stride, sh, st)) return 1;
            if (tc_gemm(sY, BB, sL, a->ldw, 1, Y0, a->ldw, a->nrhs, k, bs, a->batch, sh, sh, a->stride, -1.0f, true, st)) return 1;
        }
    }
    return 0;
}

}  // namespace rb

using namespace rb;

#ifdef RB_CB_CLK
extern "C" int romab200_debug_clk(long long* out) { return (int)cudaMemcpyFromSymbol(out, rb::g_cb_clk, sizeof(long long) * 32); }
#endif

extern "C" int romab200_gp_solve(const rb_gp_solve_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    RB_REQUIRE(a->n > 0 && a->nrhs > 0 && a->batch > 0 && a->ldw >= a->n, "gp_solve: bad shape n=%d nrhs=%d batch=%d", a->n, a->nrhs, a->batch);
    RB_REQUIRE(a->batch <= 65535, "gp_solve: batch too large");
    if (a->workspace && a->algo == 3) {
        const int64_t nblk128 = (a->n + BB - 1) / BB;
        RB_REQUIRE(a->ldw % 8 == 0 && a->stride % 8 == 0 && ((uintptr_t)a->W) % 16 == 0 && ((uintptr_t)a->workspace) % 16 == 0, "gp_solve: alignment (algo 3)");
        const int64_t need = (int64_t)a->batch * (nblk128 * BB * BB * 4 + 4 * gp_tc_scratch_halves(a->n, a->nrhs, a->ldw));
        RB_REQUIRE(a->workspace_bytes >= need, "gp_solve: workspace too small for algo 3 (%lld < %lld bytes)", (long long)a->workspace_bytes, (long long)need);
        return gp_solve_tc(a, st);
    }
    if (a->workspace && a->algo == 2) {
        const int64_t nblk128 = (a->n + BB - 1) / BB;
        RB_REQUIRE(a->ldw % 4 == 0 && ((uintptr_t)a->W) % 16 == 0 && ((uintptr_t)a->workspace) % 16 == 0, "gp_solve: alignment");
        RB_REQUIRE(a->workspace_bytes >= (int64_t)a->batch * nblk128 * BB * BB * 4, "gp_solve: workspace too small for algo 2");
        return gp_solve_block128(a, st);
    }
    if (a->workspace && a->algo == 1) {
        // single cooperative launch; workspace = [batch * ceil(n/32) * 1024 floats of diagonal factors | 1 counter word]
        RB_REQUIRE(a->ldw % 4 == 0 && ((uintptr_t)a->W) % 16 == 0, "gp_solve: W must be 16-byte aligned with ldw %% 4 == 0");
        const int64_t nblk = (a->n + NB - 1) / NB;
        const int64_t diag_floats = (int64_t)a->batch * nblk * NB * NB;
        RB_REQUIRE(a->workspace_bytes >= (diag_floats + 1) * 4, "gp_solve: workspace too small (%lld < %lld bytes)",
                   (long long)a->workspace_bytes, (long long)(diag_floats + 1) * 4);
        GpPersistParams p;
        p.W = a->W; p.diag = (float*)a->workspace; p.counter = (unsigned int*)((float*)a->workspace + diag_floats);
        p.n = a->n; p.nrhs = a->nrhs; p.batch = a->batch; p.ldw = a->ldw; p.stride = a->stride;
        RB_REQUIRE(cudaMemsetAsync(p.counter, 0, 4, st) == cudaSuccess, "gp_solve: memset failed");
        int per_sm = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gp_solve_persistent_kernel, GP_THREADS, 0);
        RB_REQUIRE(per_sm > 0, "gp_solve: cannot size the cooperative grid");
        void* kargs[] = {(void*)&p};
        cudaError_t err = cudaLaunchCooperativeKernel((void*)gp_solve_persistent_kernel, dim3(sm_count()), dim3(GP_THREADS), kargs, 0, st);
        RB_REQUIRE(err == cudaSuccess, "gp_solve: cooperative launch failed: %s", cudaGetErrorString(err));
        return check_launch("gp_solve_persistent");
    }
    const int n = a->n, total = a->n + a->nrhs;
    float* W = a->W;
    // factorisation + forward substitution on the augmented rows
    for (int k = 0; k < n; k += NB) {
        int bs = n - k < NB ? n - k : NB;
        int below = total - (k + bs);
        rb::launch_pdl(chol_diag_kernel, dim3(a->batch), dim3(32), 0, st, W, a->ldw, a->stride, k, bs);
        if (check_launch("chol_diag")) return 1;
        dim3 grid((below + 127) / 128, a->batch);
        rb::launch_pdl(chol_panel_kernel, dim3(grid), dim3(128), 0, st, W, a->ldw, a->stride, k, bs, total);
        if (check_launch("chol_panel")) return 1;
        int nt = n - (k + bs);
        if (nt > 0) {
            float* P = W + (int64_t)(k + bs) * a->ldw + k;           // panel rows below the block
            float* T = W + (int64_t)(k + bs) * a->ldw + (k + bs);    // trailing matrix
            if (sub_gemm(P, a->ldw, P, a->ldw, 0, T, a->ldw, total - (k + bs), nt, bs, a->batch, a->stride, st, 1)) return 1;   // only the lower triangle is ever read
        }
    }
    // backward substitution: X^T L = Y^T on rows n .. n+nrhs
    int last = ((n - 1) / NB) * NB;
    for (int k = last; k >= 0; k -= NB) {
        int bs = n - k < NB ? n - k : NB;
        dim3 grid((a->nrhs + 127) / 128, a->batch);
        rb::launch_pdl(trsm_back_kernel, dim3(grid), dim3(128), 0, st, W, a->ldw, a->stride, k, bs, n, a->nrhs);
        if (check_launch("trsm_back")) return 1;
        if (k > 0) {
            float* X = W + (int64_t)n * a->ldw + k;                  // solved block  [nrhs, bs]
            float* Lr = W + (int64_t)k * a->ldw;                     // L[k:k+bs, 0:k] as [K, N]
            float* Y = W + (int64_t)n * a->ldw;                      // remaining RHS [nrhs, k]
            if (sub_gemm(X, a->ldw, Lr, a->ldw, 1, Y, a->ldw, a->nrhs, k, bs, a->batch, a->stride, st)) return 1;
        }
    }
    return 0;
}
