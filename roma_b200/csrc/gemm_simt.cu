// fp32 CUDA-core GEMM with the shared fused epilogue.
//
// This is the fp32 "parity" back-end of romab200_gemm (and the GP Cholesky's trailing update): plain
// FFMA accumulation in fp32, so results agree with the reference's CPU fp32 path to rounding-order
// differences.  The fast path for 16-bit operands is the tcgen05 back-end in gemm_tc.cu.
//
// Tiling: BM x BN x 16 block tiles, 256 threads, 8xTN register tiles (split 4+4 so that shared-memory
// reads are conflict-free float4s), double-buffered shared memory with register prefetch.
#include "common.cuh"

namespace rb {

Epilogue make_epilogue(const rb_gemm_args* a) {
    Epilogue e;
    e.C = a->C; e.C_lo = a->C_lo; e.ldc = a->ldc; e.dtype_c = a->dtype_c;
    e.alpha = a->alpha;
    e.bias = a->bias; e.col_scale = a->col_scale;
    e.R = a->R; e.ldr = a->ldr; e.dtype_r = a->dtype_r;
    e.act = a->act; e.epi = a->epi;
    e.norm_a = a->norm_a; e.norm_b = a->norm_b;
    e.eps = a->eps; e.inv_t = a->inv_t; e.diag_add = a->diag_add; e.cos_normalized = a->cos_normalized;
    e.rowmap = a->rowmap; e.pad_h = a->pad_h; e.pad_w = a->pad_w;
    e.seg_in = a->seg_in; e.seg_out = a->seg_out; e.seg_off = a->seg_off;
    e.M = a->M; e.N = a->N;
    return e;
}

struct SimtParams {
    const float* A; const float* B;
    int M, N, K;
    int64_t lda, ldb;
    int trans_b;
    int batch1;
    int64_t sa0, sa1, sb0, sb1, sc0, sc1, sr0, sr1, sna0, snb0;
    int ntaps, k_per_tap; int tap_rows[9]; int64_t a_rows;
    int vec_a, vec_b;
    int lower_only;          // skip tiles that lie entirely above the diagonal (symmetric trailing updates)
    Epilogue epi;
};

constexpr int BK = 16;

template <int BM, int BN, int TN>
__global__ void __launch_bounds__(256) gemm_simt_kernel(const SimtParams p) {
    rb::pdl_wait();
    constexpr int TM = 8;
    constexpr int NT_N = BN / TN;            // threads along n
    constexpr int LDA_S = BM + 4;
    constexpr int LDB_S = BN + 4;
    constexpr int A_F4 = BM * BK / 4 / 256;  // float4 loads per thread for the A tile
    constexpr int B_F4 = (BN * BK / 4 + 255) / 256;
    static_assert((BM / TM) * NT_N == 256, "256 threads");

    __shared__ __align__(16) float As[2][BK][LDA_S];
    __shared__ __align__(16) float Bs[2][BK][LDB_S];

    const int tid = threadIdx.x;
    const int tx = tid % NT_N, ty = tid / NT_N;
    const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
    if (p.lower_only && n0 >= m0 + BM) return;
    const int z = blockIdx.z, z0 = z / p.batch1, z1 = z % p.batch1;
    // no __restrict__: the GP solve (algo 2) runs P = P L^-T and X = Y L^-1 with C aliasing A.  That is safe because those products
    // have a single N tile (N <= 128 here) and a CTA reads all of K of its own rows before its epilogue writes them; the operands
    // are therefore not promised to be read-only (gemm_tc never aliases: its operands are separate split-fp16 scratch pairs).
    const float* A = p.A + z0 * p.sa0 + z1 * p.sa1;
    const float* B = p.B + z0 * p.sb0 + z1 * p.sb1;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

    float4 ra[A_F4], rbv[B_F4];
    const int ktiles = (p.K + BK - 1) / BK;

    auto load_tile = [&](int kt) {
        const int k0 = kt * BK;
        int tap = 0, kin = k0;
        if (p.ntaps > 1) { tap = k0 / p.k_per_tap; kin = k0 - tap * p.k_per_tap; }
        const int shift = p.ntaps > 1 ? p.tap_rows[tap] : 0;
        const int klim = p.ntaps > 1 ? p.k_per_tap : p.K;   // columns available in A / this tap
#pragma unroll
        for (int i = 0; i < A_F4; ++i) {
            int idx = tid + i * 256;
            int row = idx / (BK / 4), kq = idx % (BK / 4);
            int m = m0 + row;
            int64_t ar = (int64_t)m + shift;
            int kk = kin + kq * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < p.M && ar >= 0 && ar < p.a_rows) {
                const float* src = A + ar * p.lda + kk;
                if (p.vec_a && kk + 3 < klim) v = *reinterpret_cast<const float4*>(src);
                else {
                    if (kk + 0 < klim) v.x = src[0];
                    if (kk + 1 < klim) v.y = src[1];
                    if (kk + 2 < klim) v.z = src[2];
                    if (kk + 3 < klim) v.w = src[3];
                }
            }
            ra[i] = v;
        }
#pragma unroll
        for (int i = 0; i < B_F4; ++i) {
            int idx = tid + i * 256;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (!p.trans_b) {
                int row = idx / (BK / 4), kq = idx % (BK / 4);
                if (row < BN) {
                    int n = n0 + row, kk = k0 + kq * 4;
                    if (n < p.N) {
                        const float* src = B + (int64_t)n * p.ldb + kk;
                        if (p.vec_b && kk + 3 < p.K) v = *reinterpret_cast<const float4*>(src);
                        else {
                            if (kk + 0 < p.K) v.x = src[0];
                            if (kk + 1 < p.K) v.y = src[1];
                            if (kk + 2 < p.K) v.z = src[2];
                            if (kk + 3 < p.K) v.w = src[3];
                        }
                    }
                }
            } else {   // B is [K, N]: float4 along n
                int krow = idx / (BN / 4), nq = idx % (BN / 4);
                if (krow < BK) {
                    int kk = k0 + krow, n = n0 + nq * 4;
                    if (kk < p.K) {
                        const float* src = B + (int64_t)kk * p.ldb + n;
                        if (p.vec_b && n + 3 < p.N) v = *reinterpret_cast<const float4*>(src);
                        else {
                            if (n + 0 < p.N) v.x = src[0];
                            if (n + 1 < p.N) v.y = src[1];
                            if (n + 2 < p.N) v.z = src[2];
                            if (n + 3 < p.N) v.w = src[3];
                        }
                    }
                }
            }
            rbv[i] = v;
        }
    };
    auto store_tile = [&](int buf) {
#pragma unroll
        for (int i = 0; i < A_F4; ++i) {
            int idx = tid + i * 256;
            int row = idx / (BK / 4), kq = idx % (BK / 4);
            As[buf][kq * 4 + 0][row] = ra[i].x;
            As[buf][kq * 4 + 1][row] = ra[i].y;
            As[buf][kq * 4 + 2][row] = ra[i].z;
            As[buf][kq * 4 + 3][row] = ra[i].w;
        }
#pragma unroll
        for (int i = 0; i < B_F4; ++i) {
            int idx = tid + i * 256;
            if (!p.trans_b) {
                int row = idx / (BK / 4), kq = idx % (BK / 4);
                if (row < BN) {
                    Bs[buf][kq * 4 + 0][row] = rbv[i].x;
                    Bs[buf][kq * 4 + 1][row] = rbv[i].y;
                    Bs[buf][kq * 4 + 2][row] = rbv[i].z;
                    Bs[buf][kq * 4 + 3][row] = rbv[i].w;
                }
            } else {
                int krow = idx / (BN / 4), nq = idx % (BN / 4);
                if (krow < BK) *reinterpret_cast<float4*>(&Bs[buf][krow][nq * 4]) = rbv[i];
            }
        }
    };

    load_tile(0);
    store_tile(0);
    __syncthreads();

    for (int kt = 0; kt < ktiles; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < ktiles) load_tile(kt + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
            *reinterpret_cast<float4*>(&a[0]) = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
            *reinterpret_cast<float4*>(&a[4]) = *reinterpret_cast<const float4*>(&As[buf][k][BM / 2 + ty * 4]);
            *reinterpret_cast<float4*>(&b[0]) = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            if constexpr (TN == 8)
                *reinterpret_cast<float4*>(&b[4]) = *reinterpret_cast<const float4*>(&Bs[buf][k][BN / 2 + tx * 4]);
            // two accumulator columns per step (a channel pair of fp32 FMAs)
#pragma unroll
            for (int i = 0; i < TM; ++i) {
                const float2 ai = make_float2(a[i], a[i]);
#pragma unroll
                for (int j = 0; j < TN; j += 2) {
                    float2 r = rb::fma2(ai, make_float2(b[j], b[j + 1]), make_float2(acc[i][j], acc[i][j + 1]));
                    acc[i][j] = r.x; acc[i][j + 1] = r.y;
                }
            }
        }
        if (kt + 1 < ktiles) store_tile(buf ^ 1);
        __syncthreads();
    }

    // epilogue
    Epilogue e = p.epi;
    e.C = (char*)e.C + (z0 * p.sc0 + z1 * p.sc1) * dtype_size(e.dtype_c);
    if (e.C_lo) e.C_lo = (char*)e.C_lo + (z0 * p.sc0 + z1 * p.sc1) * 2;
    if (e.R) e.R = (const char*)e.R + (z0 * p.sr0 + z1 * p.sr1) * dtype_size(e.dtype_r);
    if (e.norm_a) e.norm_a += z0 * p.sna0;
    if (e.norm_b) e.norm_b += z0 * p.snb0;
    // fast path (GP trailing updates, plain fp32 linears): whole float4 groups, branches hoisted out of the element loop
    const bool fast = e.epi == RB_EPI_LINEAR && e.rowmap == RB_ROWMAP_NONE && e.dtype_c == RB_F32 && (e.ldc & 3) == 0 &&
                      (reinterpret_cast<uintptr_t>(e.C) & 15) == 0 && (!e.R || (e.dtype_r == RB_F32 && (e.ldr & 3) == 0 &&
                      (reinterpret_cast<uintptr_t>(e.R) & 15) == 0)) && e.act == RB_ACT_NONE && !e.col_scale;
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        int m = m0 + (i < 4 ? ty * 4 + i : BM / 2 + ty * 4 + (i - 4));
        if (m >= p.M) continue;
        int64_t orow = e.map_row(m);
        if (orow < 0) continue;
#pragma unroll
        for (int jg = 0; jg < TN; jg += 4) {
            const int n = n0 + (jg < 4 ? tx * 4 : BN / 2 + tx * 4);
            if (n >= p.N) continue;
            if (fast && n + 3 < p.N) {
                float4 v = make_float4(e.alpha * acc[i][jg], e.alpha * acc[i][jg + 1], e.alpha * acc[i][jg + 2], e.alpha * acc[i][jg + 3]);
                if (e.bias) { const float4 bb = *reinterpret_cast<const float4*>(e.bias + n); v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w; }
                if (e.R) { const float4 r = *reinterpret_cast<const float4*>((const float*)e.R + orow * e.ldr + n); v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w; }
                *reinterpret_cast<float4*>((float*)e.C + orow * e.ldc + n) = v;
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (n + j < p.N) store_split_any(e.C, e.C_lo, orow * e.ldc + n + j, e.dtype_c, e.apply(acc[i][jg + j], m, n + j, orow));
            }
        }
    }
}

int gemm_simt(const rb_gemm_args* a, cudaStream_t stream, int lower_only) {
    RB_REQUIRE(a->dtype_ab == RB_F32, "gemm_simt: operands must be fp32 (got dtype %d)", a->dtype_ab);
    RB_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "gemm_simt: empty problem M=%d N=%d K=%d", a->M, a->N, a->K);
    SimtParams p;
    p.A = (const float*)a->A; p.B = (const float*)a->B;
    p.M = a->M; p.N = a->N; p.K = a->K; p.lda = a->lda; p.ldb = a->ldb; p.trans_b = a->trans_b;
    p.batch1 = a->batch1 > 0 ? a->batch1 : 1;
    int batch0 = a->batch0 > 0 ? a->batch0 : 1;
    p.sa0 = a->sa0; p.sa1 = a->sa1; p.sb0 = a->sb0; p.sb1 = a->sb1; p.sc0 = a->sc0; p.sc1 = a->sc1;
    p.sr0 = a->sr0; p.sr1 = a->sr1; p.sna0 = a->sna0; p.snb0 = a->snb0;
    p.ntaps = a->ntaps > 1 ? a->ntaps : 1;
    p.k_per_tap = a->K / p.ntaps;
    for (int i = 0; i < 9; ++i) p.tap_rows[i] = a->tap_rows[i];
    p.a_rows = a->a_rows > 0 ? a->a_rows : a->M;
    if (p.ntaps > 1) {
        RB_REQUIRE(a->K % p.ntaps == 0 && p.k_per_tap % BK == 0, "gemm_simt: K/ntaps=%d must be a multiple of %d", p.k_per_tap, BK);
        RB_REQUIRE(!a->trans_b, "gemm_simt: taps need B as [N,K]");
    }
    p.vec_a = (a->lda % 4 == 0) && (((uintptr_t)a->A) % 16 == 0) && (a->sa0 % 4 == 0) && (a->sa1 % 4 == 0);
    p.vec_b = (a->ldb % 4 == 0) && (((uintptr_t)a->B) % 16 == 0) && (a->sb0 % 4 == 0) && (a->sb1 % 4 == 0);
    p.lower_only = lower_only;
    p.epi = make_epilogue(a);
    int zdim = batch0 * p.batch1;
    RB_REQUIRE(zdim <= 65535, "gemm_simt: batch %d too large", zdim);
    if (a->N <= 32) {
        dim3 grid((a->M + 255) / 256, (a->N + 31) / 32, zdim);
        rb::launch_pdl(gemm_simt_kernel<256, 32, 4>, dim3(grid), dim3(256), 0, stream, p);
    } else if (a->N <= 64) {
        dim3 grid((a->M + 127) / 128, (a->N + 63) / 64, zdim);
        rb::launch_pdl(gemm_simt_kernel<128, 64, 4>, dim3(grid), dim3(256), 0, stream, p);
    } else {
        dim3 grid((a->M + 127) / 128, (a->N + 127) / 128, zdim);
        rb::launch_pdl(gemm_simt_kernel<128, 128, 8>, dim3(grid), dim3(256), 0, stream, p);
    }
    return check_launch("gemm_simt");
}

}  // namespace rb
