// Fused attention forward for the two transformers of the path (F.scaled_dot_product_attention,
// romatch/models/transformer/layers/attention.py:50-63): DINOv2 ViT-L (16 heads x d=64, N=1601) and the
// embedding decoder (8 heads x d=128, N=1600).  softmax(Q K^T / sqrt(d)) V without ever writing the N x N
// scores to HBM (the un-fused path moves 2 x 164 MB per layer).
//
// One CTA = one (image, head, 128-query tile), 384 threads:
//   warps 0-7   two consumer warpgroups, 64 query rows each.  Per key tile: S = Q K_j^T with wgmma (A = Q, B = K_j, both
//               K-major from shared memory) into registers, online softmax in the exp2 domain on the accumulator fragments
//               (a row lives in the 4 lanes of a quad), rescale of the fp32 O accumulator, then O += P_j V_j with P_j as the
//               register A operand (the S fragment of 16 keys is exactly the A fragment of one k-step) and V_j the MN-major
//               B operand straight from the qkv buffer; finally O / l -> global.
//   warps 8-11  TMA producer (one lane): Q once, then K/V tiles through a STAGES-deep shared-memory ring.  Its registers go
//               to the consumers (setmaxnreg).
// The two warpgroups run independently, so one's softmax overlaps the other's MMAs.
//
// Split-fp16 (RB_F16S) variant for the parity mode, head_dim 64 (DINOv2 ViT-L): fp32-class attention on the f16 tensor pipe.
//   q, k, v arrive as (hi, lo') plane pairs (value = hi + lo' * 2^-11, written by the qkv GEMM epilogue).
//   S_j = Q K_j^T with three MMAs per k-step into TWO accumulators (main: hi.hi; cross: hi.lo' + lo'.hi), score = main +
//         cross * 2^-11; key tiles of 64.
//   P V : the probabilities are written in an exponent-shifted form so that ONE accumulator suffices:
//         O' = sum_j (Pt_hi + Pt_lo) V_hi + P_hi V_lo'      with Pt = 2048 p, Pt_hi = fp16(Pt), Pt_lo = fp16(Pt - Pt_hi),
//         P_hi = fp16(p) = Pt_hi / 2048, i.e. O' = 2048 * sum p (V_hi + V_lo' / 2048) up to a 2^-22 relative term.  p <= 1, so
//         Pt <= 2048 never overflows; the unscaled low part Pt_lo only underflows for p < 6e-5, where its absolute error
//         (1.5e-11 in units of p) is irrelevant.
//   out  = O' / (2048 l) written as an RB_F16S pair for the projection GEMM.
#include "tma.cuh"
#include "wgmma.cuh"
#include <type_traits>

namespace rb {

// ---- softmax and fragment helpers ------------------------------------------------------------------------------
namespace fa {
__device__ __forceinline__ float ex2(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
template <typename T> __device__ __forceinline__ uint32_t pack2(float a, float b) {
    T h[2] = {from_f<T>(a), from_f<T>(b)};
    return *reinterpret_cast<uint32_t*>(h);
}
template <typename T> __device__ __forceinline__ float2 unpack2(uint32_t w) {
    const T* h = reinterpret_cast<const T*>(&w);
    return make_float2(to_f(h[0]), to_f(h[1]));
}
// keeps registers that an in-flight wgmma reads alive (and unmodified) until after the wait
template <int R> __device__ __forceinline__ void keep_regs(const uint32_t (&a)[R][4]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" ::"r"(a[i][0]), "r"(a[i][1]), "r"(a[i][2]), "r"(a[i][3]) : "memory");
}
}  // namespace fa

struct FaParams {
    void* out; void* out_lo; int64_t ldo;     // [Bn, N, dim] rows of pitch ldo (elements); out_lo: low plane of the split variant
    int N, heads, dim;
    float scale_log2;                         // log2(e) / sqrt(d)
};

// D = head dim; SPLIT: RB_F16S planes (D = 64, T = __half)
template <int D, bool SPLIT> struct FaCfg {
    static constexpr int BQ = 128, BKV = SPLIT ? 64 : 128;
    static constexpr int NP = SPLIT ? 2 : 1;                // operand planes
    static constexpr int Q_BYTES = BQ * D * 2;              // one plane: D / 64 blocks of [BQ rows x 128 B]
    static constexpr int KV_BYTES = BKV * D * 2;            // one plane of one of K, V: D / 64 blocks of [BKV rows x 128 B]
    static constexpr int STAGE_BYTES = 2 * NP * KV_BYTES;   // K planes, then V planes
    static constexpr int STAGES = (200 * 1024 - NP * Q_BYTES) / STAGE_BYTES > 4 ? 4 : (200 * 1024 - NP * Q_BYTES) / STAGE_BYTES;
    static constexpr int SMEM = NP * Q_BYTES + STAGES * STAGE_BYTES + 1024 + 256;
    static_assert(STAGES >= 2, "shared memory budget");
};

template <int D, typename T, bool SPLIT>
__global__ void __launch_bounds__(384, 1) flash_attn_kernel(const __grid_constant__ CUtensorMap map_hi, const __grid_constant__ CUtensorMap map_lo,
                                                            const FaParams p) {
    rb::pdl_wait();
    using namespace fa;
    using Cfg = FaCfg<D, SPLIT>;
    constexpr int STAGES = Cfg::STAGES, BQ = Cfg::BQ, BKV = Cfg::BKV, NP = Cfg::NP, DB = D / 64;
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - ((uint32_t)__cvta_generic_to_shared(smem_raw) & 1023u)) & 1023u);   // offset on the array: keeps ld/st.shared
    uint8_t* sQ = smem;                                       // plane q at sQ + q * Q_BYTES
    uint8_t* sKV = sQ + NP * Cfg::Q_BYTES;                    // stage s: K planes, V planes
    uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + STAGES * Cfg::STAGE_BYTES);
    uint64_t* q_full = bars;                  // [1]
    uint64_t* kv_full = bars + 1;             // [STAGES]
    uint64_t* kv_empty = kv_full + STAGES;    // [STAGES]  one arrival per consumer warpgroup

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * BQ, head = blockIdx.y, img = blockIdx.z;
    const int ntiles = (p.N + BKV - 1) / BKV;

    if (threadIdx.x == 0) {
        mbar_init(q_full, 1);
        for (int s = 0; s < STAGES; ++s) { mbar_init(&kv_full[s], 1); mbar_init(&kv_empty[s], 2); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ===== TMA producer: boxes of 64 rows x 64 columns (128 B) =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == 8 && lane == 0) {
            const CUtensorMap* maps[2] = {&map_hi, &map_lo};
            const int cq = head * D, ck = p.dim + head * D, cv = 2 * p.dim + head * D;
            mbar_expect_tx(q_full, NP * Cfg::Q_BYTES);
            for (int pl = 0; pl < NP; ++pl)
                for (int b = 0; b < DB; ++b)
                    for (int h = 0; h < BQ / 64; ++h)
                        tma_load_3d(sQ + pl * Cfg::Q_BYTES + b * (BQ * 128) + h * (64 * 128), maps[pl], q_full, cq + 64 * b, q0 + 64 * h, img);
            for (int j = 0; j < ntiles; ++j) {
                const int s = j % STAGES;
                mbar_wait(&kv_empty[s], ((j / STAGES) & 1) ^ 1);
                mbar_expect_tx(&kv_full[s], Cfg::STAGE_BYTES);
                uint8_t* st = sKV + s * Cfg::STAGE_BYTES;
                for (int pl = 0; pl < NP; ++pl)
                    for (int b = 0; b < DB; ++b)
                        for (int h = 0; h < BKV / 64; ++h) {
                            const int off = b * (BKV * 128) + h * (64 * 128);
                            tma_load_3d(st + pl * Cfg::KV_BYTES + off, maps[pl], &kv_full[s], ck + 64 * b, j * BKV + 64 * h, img);
                            tma_load_3d(st + (NP + pl) * Cfg::KV_BYTES + off, maps[pl], &kv_full[s], cv + 64 * b, j * BKV + 64 * h, img);
                        }
            }
        }
        return;
    }

    // ===== consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64); this thread rows r and r + 8 of them =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int wg = warp >> 2, t = threadIdx.x & 127;
    const int quad = t & 3;
    float o[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};     // l_run: this thread's part of the row sums
    const uint32_t q_addr = smem_u32(sQ) + wg * (64 * 128);
    mbar_wait(q_full, 0);
    for (int j = 0; j < ntiles; ++j) {
        const int s = j % STAGES;
        mbar_wait(&kv_full[s], (j / STAGES) & 1);
        const uint32_t k_addr = smem_u32(sKV + s * Cfg::STAGE_BYTES), v_addr = k_addr + NP * Cfg::KV_BYTES;
        float sc[BKV / 2];
        float cr[SPLIT ? BKV / 2 : 1];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < D / 16; ++k) {
            const uint32_t qoff = (k >> 2) * (BQ * 128) + (k & 3) * 32, koff = (k >> 2) * (BKV * 128) + (k & 3) * 32;   // 64-element blocks, 32 B per k-step
            const uint64_t qh = gmma_desc(q_addr + qoff, 16, 1024), kh = gmma_desc(k_addr + koff, 16, 1024);
            Wgmma<BKV, BF16>::template ss<0>(sc, qh, kh, k != 0);
            if constexpr (SPLIT) {
                const uint64_t ql = gmma_desc(q_addr + Cfg::Q_BYTES + qoff, 16, 1024), kl = gmma_desc(k_addr + Cfg::KV_BYTES + koff, 16, 1024);
                Wgmma<BKV, BF16>::template ss<0>(cr, qh, kl, k != 0);
                Wgmma<BKV, BF16>::template ss<0>(cr, ql, kh, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(sc);
        if constexpr (SPLIT) {
            wgmma_fence_regs(cr);
#pragma unroll
            for (int i = 0; i < BKV / 2; ++i) sc[i] = fmaf(cr[i], 1.0f / RB_SPLIT_SCALE, sc[i]);
        }
        // scale, mask the keys beyond N, row maxima over the quad
        const int valid = min(BKV, p.N - j * BKV);
        float mx[2] = {m_run[0], m_run[1]};
#pragma unroll
        for (int i = 0; i < BKV / 2; ++i) {
            const int col = 8 * (i >> 2) + 2 * quad + (i & 1);
            sc[i] = col < valid ? sc[i] * p.scale_log2 : -INFINITY;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
        }
        float m_ref[2], alpha[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
            mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
            m_ref[h] = mx[h] == -INFINITY ? 0.f : mx[h];
            alpha[h] = ex2(m_run[h] - m_ref[h]);          // 0 on the first tile (m_run = -inf)
            l_run[h] *= alpha[h];
            m_run[h] = mx[h];
        }
#pragma unroll
        for (int i = 0; i < D / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
        // probabilities -> A fragments: k-step kk covers accumulator columns [16 kk, 16 kk + 16) = sc[8 kk .. 8 kk + 7]
        constexpr int KS = BKV / 16;
        uint32_t ph[KS][4];
        uint32_t pl[SPLIT ? KS : 1][4], pp[SPLIT ? KS : 1][4];
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int i = 8 * kk + 2 * r, h = r & 1;
                const float p0 = ex2(sc[i] - m_ref[h]), p1 = ex2(sc[i + 1] - m_ref[h]);
                if constexpr (SPLIT) {
                    l_run[h] += p0 + p1;
                    const uint32_t th = pack2<__half>(p0 * RB_SPLIT_SCALE, p1 * RB_SPLIT_SCALE);
                    const float2 thf = unpack2<__half>(th);
                    ph[kk][r] = th;
                    pl[kk][r] = pack2<__half>(p0 * RB_SPLIT_SCALE - thf.x, p1 * RB_SPLIT_SCALE - thf.y);
                    pp[kk][r] = pack2<__half>(p0, p1);
                } else {
                    ph[kk][r] = pack2<T>(p0, p1);
                    const float2 q = unpack2<T>(ph[kk][r]);
                    l_run[h] += q.x + q.y;                   // sum what the MMA will actually see
                }
            }
        }
        // O += P V: V tile = D / 64 blocks of [BKV keys x 128 B], MN-major; 16 keys = 2048 B, the next 64 columns BKV * 128 B further
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KS; ++kk) {
            const uint64_t vh = gmma_desc(v_addr + kk * 2048, BKV * 128, 1024);
            Wgmma<D, BF16>::template rs<1>(o, ph[kk], vh, 1);
            if constexpr (SPLIT) {
                const uint64_t vl = gmma_desc(v_addr + Cfg::KV_BYTES + kk * 2048, BKV * 128, 1024);
                Wgmma<D, BF16>::template rs<1>(o, pl[kk], vh, 1);
                Wgmma<D, BF16>::template rs<1>(o, pp[kk], vl, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(o);
        keep_regs(ph);
        if constexpr (SPLIT) { keep_regs(pl); keep_regs(pp); }
        if (t == 0) mbar_arrive(&kv_empty[s]);          // this warpgroup no longer reads stage s
    }
    // ===== O / l -> global (16-bit rows, or an RB_F16S pair) =====
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float l = l_run[h];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[h] = 1.0f / (SPLIT ? l * RB_SPLIT_SCALE : l);
    }
    const int row0 = q0 + wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int qi = row0 + 8 * h;
        if (qi >= p.N) continue;
        const int64_t off = ((int64_t)img * p.N + qi) * p.ldo + head * D + 2 * quad;
#pragma unroll
        for (int c = 0; c < D / 8; ++c) {
            const float v0 = o[4 * c + 2 * h] * inv[h], v1 = o[4 * c + 2 * h + 1] * inv[h];
            if constexpr (SPLIT) {
                const uint32_t hi = pack2<__half>(v0, v1);
                const float2 hf = unpack2<__half>(hi);
                *reinterpret_cast<uint32_t*>((__half*)p.out + off + 8 * c) = hi;
                *reinterpret_cast<uint32_t*>((__half*)p.out_lo + off + 8 * c) = pack2<__half>((v0 - hf.x) * RB_SPLIT_SCALE, (v1 - hf.y) * RB_SPLIT_SCALE);
            } else {
                *reinterpret_cast<uint32_t*>((T*)p.out + off + 8 * c) = pack2<T>(v0, v1);
            }
        }
    }
}

template <int D, typename T, bool SPLIT>
static int launch_fa(const CUtensorMap& map_hi, const CUtensorMap& map_lo, const FaParams& p, int batch, cudaStream_t st) {
    using Cfg = FaCfg<D, SPLIT>;
    auto kernel = flash_attn_kernel<D, T, SPLIT>;
    if (ensure_smem<flash_attn_kernel<D, T, SPLIT>>(Cfg::SMEM, "flash_attn")) return 1;
    dim3 grid((p.N + Cfg::BQ - 1) / Cfg::BQ, p.heads, batch);
    rb::launch_pdl(kernel, dim3(grid), dim3(384), Cfg::SMEM, st, map_hi, map_lo, p);
    return check_launch(SPLIT ? "flash_attn_split" : "flash_attn");
}

}  // namespace rb

using namespace rb;

extern "C" int romab200_flash_attn(const rb_flash_attn_args* a, void* stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const bool split = a->dtype == RB_F16S;
    // RB_F16S is a pair of fp16 planes
    return with_dtype<__half, __nv_bfloat16>(split ? RB_F16 : a->dtype, "flash_attn", [&](auto t) {
        using T = typename decltype(t)::type;
        RB_REQUIRE(a->head_dim == 64 || (a->head_dim == 128 && !split), "flash_attn: head_dim %d unsupported (64, 128; split-fp16: 64)", a->head_dim);
        RB_REQUIRE(!split || (a->qkv_lo && a->out_lo && ((uintptr_t)a->qkv_lo) % 16 == 0 && ((uintptr_t)a->out_lo) % 16 == 0),
                   "flash_attn: split-fp16 needs 16-byte aligned qkv_lo and out_lo planes");
        const int dim = a->heads * a->head_dim;
        RB_REQUIRE(a->ld_qkv >= 3 * dim && (a->ld_qkv * 2) % 16 == 0 && ((uintptr_t)a->qkv) % 16 == 0, "flash_attn: qkv pitch/alignment");
        RB_REQUIRE(a->ld_out >= dim && (a->ld_out * 2) % 16 == 0 && ((uintptr_t)a->out) % 16 == 0, "flash_attn: out pitch/alignment");
        RB_REQUIRE(a->batch > 0 && a->batch <= 65535 && a->n_tokens > 0, "flash_attn: bad batch / token count");
        // [batch, tokens, 3 * dim] with boxes of 64 tokens x 64 columns, 128B-swizzled: one plane (hi) or two (hi, lo)
        cuuint64_t dims[3] = {(cuuint64_t)(3 * dim), (cuuint64_t)a->n_tokens, (cuuint64_t)a->batch};
        cuuint64_t strides[2] = {(cuuint64_t)a->ld_qkv * 2, (cuuint64_t)a->ld_qkv * 2 * (cuuint64_t)a->n_tokens};
        cuuint32_t box[3] = {64, 64, 1};
        CUtensorMap map_hi, map_lo;
        if (encode_tiled(&map_hi, "flash_attn", tma_dtype(a->dtype), 3, a->qkv, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B)) return 1;
        map_lo = map_hi;
        if (split && encode_tiled(&map_lo, "flash_attn (lo plane)", tma_dtype(a->dtype), 3, a->qkv_lo, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
            return 1;
        FaParams p;
        p.out = a->out; p.out_lo = a->out_lo; p.ldo = a->ld_out; p.N = a->n_tokens; p.heads = a->heads; p.dim = dim;
        p.scale_log2 = 1.4426950408889634f / sqrtf((float)a->head_dim);
        if constexpr (std::is_same_v<T, __half>)
            if (split) return launch_fa<64, __half, true>(map_hi, map_lo, p, a->batch, st);
        return a->head_dim == 64 ? launch_fa<64, T, false>(map_hi, map_lo, p, a->batch, st) : launch_fa<128, T, false>(map_hi, map_lo, p, a->batch, st);
    });
}
