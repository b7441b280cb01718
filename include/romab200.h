/*
 * romab200.h — C ABI of the H100-native RoMa dense-matching kernels (libromab200.so).
 *
 * Drop-in boundary for ONE path: RoMa's dense match()/sample() inference.  The reference
 * (Parskatt/RoMa) is pure Python/PyTorch; the only native operator boundary it has on this path is
 * the optional third-party wheel `local_corr.local_corr` (romatch/utils/local_correlation.py:22-35).
 * Every entry point below cites the reference code it replaces.  Conventions:
 *
 *   - plain pointers and sizes only (no torch types); every pointer is DEVICE memory owned by the
 *     caller (PyTorch's allocator in the host package); nothing is allocated or synchronised inside;
 *   - every call enqueues work on the given CUDA stream (a `cudaStream_t` passed as void*) and returns
 *     immediately: 0 = ok, non-zero = error, message via romab200_last_error() (thread-local);
 *   - activations are channels-last ("NHWC"): a [B,H,W,C] map is a row-major [B*H*W, C] matrix with an
 *     explicit row pitch, so 1x1 convolutions and Linear layers are the same GEMM;
 *   - dtypes: RB_F32 / RB_F16 / RB_BF16; accumulation is always fp32.  An entry point refuses a dtype code it has no kernel
 *     for, before any CUDA call: non-zero return, message "<op>: unsupported dtype <code>".
 *   - RB_F64 exists for the float64 evaluation geometry only (romab200_warp_kpts and its two siblings, which take float32 or
 *     float64 depth maps and points and compute in float64); every other entry point refuses it like any code it has no kernel for.
 *   - RB_F16S ("split fp16 pair") is the storage format of the tensor-core parity mode: a matrix is held as TWO fp16
 *     planes of the same pitch, hi = fp16(x) and lo = fp16((x - hi) * 2^11), value = hi + lo * 2^-11: 22 significand bits
 *     with the exponent range of fp16 (the reference's own CUDA autocast range).  romab200_gemm contracts such operands
 *     with three wgmma MMAs per k-step (hi.hi + 2^-11 (hi.lo + lo.hi), fp32 accumulation in registers), which reproduces an
 *     fp32 GEMM to ~2^-22 relative; arguments named *_lo carry the second plane.
 */
#ifndef ROMAB200_H
#define ROMAB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ROMAB200_ABI_VERSION 4

enum rb_dtype { RB_F32 = 0, RB_F16 = 1, RB_BF16 = 2, RB_F16S = 3, RB_F64 = 4 };
enum rb_act { RB_ACT_NONE = 0, RB_ACT_RELU = 1, RB_ACT_GELU = 2 };
enum rb_rowmap { RB_ROWMAP_NONE = 0, RB_ROWMAP_PAD_KEEP = 1, RB_ROWMAP_PAD_TO_COMPACT = 2, RB_ROWMAP_SEGMENT = 3 };
enum rb_epi { RB_EPI_LINEAR = 0, RB_EPI_COSKERNEL = 1 };
enum rb_backend { RB_BACKEND_AUTO = 0, RB_BACKEND_SIMT = 1, RB_BACKEND_TCGEN05 = 2 };

int romab200_abi_version(void);
const char* romab200_last_error(void);
/* number of CUDA kernels this library has launched so far in this process */
unsigned long long romab200_launch_count(void);
/* 1 if the running device is sm_90 (H100) and the wgmma/TMA kernels may be launched */
int romab200_device_ok(void);

/* ------------------------------------------------------------------------------------------------
 * GEMM with fused epilogue:  C[m,n] = epi( sum_k A[m + tap(k), k] * B[n,k] )
 *
 * Replaces every nn.Linear / 1x1 nn.Conv2d (+ folded BatchNorm) / 3x3 nn.Conv2d on the path:
 *   ViT + decoder Linear layers      romatch/models/transformer/layers/{attention.py:50-63,mlp.py:35-41}
 *   proj[s] 1x1 conv + BN            romatch/models/model_zoo/roma_models.py:156-169 (matcher.py:441-450)
 *   ConvRefiner pointwise convs      romatch/models/matcher.py:121 (create_block conv2)
 *   VGG19-BN 3x3 conv + BN + ReLU    romatch/models/encoders.py:17-27 (as a 9-tap shifted GEMM on a
 *                                    zero-padded NHWC map: tap t reads rows m + tap_rows[t])
 *   CosKernel all-pairs contraction  romatch/models/matcher.py:191-200 (RB_EPI_COSKERNEL)
 *   attention QK^T / PV, GP K_xy@alpha, Cholesky trailing updates (batched, strided)
 *
 * A: [M, K] row-major (pitch lda).  B: [N, K] row-major (pitch ldb), or [K, N] when trans_b != 0.
 * K = ntaps * k_per_tap; element k belongs to tap k / k_per_tap and reads A row m + tap_rows[tap]
 * (rows outside [0, a_rows) read as zero).  Batching: grid over batch0 x batch1 with element strides.
 *
 * Epilogue RB_EPI_LINEAR:    v = alpha*acc + bias[n]; v = act(v); v *= col_scale[n]; v += R[m,n]
 * Epilogue RB_EPI_COSKERNEL: c = acc * s(m,n), s = 1/(na[m]*nb[n]+eps)            (cos_normalized == 0)
 *                                              s = na[m]*nb[n]/(na[m]*nb[n]+eps)  (operands pre-normalised)
 *                            v = exp((c - 1) * inv_t) + (m == n ? diag_add : 0)
 * Row map of the store: NONE; PAD_KEEP (m indexes a zero-padded [*,pad_h,pad_w] grid; border rows are not
 * computed: they are left alone or rewritten with zeros, the value they hold in every map of the path); PAD_TO_COMPACT (same, interior rows are written to the un-padded row index);
 * SEGMENT (row m -> (m / seg_in) * seg_out + m % seg_in + seg_off).
 * Output pitch: when ldc (and the batch strides) are multiples of 16 bytes, the row map is NONE or PAD_KEEP and there is no
 * residual operand, the tensor-core back-end also writes zeros into the pad columns N .. roundup(N, 16 bytes) of every written row
 * (columns beyond are untouched).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    const void* A; const void* B; void* C;
    int32_t M, N, K;
    int64_t lda, ldb, ldc;
    int32_t dtype_ab, dtype_c;
    int32_t trans_b;
    int32_t batch0, batch1;
    int64_t sa0, sa1, sb0, sb1, sc0, sc1;
    int32_t ntaps; int32_t tap_rows[9]; int64_t a_rows;
    float alpha;
    const float* bias; const float* col_scale;
    const void* R; int64_t ldr, sr0, sr1; int32_t dtype_r;
    int32_t act;
    int32_t epi;
    const float* norm_a; const float* norm_b; int64_t sna0, snb0;
    float eps, inv_t, diag_add; int32_t cos_normalized;
    int32_t rowmap, pad_h, pad_w, seg_in, seg_out, seg_off;
    int32_t backend;
    /* second planes of RB_F16S operands / output (dtype_ab == RB_F16S: A_lo and B_lo, same geometry as A and B;
       dtype_c == RB_F16S: C_lo, same pitch as C); NULL otherwise */
    const void* A_lo; const void* B_lo; void* C_lo;
    /* tensor-core back-end: upper bound on the persistent grid (0 = one CTA per SM).  A GEMM running on a side stream beside a chain of short
       dependent kernels (the GP solve) leaves the remaining SMs free, so that those kernels start without waiting for a whole GEMM. */
    int32_t max_ctas;
} rb_gemm_args;
int romab200_gemm(const rb_gemm_args* args, void* stream);

/* LayerNorm over the last dim (nn.LayerNorm in block.py:50 / dinov2.py:88): y = (x-mu)/sqrt(var+eps)*g + b */
typedef struct {
    const void* x; void* y; const float* gamma; const float* beta;
    int64_t rows; int32_t cols; int64_t ldx, ldy; int32_t dtype_x, dtype_y; float eps;
    void* y_lo;   /* second plane when dtype_y == RB_F16S */
} rb_layernorm_args;
int romab200_layernorm(const rb_layernorm_args* args, void* stream);

/* Row softmax of attention scores: s = softmax(scale * s) over `cols` (SDPA, attention.py:59); in place, or (out_hi != NULL,
 * dtype RB_F32) written as an RB_F16S pair of planes [rows, ldo] for the split-fp16 PV product (pad columns receive 0) */
typedef struct { void* s; int64_t rows; int32_t cols; int64_t lds; int32_t dtype; float scale;
                 void* out_hi; void* out_lo; int64_t ldo; } rb_softmax_args;
int romab200_softmax_rows(const rb_softmax_args* args, void* stream);

/* Fused attention forward (F.scaled_dot_product_attention, attention.py:50-63), 16-bit tensor-core path:
 * qkv [batch, n_tokens, ld_qkv] holds q | k | v (each heads*head_dim wide, heads contiguous); out [batch, n_tokens, ld_out].
 * out[b, i, h*d:(h+1)*d] = softmax_j(q_i . k_j / sqrt(d)) v_j.  head_dim 64 or 128. */
typedef struct {
    const void* qkv; void* out; int64_t ld_qkv, ld_out; int32_t batch, n_tokens, heads, head_dim, dtype;
    /* dtype == RB_F16S (head_dim 64): qkv and out are split-fp16 pairs, these are their second planes; fp32-class result */
    const void* qkv_lo; void* out_lo;
} rb_flash_attn_args;
int romab200_flash_attn(const rb_flash_attn_args* args, void* stream);

/* L2 norm of every row: out[r] = ||x[r,:]||  (CosKernel, matcher.py:192-194) */
typedef struct { const void* x; float* out; int64_t rows; int32_t cols; int64_t ldx; int32_t dtype; } rb_rownorm_args;
int romab200_row_norms(const rb_rownorm_args* args, void* stream);

/* Strided 2-D copy / cast: dst[r, c] = (dst_dtype) src[r, c] * scale[r]  (scale may be NULL) */
typedef struct {
    const void* src; void* dst; int64_t rows; int32_t cols; int64_t lds, ldd; int32_t dtype_src, dtype_dst;
    const float* row_scale; int32_t row_scale_reciprocal;
} rb_copy2d_args;
int romab200_copy2d(const rb_copy2d_args* args, void* stream);

/* Indexed copy of whole rows of bytes: for i < count, row dst_index[i] of dst = row src_index[i] of src (a NULL index stands
 * for i).  Rows are row_bytes long and ld_src / ld_dst bytes apart; row_bytes, both pitches and both pointers are multiples of
 * 16.  An index outside [0, src_rows) or [0, dst_rows) leaves its destination row unwritten.  The indices are read on the
 * device, so a captured graph of the call replays for any index list of the same count (match_pairs: images between a
 * per-image feature bank and the batch buffers of the encoders and of the pair stage). */
typedef struct {
    const void* src; void* dst; const int32_t* src_index; const int32_t* dst_index;
    int32_t count; int64_t row_bytes, ld_src, ld_dst; int32_t src_rows, dst_rows;
} rb_gather_rows_args;
int romab200_gather_rows(const rb_gather_rows_args* args, void* stream);

/* fp16 hi/lo operand split for fp32-class accuracy on the f16 tensor pipe:
 * dst[r, 0:C] = hi, dst[r, C:2C] = lo (or hi), dst[r, 2C:3C] = hi (or lo) of x[r,:]/scale[r]
 * layout A: [hi | lo | hi], layout B: [hi | hi | lo]  so that A'.B'^T = hi.hi + lo.hi + hi.lo */
typedef struct {
    const float* x; void* dst; int64_t rows; int32_t cols; int64_t ldx, ldd; const float* row_norm;
    int32_t layout_b;
} rb_split_args;
int romab200_split_f16x3(const rb_split_args* args, void* stream);

/* fp32 matrix -> RB_F16S planes: hi[r,c] = fp16(v), lo[r,c] = fp16((v - hi) * 2^11), v = x[r,c] (/ row_norm[r] if given).
 * The producer of every split-fp16 GEMM operand that is not written in that format by its own kernel. */
typedef struct {
    const float* x; void* hi; void* lo; int64_t rows; int32_t cols; int64_t ldx, ldd; const float* row_norm;
} rb_split_pair_args;
int romab200_split_f16s(const rb_split_pair_args* args, void* stream);

/* ---- VGG19-BN pieces that are not GEMMs (encoders.py:17-27) ------------------------------------ */
/* First conv (3 -> 64) + folded BN + ReLU, NCHW fp32 image -> zero-padded NHWC [B,H+2,W+2,64] */
typedef struct {
    const float* image; void* out; const float* weight /* [64][27] folded */; const float* bias /* [64] */;
    int32_t batch, height, width, cout; int32_t dtype_out;
    void* out_lo;   /* second plane when dtype_out == RB_F16S */
} rb_conv_first_args;
int romab200_conv3x3_first(const rb_conv_first_args* args, void* stream);
/* 2x2/2 max-pool between zero-padded NHWC maps: [B,H+2,W+2,C] -> [B,H/2+2,W/2+2,C] */
typedef struct { const void* in; void* out; int32_t batch, height, width, channels, dtype;
                 const void* in_lo; void* out_lo; /* second planes when dtype == RB_F16S */ } rb_maxpool_args;
int romab200_maxpool2x2_padded(const rb_maxpool_args* args, void* stream);

/* ---- DINOv2 tokenisation (dinov2.py:192-201, patch_embed.py:69-82) ------------------------------ */
/* im2col of non-overlapping 14x14 patches: NCHW fp32 image -> [B*hp*wp, ldo] rows of (c,ky,kx) */
typedef struct { const float* image; void* out; int32_t batch, height, width, patch; int64_t ldo; int32_t dtype_out; } rb_im2col_args;
int romab200_im2col_patch(const rb_im2col_args* args, void* stream);
/* tokens[b,0,:] = cls + pos[0]; tokens[b,1+p,:] = patch[b,p,:] + pos[1+p]   (fp32 residual stream) */
typedef struct { const float* patch; const float* cls; const float* pos; float* tokens; int32_t batch, npatch, dim; } rb_tokens_args;
int romab200_assemble_tokens(const rb_tokens_args* args, void* stream);

/* ---- GP posterior (matcher.py:291-323): batched Cholesky + solves --------------------------------
 * W is a batch of workspaces [n + nrhs, n] (row-major, pitch ldw): rows 0..n-1 hold the SPD matrix
 * K_yy + sigma*I (lower triangle is read), rows n.. hold F^T ([nrhs, n]).  On return rows n.. hold
 * X^T where (K_yy + sigma I) X = F, i.e. alpha^T, ready to be the [N,K] operand of mu = K_xy @ alpha.
 * With algo 0 and 2 the lower triangle of rows 0..n-1 holds the Cholesky factor afterwards; the strict upper triangle is
 * unspecified (symmetric trailing updates only maintain the lower half).
 * Replaces torch.linalg.cholesky + torch.cholesky_solve (matcher.py:307-308). */
typedef struct {
    float* W; int32_t n, nrhs, batch; int64_t ldw, stride;
    void* workspace; int64_t workspace_bytes;
    int32_t algo;   /* 0: 32-wide panels, chain of small launches (no workspace)
                       1: the same as ONE cooperative persistent kernel; workspace >= (batch*ceil(n/32)*1024 + 1)*4 bytes
                       2: 128-wide blocks factored in shared memory with explicit block inverses, all O(n^2) work as K=128
                          GEMMs; workspace >= batch*ceil(n/128)*65536 bytes (receives the diagonal-block inverses)
                       3: the schedule of 2 with those GEMMs on the tensor cores (split-fp16 operand pairs, fp32-class; the symmetric
                          trailing update is an in-place TMA reduce-add); ldw % 8 == 0, stride % 8 == 0; workspace >=
                          batch * (ceil(n/128)*65536 + 4*max((n+nrhs)*128 + 16384, nrhs*128 + 16384 + 128*ldw)) bytes */
} rb_gp_solve_args;
int romab200_gp_solve(const rb_gp_solve_args* args, void* stream);
/* ---- classifier head -> coarse flow (utils.py:300-322) ------------------------------------------
 * logits [rows, ldl] fp32/16 with 4096 anchor logits followed by the certainty logit; writes
 * state[row] = (flow_x, flow_y, certainty_logit). */
typedef struct { const void* logits; float* state; int64_t rows; int64_t ldl; int32_t res; int32_t dtype; } rb_cls_args;
int romab200_cls_to_flow_refine(const rb_cls_args* args, void* stream);

/* ---- ConvRefiner (matcher.py:124-179) ------------------------------------------------------------
 * feat: projected features of all encoder images [n_img, h, w, ldf] (channels-last, `cf` channels).
 * For decoder item i the query image is `i` and the support image is (i + y_shift) % n_img.
 * state: [D, h, w, 3] = (flow_x, flow_y, certainty_logit) fp32.
 * prologue writes d[D,h,w,ldd] = [x | grid_sample(y, flow) | disp_emb(40/32*sf*(flow-grid)) | local_corr | 0-pad]
 *   (matcher.py:132-168; local correlation per local_correlation.py:77-142 / local_corr.local_corr) */
typedef struct {
    const void* feat; int64_t ldf; int32_t n_img, y_shift;
    const float* state; void* d; int64_t ldd;
    int32_t D, h, w, cf, emb, radius; int32_t dtype;
    const float* emb_weight /* [emb][2] */; const float* emb_bias; float disp_scale;
    const float* grid_x; const float* grid_y;   /* linspace(-1+1/w, 1-1/w, w), linspace(-1+1/h, 1-1/h, h) (matcher.py:136-143) */
    const float* win_x; const float* win_y;     /* linspace(-2r/w, 2r/w, 2r+1), linspace(-2r/h, 2r/h, 2r+1) (local_correlation.py:93-103) */
    /* optional workspace (caller-owned, like every buffer): one byte per tile of the tile-cooperative pass for fp32 maps with a local
     * correlation (radius 7: 8x2 pixels (x by y), radius 3 / 2: 8x4 pixels per tile; D * ceil(h/Ty) * ceil(w/Tx) tiles).  When given, tiles whose
     * windows overlap (coherent flow) are produced by one CTA from a shared-memory copy of the union of their windows; the rest by the
     * per-pixel kernel.  NULL: per-pixel kernel only.  Same results either way up to the summation order of the dot products. */
    void* tile_done; int32_t tile_done_len;
    /* optional all-pairs table (radius > 0): corr_table[(item*h*w + p) * ld_corr_table + q] = <x[item, p, :], y[item, q, :]> / sqrt(cf) for every
     * position q of the other map, e.g. one romab200_gemm per direction at the coarsest scale, where the table is small (h*w = 1600) and the
     * contraction is the one the GP kernel matrix performs anyway (matcher.py:298-300).  The window dot products then are a gather of
     * (2r+2)^2 table entries per pixel instead of (2r+2)^2 * cf multiply-adds.  NULL: the dot products are computed here. */
    const float* corr_table; int64_t ld_corr_table;
} rb_refiner_prologue_args;
int romab200_refiner_prologue(const rb_refiner_prologue_args* args, void* stream);

/* Stand-alone local correlation with the reference wheel's semantics (local_correlation.py:22-35):
 * corr[b, p, k] = sum_c f0[b,p,c] * bilinear(f1[b], flow[b,p] + window[k])  (f0 already scaled by caller or
 * `scale` applied here), zero padding, k = (dy+r)*(2r+1) + (dx+r).  out pitch ldo (channels-last slice). */
typedef struct {
    const void* f0; const void* f1; int64_t ldf0, ldf1; int64_t f0_img_stride, f1_img_stride;
    const float* flow; int64_t ldflow; void* out; int64_t ldo;
    int32_t batch, h, w, c, radius; float scale; int32_t dtype_f, dtype_out;
    int32_t n_img, y_shift;   /* f1 image of item i = (i + y_shift) % n_img ; f0 image = i */
    const float* win_x; const float* win_y;   /* window offsets in normalised coordinates, 2r+1 each */
} rb_local_corr_args;
int romab200_local_corr(const rb_local_corr_args* args, void* stream);

/* The fused-local-corr wheel's operator, signature for signature (`local_corr.local_corr`, local_correlation.py:22-35):
 * out[b, p, k] = sum_c f0[b, p, c] * sample(f1[b], warp[b, p, k, :]), sample = bilinear (mode 0) or nearest (mode 1) lookup at the
 * normalised (x, y) position, align_corners=False, zero padding (grid_sample semantics); f0 is used as given (the caller pre-scales
 * by 1/sqrt(C) like `local_corr_wrapper` does).  f0 [B, HW, C] fp32 (pitch ldf0), f1 [B, H, W, C] fp32 channels-last (pitch ldf1),
 * warp [B, HW, K, 2] fp32 contiguous, out [B, HW, K] fp32 contiguous.  Arbitrary warps: nothing is assumed about a window lattice. */
typedef struct {
    const float* f0; const float* f1; int64_t ldf0, ldf1; const float* warp; float* out;
    int32_t batch, h, w, c, k; int32_t mode;
} rb_local_corr_warp_args;
int romab200_local_corr_warp(const rb_local_corr_warp_args* args, void* stream);

/* depthwise 5x5 conv (pad 2) + folded BN + ReLU on channels-last maps (create_block conv1+norm+relu,
 * matcher.py:106-120).  weight [25][ldw] fp32 (tap-major), bias [C] */
typedef struct {
    const void* in; void* out; int64_t ldi, ldo; const float* weight; int64_t ldw; const float* bias;
    int32_t batch, h, w, c; int32_t dtype;
    void* out_lo;   /* dtype == RB_F32 only: when non-NULL the result is written as an RB_F16S pair (out = hi plane, out_lo =
                       lo plane, pitch ldo in fp16 elements) so that the pointwise GEMM can consume it directly */
} rb_dwconv_args;
int romab200_dwconv5x5_relu(const rb_dwconv_args* args, void* stream);

/* Fused thin-map ConvRefiner block (C = 24, stride-1 maps): out = PW(ReLU(BN(DW5x5(in)))) in one pass.
 * in/out: channels-last 16-bit maps [batch, h, w, ld] (in != out); dw_weight [25][ldw] fp32 tap-major (BN folded), device.
 * pw_weight_host [c][c] fp32 row-major and pw_bias_host [c] are HOST arrays: the pointwise weights are passed to the
 * kernel as launch parameters (constant bank), they are read during this call only.  (create_block, matcher.py:92-122) */
typedef struct {
    const void* in; void* out; int64_t ld; const float* dw_weight; int64_t ldw; const float* dw_bias;
    const float* pw_weight_host; const float* pw_bias_host; int32_t batch, h, w, c; int32_t dtype;
} rb_refiner_block_small_args;
int romab200_refiner_block_small(const rb_refiner_block_small_args* args, void* stream);

/* Fused ConvRefiner block for the stride-2 maps (C = 144): depthwise 5x5 + BN + ReLU on the CUDA cores feeding a
 * wgmma pointwise GEMM whose weights stay resident in shared memory; one read + one write of the map.
 * in/out [batch, h, w, ld] 16-bit (in != out); dw_weight [25][ldw] fp32 (BN folded), pw_weight [144][ld_pw] 16-bit. */
typedef struct {
    const void* in; void* out; int64_t ld; const float* dw_weight; int64_t ldw; const float* dw_bias;
    const void* pw_weight; int64_t ld_pw; const float* pw_bias; int32_t batch, h, w, c; int32_t dtype;
} rb_refiner_block_c144_args;
int romab200_refiner_block_c144(const rb_refiner_block_c144_args* args, void* stream);

/* The same block in the parity mode: fp32 maps, split-fp16 pointwise GEMM.  Bit-identical to romab200_dwconv5x5_relu (fp32 in,
 * RB_F16S out) followed by romab200_gemm (RB_F16S operands, fp32 out, bias), with the RB_F16S intermediate kept on chip.
 * in/out [batch, h, w, ld] fp32 (in != out; ld % 8 == 0, ld >= 144); dw_weight [25][ldw] fp32 (BN folded);
 * pw_weight / pw_weight_lo: the hi / lo fp16 planes of the RB_F16S weights [144][ld_pw] (ld_pw % 8 == 0, ld_pw >= 144);
 * all pointers 16-byte aligned. */
typedef struct {
    const float* in; float* out; int64_t ld; const float* dw_weight; int64_t ldw; const float* dw_bias;
    const void* pw_weight; const void* pw_weight_lo; int64_t ld_pw; const float* pw_bias; int32_t batch, h, w, c;
} rb_refiner_block_c144_split_args;
int romab200_refiner_block_c144_split(const rb_refiner_block_c144_split_args* args, void* stream);

/* out_conv (fp32 1x1, C -> 3) + flow/certainty update (matcher.py:177-179, 496-506):
 * state[...,0] += scale_x * o0 ; state[...,1] += scale_y * o1 ; state[...,2] += o2 */
typedef struct {
    const void* d; int64_t ldd; const float* weight /* [3][ldw] */; int64_t ldw; const float* bias;
    float* state; int64_t rows; int32_t c; float scale_x, scale_y; int32_t dtype; float* delta_out /* optional [rows,3] */;
} rb_refiner_tail_args;
int romab200_refiner_tail(const rb_refiner_tail_args* args, void* stream);

/* bilinear resize, align_corners=False, no antialias (F.interpolate, matcher.py:424-435,513-523) of a
 * channels-last fp32 map [B, hi, wi, c] -> [B, ho, wo, c] */
typedef struct { const float* in; float* out; int32_t batch, hi, wi, ho, wo, c; } rb_resize_args;
int romab200_bilinear_resize(const rb_resize_args* args, void* stream);

/* match() epilogue (matcher.py:839-850, 891-927): certainty attenuation by the stride-16 logit, sigmoid,
 * out-of-range mask, clamp, identity grids and the symmetric concat.
 * state [D,H,W,3]; coarse_state [D,hc,wc,3] = the stride-16 state (NULL = no attenuation); warp [b,H,W*(sym?2:1),4]; cert [b,H,W*(sym?2:1)] */
typedef struct {
    const float* state; const float* coarse_state; int32_t hc, wc;
    float* warp; float* cert; int32_t b, H, W, symmetric;
    const float* grid_x; const float* grid_y;   /* pixel-centre linspaces of length W and H (matcher.py:904-912) */
} rb_match_epilogue_args;
int romab200_match_epilogue(const rb_match_epilogue_args* args, void* stream);

/* sample(): Gaussian KDE density (kde.py:4-12) without materialising the NxN matrix.
 * x [n,4] fp32; density[i] = sum_j exp(-||h(x_i)-h(x_j)||^2 / (2 std^2)), h = fp16 rounding when half != 0 */
typedef struct { const float* x; float* density; int32_t n; float std; int32_t half;
                 /* optional: workspace of splits * n floats; the j range is then cut into `splits` parts summed in a fixed order by a second
                  * kernel (more CTAs than SMs for the 40000-point problem of sample()).  NULL / splits <= 1: one pass */
                 float* workspace; int32_t splits;
                 /* half mode only: evaluate the block pairs (I, J >= I) of 256 x 256 points once and credit both the row and the column sums
                  * (exp(-d2) is symmetric); workspace of (splits + ceil(n / 256)) * n floats, its size in workspace_floats.  0: every pair twice */
                 int32_t symmetric; int64_t workspace_floats;
                 /* batch > 1: `batch` independent problems of n points (the per-item KDE of a batched sample(), matcher.py:598-629,
                  * tiny.py:234-266): item b reads x + b*4n, writes density + b*n and uses its own slice of the workspace (splits * n, or
                  * (splits + ceil(n/256)) * n floats in the symmetric schedule; workspace_floats covers all items).  Every item runs the
                  * schedule of a single call of size n, so its densities equal that call's bit for bit.  0 or 1: one problem */
                 int32_t batch; } rb_kde_args;
int romab200_kde_density(const rb_kde_args* args, void* stream);

/* sample(): weighted sampling WITHOUT replacement on the device (the two torch.multinomial draws of matcher.py:613-617, 626-628).
 * For every batch item b: draws k distinct indices i in [0, n) with probabilities proportional to w_i = T(values[b*stride + i]),
 *   T = identity (RB_SAMPLE_IDENTITY), certainty thresholding `v > param ? 1 : v` (RB_SAMPLE_THRESHOLD, matcher.py:604-607), or density
 *   balancing `v < 10 ? 1e-7 : 1/(v+1)` of a KDE density v (RB_SAMPLE_BALANCE, matcher.py:622-625),
 * by an exponential race (key = -log(u)/w, k smallest keys; Philox4x32-10 keyed by `seed`, counter = element index).  out_idx [batch, k]
 * int32 in no particular order; out_weights (optional) [batch, k] receives the transformed weights of the drawn items; keys = workspace of
 * batch * n floats, scratch = workspace of batch * 2056 int32.  Items of zero weight are only drawn when fewer than k positive weights exist. */
enum rb_sample_transform { RB_SAMPLE_IDENTITY = 0, RB_SAMPLE_THRESHOLD = 1, RB_SAMPLE_BALANCE = 2 };
typedef struct {
    const float* values; int64_t n; int32_t k; int32_t batch; int64_t stride; uint64_t seed; int32_t transform; float param;
    int32_t* out_idx; float* out_weights; float* keys;
    void* scratch;   /* batch * 2056 * 4 bytes: histograms and selection state (cleared inside the call) */
    const uint64_t* seed_dev;   /* optional: the seed is read from this DEVICE word instead of `seed` (CUDA-graph replays with fresh seeds) */
    /* Batches of independent sample() calls (matcher.py:598-629, tiny.py:234-266 run once per item):
     *   seed_stride > 0 (needs seed_dev): item b reads its own seed seed_dev[b * seed_stride] and keys Philox with it alone, so it draws
     *     exactly what a batch-1 call with that seed draws; 0: every item shares one seed and b is mixed into the Philox key;
     *   repeats > 1: item b draws from values + (b / repeats) * stride, so the `repeats` draws of one pair read one map; 0 or 1: row b. */
    int64_t seed_stride; int32_t repeats;
} rb_sample_args;
int romab200_weighted_sample(const rb_sample_args* args, void* stream);

/* The row gathers of sample() after each draw (matches[sel], certainty[sel] and the certainty threshold, matcher.py:604-617, 626-629,
 * tiny.py:240-266), for `items` draws at once: for item i and j < k, with p = i / repeats (0 or 1 repeats: p = i) and r = idx[i*k + j],
 *   out_matches[i*k + j] = matches[p*n + r] (4 floats)   out_certainty[i*k + j] = threshold && c > thresh ? 1 : c,  c = certainty[p*n + r].
 * matches [pairs, n, 4] and out_matches 16-byte aligned; idx [items, k] int32 (the drawn indices, sorted per item by the caller). */
typedef struct {
    const float* matches; const float* certainty; int64_t n;
    const int32_t* idx; int32_t items, k, repeats;
    int32_t threshold; float thresh;
    float* out_matches; float* out_certainty;
} rb_sample_gather_args;
int romab200_sample_gather(const rb_sample_gather_args* args, void* stream);

/* Image preprocessing in front of match() on the device: RGB uint8 image -> normalised fp32 [3, out_h, out_w]
 * (get_tuple_transform_ops(resize=(h, w), normalize=True), utils.py:164-173 = PIL.Image.resize((w, h), BICUBIC), /255, ImageNet mean/std;
 * called at matcher.py:812-815, 855-866).  Bit-exact with Pillow's 8-bit resampling (src/libImaging/Resample.c: 22-bit fixed-point weights,
 * horizontal pass into a uint8 image, then the vertical pass) and with the reference's fp32 operation order.
 *
 * romab200_resample_coeffs is HOST-ONLY arithmetic (no CUDA call, `stream` ignored): the weight table of one axis for in_size -> out_size,
 * bounds [out_size][2] = (first input sample, count), kk [out_size][ksize] zero-padded rows.  Call it with kk = bounds = NULL to get *ksize
 * first.  The tables depend on the two sizes only; keep device copies per size pair. */
typedef struct { int32_t in_size, out_size; int32_t* bounds; int32_t* kk; int32_t* ksize; } rb_resample_coeffs_args;
int romab200_resample_coeffs(const rb_resample_coeffs_args* args, void* stream);

typedef struct {
    const uint8_t* in; int64_t ld_in /* bytes per row */; int32_t in_h, in_w;   /* interleaved RGB, 3 bytes per pixel */
    int32_t out_h, out_w;
    const int32_t* bounds_x; const int32_t* kk_x; int32_t ksize_x;   /* DEVICE tables for in_w -> out_w (ignored when out_w == in_w) */
    const int32_t* bounds_y; const int32_t* kk_y; int32_t ksize_y;   /* DEVICE tables for in_h -> out_h (ignored when out_h == in_h) */
    uint8_t* tmp;      /* in_h * out_w * 3 bytes: the horizontally resampled image (unused when out_w == in_w) */
    uint8_t* out_u8;   /* optional [out_h, out_w, 3]: the resized 8-bit image, what PIL.Image.resize returns */
    float* out;        /* optional [3, out_h, out_w]: (u8 / 255 - mean) / std */
    float mean[3]; float std[3];
} rb_preprocess_args;
int romab200_preprocess_rgb8(const rb_preprocess_args* args, void* stream);

/* transpose a batched strided 2-D matrix: dst[b][c][r] = src[b][r][c]  (V^T for the PV product) */
typedef struct {
    const void* src; void* dst; int32_t rows, cols; int64_t lds, ldd; int32_t batch0, batch1;
    int64_t ss0, ss1, sd0, sd1; int32_t dtype;
} rb_transpose_args;
int romab200_transpose(const rb_transpose_args* args, void* stream);

/* ---- match_keypoints (matcher.py:743-762): grid samples at the keypoints + mutual nearest neighbours in O(N_A + N_B) memory ----
 * romab200_keypoints_sample replaces the two F.grid_sample calls (matcher.py:743-754):
 *   x_to_B[i] = grid_sample(warp[..., 0:2], x[i]), cert_out[i] = grid_sample(cert, x[i]); bilinear, zero padding, align_corners=False,
 *   ATen's unnormalisation ((x + 1) * size - 1) / 2; a NaN position gives NaN.  x [n, 2] fp32 contiguous (normalised (x, y));
 *   warp: element (y, x, c) of the two sampled channels at warp[y * warp_ld_row + x * warp_ld_px + c * warp_ld_ch] (strides in floats,
 *   so views such as the A half of a symmetric warp are read in place); cert: element (y, x) at cert[y * cert_ld_row + x * cert_ld_px];
 *   x_to_B [n, 2], cert_out [n]. */
typedef struct {
    const float* x; int32_t n;
    const float* warp; int32_t warp_h, warp_w; int64_t warp_ld_row, warp_ld_px, warp_ld_ch;
    const float* cert; int32_t cert_h, cert_w; int64_t cert_ld_row, cert_ld_px;
    float* x_to_B; float* cert_out;
} rb_keypoints_sample_args;
int romab200_keypoints_sample(const rb_keypoints_sample_args* args, void* stream);

/* romab200_keypoints_mnn_count + romab200_keypoints_mnn_emit replace torch.cdist and the mutual-nearest-neighbour nonzero
 * (matcher.py:755-762) without an N_A x N_B buffer.  With D[i, j] = sqrt_rn(dx*dx + dy*dy), dx = x_A_to_B[i].x - x_B[j].x (every
 * operation rounded to fp32, no FMA contraction: the exact-difference distance), the pair (i, j) is a match iff
 *   D[i,j] == min_j' D[i,j'] && D[i,j] == min_i' D[i',j] && cert_A[i] > cert_th && D[i,j] < max_dist,
 * minima with torch.min's NaN propagation (a NaN anywhere in a row or column leaves it without matches); ties are all kept.
 * x_A_to_B [n_a, 2], cert_A [n_a], x_B [n_b, 2] fp32 contiguous; n_a, n_b > 0.
 * workspace: >= (16 + 1) * (n_a + n_b) floats; it holds the row and column minima between the two calls (pass it unchanged).
 * count: offsets [n_a + 1] int64 receives the exclusive prefix sums of the per-row match counts, offsets[n_a] = number of matches.
 * emit (after the caller has read offsets[n_a] and sized the outputs): inds_A, inds_B [offsets[n_a]] int64 receive the matches in
 * row-major order (i ascending, then j), the order of torch.nonzero.  Deterministic. */
typedef struct {
    const float* x_A_to_B; const float* cert_A; const float* x_B; int32_t n_a, n_b;
    float cert_th, max_dist;
    float* workspace; int64_t workspace_floats;
    int64_t* offsets;
    int64_t* inds_A; int64_t* inds_B;   /* emit only */
} rb_keypoints_mnn_args;
int romab200_keypoints_mnn_count(const rb_keypoints_mnn_args* args, void* stream);
int romab200_keypoints_mnn_emit(const rb_keypoints_mnn_args* args, void* stream);

/* ---- TinyRoMa (romatch/models/tiny.py), fp32 throughout like the reference ------------------------ */
/* Direct convolution on channels-last fp32 maps, CUDA-core FFMA (the XFeat backbone convs, tiny.py:87-97, and the
 * BasicLayer / 1x1 heads of the coarse and fine matchers, tiny.py:47-61,208-215):
 *   out[b,y,x,n] = epi( sum_{ky,kx,c} in[b, y*stride+ky-k/2, x*stride+kx-k/2, c] * weight[(ky*k+kx)*cin + c][n] ),
 * zero padding k/2, epi(v) = ((v + bias[n]) -> ReLU if relu) * col_scale[n] + R[b,y,x,n]  (bias / col_scale / R optional: NULL).
 * weight [k*k*cin][ldw] fp32 (BN folded), ldw a multiple of 4 >= cout with zero columns beyond cout; k in {1,3}, stride in {1,2}.
 * in [B,hi,wi,ldi], out / R [B,ho,wo,ldo / ldr]; ho = (hi - 1) / stride + 1, wo = (wi - 1) / stride + 1 (nn.Conv2d with padding k/2). */
typedef struct {
    const float* in; float* out; const float* weight; const float* bias; const float* col_scale; const float* R;
    int64_t ldi, ldo, ldw, ldr;
    int32_t batch, hi, wi, ho, wo, cin, cout, ksize, stride, relu;
} rb_tiny_conv_args;
int romab200_tiny_conv(const rb_tiny_conv_args* args, void* stream);

/* Channel mean of an NCHW fp32 image batch (x.mean(dim=1), tiny.py:85) followed, when instance_norm != 0, by the
 * per-image InstanceNorm2d(1) without affine or running statistics (biased variance, eps; tiny.py:86):
 * in [B,C,H,W] -> out [B,H,W] (a 1-channel channels-last map). */
typedef struct { const float* in; float* out; int32_t batch, channels, h, w, instance_norm; float eps; } rb_tiny_gray_args;
int romab200_tiny_gray(const rb_tiny_gray_args* args, void* stream);

/* AvgPool2d(4, 4) on a channels-last fp32 map (XFeat skip1, tiny.py:89): [B,hi,wi,c] -> [B,hi/4,wi/4,c], pitch = c */
typedef struct { const float* in; float* out; int32_t batch, hi, wi, c; } rb_tiny_avgpool_args;
int romab200_tiny_avgpool4(const rb_tiny_avgpool_args* args, void* stream);

/* out[i] = (a[i] + b[i]) + c[i] over n floats: x3 + x4 + x5 in front of block_fusion (tiny.py:95-97) */
typedef struct { const float* a; const float* b; const float* c; float* out; int64_t n; } rb_tiny_add3_args;
int romab200_tiny_add3(const rb_tiny_add3_args* args, void* stream);

/* Fused coarse-match embedding: correlation + first-index argmax + low-resolution softmax + expectation
 * (corr_volume + pos_embed, tiny.py:115-140,178-191), without materialising the [h1*w1, h0*w0] volume.
 * For pixel i of image 0: s_j = <f1[b,j,:], f0[b,i,:]> / scale for every pixel j of image 1, best = first argmax_j s_j;
 *   exact == 0: P = softmax over {s_j : j on the stride-4 lattice (y % 4 == 0, x % 4 == 0)} U {(float)best}  (the extra logit is the
 *               argmax INDEX, as the reference computes it), pos = sum_k P_k grid_lr[k] + P_last * grid[best];
 *   exact != 0: pos = sum_j softmax(s)_j grid[j].
 * f0 [B, h0*w0, c], f1 [B, h1*w1, c] fp32 contiguous, c == 64; state [B, h0*w0, 3] receives (pos_x, pos_y, 0).
 * grid_x / grid_y: linspace(-1+1/w1, 1-1/w1, w1), linspace(-1+1/h1, 1-1/h1, h1); grid_lr_x / grid_lr_y: linspace(-1+4/w1, 1-4/w1, w1/4),
 * linspace(-1+4/h1, 1-4/h1, h1/4) (not the centres of the sub-sampled pixels; reproduced as the reference has them).  h1 % 4 == w1 % 4 == 0. */
typedef struct {
    const float* f0; const float* f1; float* state;
    int32_t batch, h0, w0, h1, w1, c; float scale; int32_t exact;
    const float* grid_x; const float* grid_y; const float* grid_lr_x; const float* grid_lr_y;
} rb_tiny_pos_embed_args;
int romab200_tiny_pos_embed(const rb_tiny_pos_embed_args* args, void* stream);

/* Warp-and-concat prologue of the matcher heads (tiny.py:205-214): out[b,p,:] = [f0[b,p,0:c] | grid_sample(f1[b], flow) | flow],
 * flow = state[b,p,0:2]; bilinear, zero padding, align_corners=False.  f0 [B,h0,w0,ldf0], f1 [B,h1,w1,ldf1], state [B,h0,w0,lds],
 * out [B,h0,w0,ldo] (columns 2c+2 .. ldo-1 untouched). */
typedef struct {
    const float* f0; const float* f1; const float* state; float* out;
    int64_t ldf0, ldf1, lds, ldo; int32_t batch, h0, w0, h1, w1, c;
} rb_tiny_warp_concat_args;
int romab200_tiny_warp_concat(const rb_tiny_warp_concat_args* args, void* stream);

/* match() epilogue of TinyRoMa (tiny.py:216-232): state [B,H,W,3] (already resized to the input size) ->
 * warp [B,H,W,4] = (grid_x[x], grid_y[y], state.x, state.y), cert [B,H,W] = sigmoid(state.z).  No clamp, no mask. */
typedef struct { const float* state; float* warp; float* cert; int32_t batch, h, w; const float* grid_x; const float* grid_y; } rb_tiny_epilogue_args;
int romab200_tiny_match_epilogue(const rb_tiny_epilogue_args* args, void* stream);

/* ---- JPEG decoding (roma_b200/jpeg.py), byte-identical to libjpeg-turbo's default decompression (Pillow's Image.open) ----
 * One launch set decodes a batch of baseline / extended sequential Huffman JPEGs that roma_b200.jpeg.parse accepted:
 * romab200_jpeg_entropy (unstuff + restart markers, self-synchronising parallel Huffman decode, coefficient emit, DC
 * prediction), then romab200_jpeg_pixels (dequantise + ISLOW IDCT into planes, fancy upsampling + YCbCr -> RGB).
 * The host fills `desc` (int64 [batch, 64], layout D_* in jpeg.py) and `tables` (int32 [batch, 6 * 804 + 192]: per scan
 * component a DC and an AC Huffman lookup, then 3 quantisation tables in natural order) and sizes every buffer from the
 * headers alone.  A stream the decoder rejects (corrupt entropy data, restart markers out of sequence, no EOI after the scan)
 * sets state[b * 8 + 1] (a status word per image, 0 = ok) instead of faulting; every read is bounded by the stream length
 * and every write by the header's block count, for any byte string.  Deterministic: no output depends on timing. */
typedef struct {
    int32_t batch;
    const uint8_t* stream;    /* entropy-coded data of every image (from the byte after SOS to the end of the file), each zero-padded by >= 16 bytes */
    const int64_t* desc;      /* [batch, 64] */
    const int32_t* tables;    /* [batch, 6 * 804 + 192] */
    uint8_t* comp;            /* compacted (unstuffed) bitstreams, stream_len + 16 bytes per image */
    int32_t* chunks;          /* [2 * chunks]: kept bytes / RST markers per 4096-byte chunk, scanned in place */
    int32_t* istart;          /* [sum (n_intervals + 1)]: first byte of every restart interval in the compacted stream, then its length */
    int64_t* exits;           /* [2 * total_slots]: decoder exit states of the sync passes (double-buffered) */
    int32_t* counts;          /* [2 * total_slots]: blocks started per subsequence | first block of each subsequence in its interval */
    int16_t* coef;            /* [total_blocks, 64] natural order, zero-filled by the caller; DC resolved after the entropy stage */
    int32_t* state;           /* [batch, 8]: scan end, status, compacted length, RST count, completed blocks */
    int32_t* flags;           /* [8] zero-filled: change flags of the sync passes, pass count (flags[3]), barrier counter, no-convergence */
    int32_t max_chunks, max_intervals;
    int64_t total_slots, total_blocks;
    uint8_t* planes;          /* pixels: per-component IDCT output planes (desc D_PLANE_*) */
    uint8_t* out;             /* pixels: uint8 [H, W, C] per image at desc D_OUT_OFF */
    int64_t max_pixels;       /* pixels: max H * W over the batch */
} rb_jpeg_args;
int romab200_jpeg_entropy(const rb_jpeg_args* args, void* stream);
int romab200_jpeg_pixels(const rb_jpeg_args* args, void* stream);

/* ---- relative pose: `estimate_pose` (romatch/utils/utils.py:30-51) = cv2.findEssentialMat (five-point RANSAC) + cv2.recoverPose ----
 * B pairs with ragged point counts, packed: pair b owns points [offsets[b], offsets[b+1]).  All arithmetic is float64.
 *   romab200_pose_hypotheses  normalises every point, xn = inv(K[:2,:2]) (x - K[:2,2]) with the closed-form 2x2 inverse
 *                             (utils.py:33-37), then draws and solves the RB_POSE_ROUND hypotheses of round `round`:
 *                             hypothesis h of pair b takes 5 distinct indices from Philox4x32-10 with key (seed lo, seed hi) and
 *                             counter (h, b, s, 0), s = 0, 1, ...; the four words of each block are used in order, word w
 *                             gives index (w * n) >> 32, a repeated index is skipped.  Nister's five-point solver gives up
 *                             to RB_POSE_MAX_SOL essential matrices, unit Frobenius norm, largest-magnitude entry positive.
 *                             A pair with n == 5 solves its 5 points once (hypothesis 0).
 *   romab200_pose_score       inlier counts of every solution: OpenCV's E error (Sampson) in float64 without contraction,
 *                             rounded to float, <= (float)(thresh^2); point slices over grid.y, partial counts, no atomics.
 *   romab200_pose_select      one thread per pair replays OpenCV's sequential RANSAC loop over the round (best model changes
 *                             iff count > max(best, 4), niters = RANSACUpdateNumIters(conf, (n - count) / n, 5, niters), stop
 *                             at iter >= niters), keeps the best E and sets running[0] when a pair needs another round.
 *   romab200_pose_recover     recoverPose(E, xn0, xn1, I, 1e9, mask) on the best E (n == 5: on every solution in turn, the
 *                             mask carried from one call to the next, as the reference's loop does): SVD decomposition,
 *                             DLT triangulation of the four (R, +-t), chirality and distance tests, OpenCV's candidate order.
 * The caller zero-fills `state` before round 0 and calls hypotheses / score / select for rounds 0, 1, ... while
 * running[0] != 0 and round * RB_POSE_ROUND < max_iters, then recover once. */
#define RB_POSE_ROUND 1024
#define RB_POSE_MAX_SOL 10
#define RB_POSE_MAX_SPLITS 16
#define RB_POSE_STATE 8       /* state[b, :]: iter, niters, best count, best hypothesis, best solution, E to recover, running, n */
typedef struct {
    int32_t batch;
    const double* x0; const double* x1;   /* [total, 2] pixel coordinates in image 0 / image 1 */
    const int64_t* offsets;               /* [batch + 1] */
    const double* K;                      /* [batch, 2, 3, 3]: K0, K1 of each pair */
    int64_t max_n;                        /* largest pair (sizes the point slices of the score) */
    double thresh, conf;
    int32_t max_iters, round;
    uint64_t seed;
    double* xn;                           /* [total, 4] normalised (x0, y0, x1, y1) */
    int32_t* sample;                      /* [batch, RB_POSE_ROUND, 5] drawn indices of the round */
    double* E;                            /* [batch, RB_POSE_ROUND, RB_POSE_MAX_SOL, 9] solutions of the round, row-major */
    int32_t* nsol;                        /* [batch, RB_POSE_ROUND] */
    int32_t* counts;                      /* [batch, RB_POSE_MAX_SPLITS, RB_POSE_MAX_SOL, RB_POSE_ROUND] partial inlier counts */
    int32_t* state;                       /* [batch, RB_POSE_STATE] */
    double* best_E;                       /* [batch, RB_POSE_MAX_SOL, 9] */
    int32_t* running;                     /* [1] */
    double* R; double* t;                 /* [batch, 3, 3], [batch, 3] */
    uint8_t* ok;                          /* [batch] */
    uint8_t* mask;                        /* [total] */
} rb_pose_args;
int romab200_pose_hypotheses(const rb_pose_args* args, void* stream);
int romab200_pose_score(const rb_pose_args* args, void* stream);
int romab200_pose_select(const rb_pose_args* args, void* stream);
int romab200_pose_recover(const rb_pose_args* args, void* stream);

/* ---- homography: cv2.findHomography(pos_a, pos_b, cv2.RANSAC, ...) of the HPatches harness
 *      (romatch/benchmarks/hpatches_sequences_homog_benchmark.py:80-86), OpenCV 4.13's estimator with the sample stream replaced ----
 * B pairs with ragged point counts, packed: pair b owns points [offsets[b], offsets[b+1]).  The points are float32, as cv2 converts them.
 *   romab200_homography_hypotheses  one thread per hypothesis of round `round`.  Hypothesis h of pair b, attempt a (a = 0, 1, ...)
 *                             draws 4 distinct indices from Philox4x32-10 with key (seed lo, seed hi) and counter (h, b, a, s),
 *                             s = 0, 1, ...; the four words of each block are used in order, word w gives index (w * n) >> 32, a
 *                             repeated index is skipped.  The attempt is rejected, and attempt a + 1 drawn, when OpenCV's checkSubset
 *                             fails: haveCollinearPoints on either image (the last point against every pair of earlier ones,
 *                             |dx2 dy1 - dy2 dx1| <= FLT_EPSILON (|dx1| + |dy1| + |dx2| + |dy2|), differences taken in float, the test
 *                             in double), or the signs of det(A) det(B) over the triples 012, 123, 023, 130 are not all equal.  After
 *                             RB_HOMOG_MAX_ATTEMPTS rejections the hypothesis is "not found" (status -1).  Otherwise the 4 points are
 *                             solved with OpenCV's normalisation (centroid, scale = count / sum |x - c| per axis, no model when a sum is
 *                             below DBL_EPSILON) and the null vector of the normalised 8x9 system by Gauss-Jordan with partial pivoting
 *                             (no model on a pivot that is not finite or below 1e-12 of the first), de-normalised and multiplied by
 *                             1 / H[2][2] (status 1; 0 = no model).  A pair with n == 4 solves its 4 points once (hypothesis 0, no check).
 *   romab200_homography_score  inlier counts: OpenCV's computeError in float32 with every operation rounded separately, H cast to
 *                             float, ww = 1 / (h6 x + h7 y + 1), dx = (h0 x + h1 y + h2) ww - x', err = dx^2 + dy^2 <= (float)(thresh^2);
 *                             point slices over grid.y, integer partial counts, no atomics.
 *   romab200_homography_select one warp per pair replays OpenCV's sequential loop over the round, 32 hypotheses per step: the best
 *                             model changes iff count > max(best, 3), then niters = RANSACUpdateNumIters(conf, (n - count) / n, 4, niters);
 *                             a "not found" hypothesis ends the loop (at iteration 0: no model); the loop stops at iter >= niters.
 *                             Sets running[0] when a pair needs another round.
 *   romab200_homography_refine one CTA per pair: the mask of the best model (the score's test), then (n > 4) the normalised DLT on
 *                             all inliers (the smallest eigenvector of the 9x9 L^T L, cyclic Jacobi) and at most 10 Levenberg-Marquardt
 *                             steps on the 8 parameters with H[2][2] = 1 (OpenCV's HomographyRefineCallback residual, in double).  Every
 *                             sum over the inliers runs in a fixed order.  method == 0: the same on all points, without RANSAC.
 *                             For n > 4 the returned mask is the inlier set of the refined model by the score's test, which is what
 *                             cv2 4.13 returns (n == 4: all ones).
 * The caller zero-fills `state` before round 0 and calls hypotheses / score / select for rounds 0, 1, ... while running[0] != 0 and
 * round * RB_HOMOG_ROUND < max_iters, then refine once (method 0: refine only). */
#define RB_HOMOG_ROUND 2048
#define RB_HOMOG_MAX_SPLITS 32
#define RB_HOMOG_MAX_ATTEMPTS 10000
#define RB_HOMOG_STATE 8      /* state[b, :]: iter, niters, best count, best hypothesis, running, n, failed, unused */
typedef struct {
    int32_t batch;
    const float* src; const float* dst;   /* [total, 2] points in image A / image B */
    const int64_t* offsets;               /* [batch + 1] */
    int64_t max_n;                        /* largest pair (sizes the point slices of the score) */
    double thresh, conf;
    int32_t max_iters, round, method;     /* method: 0 (least squares on all points) or 8 (RANSAC) */
    uint64_t seed;
    int32_t* sample;                      /* [batch, RB_HOMOG_ROUND, 4] drawn indices of the round */
    int32_t* attempts;                    /* [batch, RB_HOMOG_ROUND] rejected attempts before the drawn subset */
    int32_t* status;                      /* [batch, RB_HOMOG_ROUND]: 1 model, 0 no model, -1 not found */
    double* H;                            /* [batch, RB_HOMOG_ROUND, 9] models of the round, row-major */
    int32_t* counts;                      /* [batch, RB_HOMOG_MAX_SPLITS, RB_HOMOG_ROUND] partial inlier counts */
    int32_t* state;                       /* [batch, RB_HOMOG_STATE] */
    double* best_H;                       /* [batch, 9] the best RANSAC model */
    int32_t* running;                     /* [1] */
    double* out_H;                        /* [batch, 9] the refined model */
    uint8_t* ok;                          /* [batch] */
    uint8_t* mask;                        /* [total] */
} rb_homography_args;
int romab200_homography_hypotheses(const rb_homography_args* args, void* stream);
int romab200_homography_score(const rb_homography_args* args, void* stream);
int romab200_homography_select(const rb_homography_args* args, void* stream);
int romab200_homography_refine(const rb_homography_args* args, void* stream);

/* ---- fundamental matrix: cv2.findFundamentalMat(kptsA, kptsB, ransacReprojThreshold, cv2.USAC_MAGSAC, confidence, maxIters) of the
 *      reference's usage example (README.md:62-78, demo/demo_fundamental.py): MAGSAC++ over seven-point samples ----
 * B pairs with ragged point counts, packed: pair b owns points [offsets[b], offsets[b+1]).  x1^T F x0 = 0.  All arithmetic is float64
 * and, where a stage is restated bit for bit (oracle/fundamental_ransac.py), every operation is rounded separately.
 *   romab200_fund_hypotheses  round 0 first normalises every pair (one CTA per pair; the rows whose four coordinates are finite give
 *                             centroids and mean distances to them through fixed-order sums, scale = sqrt(2) / mean distance; norm[b] =
 *                             (cx0, cy0, s0, cx1, cy1, s1), xn = ((x - c) s) per image).  Then one thread per hypothesis of the round:
 *                             hypothesis h of every pair takes 7 distinct indices from Philox4x32-10 with key (seed lo, seed hi) and
 *                             counter (h, s, 0, RB_FUND_CTR), s = 0, 1, ...; words in order, index (w * n) >> 32, repeats skipped.  The
 *                             counter does not name the pair, so a pair's result does not depend on its place in the batch.  The 7x9 system
 *                             of the normalised points is reduced by Gauss-Jordan with partial pivoting (no model on a pivot that is not
 *                             finite or below 1e-12 of the first), giving the pencil F2 + l (F1 - F2); the real roots of the cubic
 *                             det(F2 + l (F1 - F2)) are bracketed by the critical points and the Cauchy bound and bisected to adjacent
 *                             doubles.  A root is kept if (e' x x_i) . (F x_i) has the same strict sign on all 7 points (the oriented
 *                             epipolar constraint; e' the largest of the three cross products of F's columns).  The kept models, in
 *                             ascending l, are de-normalised (T1^T F T0) and scaled to unit Frobenius norm.  A pair with n == 7 solves
 *                             its 7 points once (hypothesis 0).
 *   romab200_fund_score       thread = (hypothesis, model slot).  Per point the squared Sampson distance r2 = (x1^T F x0)^2 /
 *                             ((F x0)_0^2 + (F x0)_1^2 + (F^T x1)_0^2 + (F^T x1)_1^2); the MAGSAC++ loss (sigma_max = thresh) is 1
 *                             unless r2 < l2 = RB_FUND_K2 thresh^2, then table[0] interpolated linearly at p = r2 (RB_FUND_TABLE / l2):
 *                             t[i] + (p - i) (t[i + 1] - t[i]), i = min(floor(p), RB_FUND_TABLE - 1).  Slice y holds points
 *                             [y RB_FUND_SLICE, (y + 1) RB_FUND_SLICE) of its pair, whatever the batch; its loss is the sequential sum
 *                             over them in index order and its count the points with r2 < thresh^2.
 *   romab200_fund_select      one warp per pair replays the sequential loop: the slices of a model add up in slice order, a model
 *                             replaces the best iff its loss is lower, then niters = RANSACUpdateNumIters(conf, (n - count) / n, 7,
 *                             niters); the loop stops at iter >= niters.  Sets running[0] when a pair needs another round.
 *   romab200_fund_refine      one CTA per pair, sigma-consensus++: (n >= 8) at most RB_FUND_REFINE_ITERS times, weights table[1]
 *                             interpolated as above, the weighted normalised eight-point fit (the smallest eigenvector of the 9x9 sum
 *                             of w a a^T, cyclic Jacobi), rank 2 by a 3x3 SVD, de-normalised; the fit is kept while the loss (summed
 *                             over the CTA in a fixed order) decreases.  mask = r2 < thresh^2 under the returned F, which has unit
 *                             Frobenius norm and its largest-magnitude entry positive.  ok[b] = 0, F and mask zero, when no model.
 * `table` is [2, RB_FUND_TABLE + 1] float64: the normalised MAGSAC++ loss and weight at r^2 = (i / RB_FUND_TABLE) RB_FUND_K2 thresh^2
 * (roma_b200/geometry.py, DESIGN.md); RB_FUND_K2 is the 0.99 quantile of chi^2 with 4 degrees of freedom.  The caller zero-fills `state` before round 0 and calls hypotheses / score / select for rounds
 * 0, 1, ... while running[0] != 0 and round * RB_FUND_ROUND < max_iters, then refine once. */
#define RB_FUND_ROUND 1024
#define RB_FUND_MODELS 3
#define RB_FUND_SLICE 512
#define RB_FUND_TABLE 1024
#define RB_FUND_REFINE_ITERS 10
#define RB_FUND_CTR 0x46370000u
#define RB_FUND_K2 13.276704135987622
#define RB_FUND_STATE 8       /* state[b, :]: iter, niters, best hypothesis, best slot, running, n, unused, unused */
typedef struct {
    int32_t batch;
    const double* x0; const double* x1;   /* [total, 2] points in image A / image B */
    const int64_t* offsets;               /* [batch + 1] */
    int64_t max_n;                        /* largest pair (sizes the grid of the score) */
    double thresh, conf;
    int32_t max_iters, round;
    uint64_t seed;
    const double* table;                  /* [2, RB_FUND_TABLE + 1] loss, weight */
    double* norm;                         /* [batch, 6] */
    double* xn;                           /* [total, 4] normalised (x0, y0, x1, y1) */
    int32_t* sample;                      /* [batch, RB_FUND_ROUND, 7] drawn indices of the round */
    int32_t* nmod;                        /* [batch, RB_FUND_ROUND] models of each hypothesis */
    double* F;                            /* [batch, RB_FUND_ROUND, RB_FUND_MODELS, 9] models of the round, row-major */
    int32_t* counts;                      /* [batch, ceil(max_n / RB_FUND_SLICE), RB_FUND_ROUND * RB_FUND_MODELS] */
    double* losses;                       /* [batch, ceil(max_n / RB_FUND_SLICE), RB_FUND_ROUND * RB_FUND_MODELS] */
    int32_t* state;                       /* [batch, RB_FUND_STATE] */
    double* best_F;                       /* [batch, 9] the best model of the loop */
    double* best_loss;                    /* [batch] its loss */
    int32_t* running;                     /* [1] */
    double* out_F;                        /* [batch, 9] the refined model */
    uint8_t* ok;                          /* [batch] */
    uint8_t* mask;                        /* [total] */
} rb_fund_args;
int romab200_fund_hypotheses(const rb_fund_args* args, void* stream);
int romab200_fund_score(const rb_fund_args* args, void* stream);
int romab200_fund_select(const rb_fund_args* args, void* stream);
int romab200_fund_refine(const rb_fund_args* args, void* stream);

/* ---- depth-based ground-truth warps and the MegaDepth dense metric: `warp_kpts`, `get_gt_warp` (romatch/utils/utils.py:325-454)
 *      and `MegadepthDenseBenchmark.geometric_dist` (romatch/benchmarks/megadepth_dense_benchmark.py:17-42) ----
 * One float64 statement of the geometry, shared by the three entry points.  For a normalised point (x, y) of view 0 of pair b:
 *   d0 = grid_sample(depth0[b], (x, y))            zero padding, align_corners=False, ATen's unnormalisation ((x + 1) * w0 - 1) / 2;
 *                                                  mode 0 bilinear (corners accumulated nw, ne, sw, se), mode 1 nearest (nearbyint)
 *   X  = inv(K0[b]) ((w0 (x + 1) / 2, h0 (y + 1) / 2, 1) d0),  Y = R X + t with [R | t] = T[b, :3, :4],  z = Y[2]
 *   p  = K1[b] Y,  u = p[0] / (p[2] + 1e-4),  v = p[1] / (p[2] + 1e-4)
 *   warped = (2 u / w1 - 1, 2 v / h1 - 1),  d1 = grid_sample(depth1[b], warped)
 *   valid = d0 != 0  &&  0 < u < w1 - 1  &&  0 < v < h1 - 1  &&  |(d1 - z) / d1| < rel_threshold   (a NaN compares false)
 * Every operation is a separately rounded float64 operation (no FMA contraction), so the three entry points give the same bits
 * for the same point.  inv(K0) is the adjugate over the determinant, computed once per CTA; nothing is inverted on the host.
 * depth0 [batch, h0, w0] and depth1 [batch, h1, w1] are contiguous maps of dtype `depth_dtype` (RB_F32 or RB_F64, converted in
 * registers; the two views may differ in size); T [batch, T_rows, 4] (T_rows 3 or 4), K0, K1 [batch, 3, 3] contiguous float64.
 * warped is written for every point, valid or not.  Deterministic.
 *
 * romab200_warp_kpts: arbitrary points kpts [batch, L, 2] of dtype `kpts_dtype` (RB_F32 or RB_F64) -> warped [batch, L, 2] float64,
 * valid [batch, L] uint8 (utils.py:399-454 with smooth_mask = False, return_relative_depth_error = False). */
typedef struct {
    const void* depth0; const void* depth1; int32_t depth_dtype; int32_t h0, w0, h1, w1;
    const double* T; int32_t T_rows; const double* K0; const double* K1;
    int32_t batch; int32_t mode; double rel_threshold;
    const void* kpts; int32_t kpts_dtype; int64_t L;
    double* warped; uint8_t* valid;
} rb_warp_kpts_args;
int romab200_warp_kpts(const rb_warp_kpts_args* args, void* stream);

/* get_gt_warp (utils.py:325-354): the points are the pixel centres of an H x W image, point (i, j) = (grid_x[j], grid_y[i]).
 * grid_x [W], grid_y [H] are the float32 linspace(-1 + 1/n, 1 - 1/n, n) vectors the reference builds (it widens them to float64
 * afterwards; the closed form -1 + (2 i + 1) / n in float64 differs from them in the 8th digit for most n, so they are taken
 * as data).  x2 [batch, H, W, 2] float64 = warped, prob [batch, H, W] float32 = valid as 0 / 1.  Apart from the two depth maps
 * nothing of size batch * H * W is read. */
typedef struct {
    const void* depth0; const void* depth1; int32_t depth_dtype; int32_t h0, w0, h1, w1;
    const double* T; int32_t T_rows; const double* K0; const double* K1;
    int32_t batch; int32_t mode; double rel_threshold;
    const float* grid_x; const float* grid_y; int32_t H, W;
    double* x2; float* prob;
} rb_gt_warp_args;
int romab200_gt_warp(const rb_gt_warp_args* args, void* stream);

/* MegadepthDenseBenchmark.geometric_dist (megadepth_dense_benchmark.py:17-42), bilinear, rel_threshold as given (the harness: 0.05).
 * dense_matches [batch, H, W, 4] float32 is read in place: element (b, i, j, c) at dense_matches[b * dm_sb + i * dm_sy + j * dm_sx +
 * c * dm_sc] (strides in floats, so the left half of a symmetric warp [batch, H, 2W, 4] needs no copy).  Per pixel: warp
 * dense_matches[..., 0:2]; ground truth in pixels (W (wx + 1) / 2, H (wy + 1) / 2) in float64; prediction in pixels from
 * dense_matches[..., 2:4] by the same expression in float32, as the harness computes it; gd = sqrt(dx^2 + dy^2) in float64.
 * gd [batch, H, W] float64 receives the distance, NaN where the pixel is not valid; prob [batch, H, W] float32 = valid as 0 / 1.
 * The ground-truth warp itself is never written.
 * The same launch leaves one partial per CTA (float64 sum of gd over its valid pixels, and the counts of valid, gd < 1, gd < 3,
 * gd < 5) in partial_sum [batch, RB_DEPTH_WARP_MAX_CTAS] and partial_cnt [batch, RB_DEPTH_WARP_MAX_CTAS, 4]; a second, single-CTA
 * kernel adds them in a fixed order: pair_sum [batch] float64, pair_cnt [batch, 4] int64 (valid, < 1, < 3, < 5), and over all pairs
 * pck [3] float32 = (float)count_t * (1.f / (float)count_valid), which is what (gd[prob == 1] < t).float().mean() evaluates to on
 * the device, and epe [1] float64 = sum * (1 / count_valid).  No pair valid: NaN.  No atomics: the result does not depend on timing. */
#define RB_DEPTH_WARP_MAX_CTAS 512
typedef struct {
    const void* depth0; const void* depth1; int32_t depth_dtype; int32_t h0, w0, h1, w1;
    const double* T; int32_t T_rows; const double* K0; const double* K1;
    int32_t batch; double rel_threshold;
    const float* dense_matches; int64_t dm_sb, dm_sy, dm_sx, dm_sc; int32_t H, W;
    double* gd; float* prob;
    double* partial_sum; int32_t* partial_cnt;
    double* pair_sum; int64_t* pair_cnt; float* pck; double* epe;
} rb_dense_geometric_dist_args;
int romab200_dense_geometric_dist(const rb_dense_geometric_dist_args* args, void* stream);

/* ---- structure-from-motion match graph: per-image keypoints and one-to-one pair matches from sampled dense matches ----
 * Not in the reference (its users snap `sample()` output to pixels on the host).  For pair k = (i, j) = pairs[k] and sample s < n,
 * side 0 is (u, v) = matches[k, s, 0:2] in image i and side 1 is matches[k, s, 2:4] in image j, both with certainty[k, s].  For an
 * image of image_sizes[img] = (H, W): x = (W / 2) * (u + 1), y = (H / 2) * (v + 1), each operation rounded to fp32 (matcher.py:713-717);
 * the side is ignored unless certainty > min_certainty (>= 0) and u, v and the certainty are finite.
 * cell (cx, cy) = (min(max(floor(x), 0), W - 1) / cell_size, the same for y) (integer division), index cy * gw + cx with
 * gw = ceil(W / cell_size), gh = ceil(H / cell_size).  The winner of a cell is the side landing in it with the largest certainty,
 * ties to the smallest g = (k * n + s) * 2 + side; it gives the keypoint's position (x, y) and score.  Ids: occupied cells in raster
 * order within each image.  Everything is exact and order-free (integer atomics on monotone keys only), so the result does not
 * depend on timing or on how images and pairs are grouped.
 *
 * romab200_match_graph_keypoints: the images [img_begin, img_end) (one group) in one call.  cell_start / tile_start [num_images + 1]
 * int64 are the cumulative cell and tile counts over all images (an image no pair references has none); the group's grid is
 * grid_bits [cells] (uint32, the winning certainty's bits, then the cell's id) and grid_g [cells] (uint64, the winning g), cells =
 * cell_start[img_end] - cell_start[img_begin] = grid_cells; tile_scan [grid_tiles + 1] int64, grid_tiles the same difference of
 * tile_start (a tile is RB_MG_TILE consecutive cells of one image).  The caller passes the two extents it built the tables with.  kp_offsets [num_images + 1] int64: entry img_begin must hold the keypoints of the
 * images before the group (0 for the first); the call writes entries img_begin + 1 .. img_end, and the keypoints [kp_capacity, 2],
 * kp_scores [kp_capacity] of the group's images at those offsets.  sid [num_pairs, n, 2] int32 receives, for every side whose image
 * is in the group, its keypoint id, or -1 when ignored.
 *
 * romab200_match_graph_count + romab200_match_graph_emit: the one-to-one matches of pairs [pair_begin, pair_end) from sid, one CTA
 * per pair.  A sample is used iff both sides have an id (a, b).  best_b(a) = b of the used sample with that a of the largest
 * certainty, ties to the smallest s; best_a(b) likewise; (a, best_b(a)) is kept iff best_a(best_b(a)) == a, with that certainty as
 * its score, in ascending a.  A CTA sorts 64-bit keys three times (certainty rank, then (b, rank), then (a, rank)).  It needs
 * pair_bytes = 8 * n2 + 5 * n rounded up to a multiple of 16 (n2 the smallest power of two >= n): shared memory when
 * pair_bytes <= RB_MG_PAIR_SMEM, otherwise scratch of pair_bytes per pair of the call.
 * count writes pair k's match count to match_offsets[k]; the call with pair_end == num_pairs then turns match_offsets [num_pairs + 1]
 * into exclusive offsets with the total last.  emit (after the caller has sized the outputs) writes matches [match_capacity, 2]
 * int32 (a, b) and match_scores at those offsets. */
#define RB_MG_TILE 2048
#define RB_MG_PAIR_SMEM 230400
typedef struct {
    const int64_t* pairs; int32_t num_pairs, n;
    const float* matches; const float* certainty;
    const int32_t* image_sizes; int32_t num_images, cell_size; float min_certainty;
    const int64_t* cell_start; const int64_t* tile_start; int32_t img_begin, img_end;
    uint32_t* grid_bits; uint64_t* grid_g; int64_t grid_cells;
    int64_t* tile_scan; int64_t grid_tiles;
    int64_t* kp_offsets; float* keypoints; float* kp_scores; int64_t kp_capacity;
    int32_t* sid;
} rb_match_graph_keypoints_args;
int romab200_match_graph_keypoints(const rb_match_graph_keypoints_args* args, void* stream);

typedef struct {
    const int32_t* sid; const float* certainty; int32_t num_pairs, n;
    int32_t pair_begin, pair_end;
    uint8_t* scratch; int64_t scratch_bytes;
    int64_t* match_offsets;
    int32_t* matches; float* match_scores; int64_t match_capacity;   /* emit only */
} rb_match_graph_pairs_args;
int romab200_match_graph_count(const rb_match_graph_pairs_args* args, void* stream);
int romab200_match_graph_emit(const rb_match_graph_pairs_args* args, void* stream);

/* ---- feature tracks of a match graph: connected components of its keypoint matches ----
 * Not in the reference.  The input is a match graph as consolidate_matches returns it, with pairs [num_pairs, 2] int64 (the pairs
 * it was built from), kp_offsets [num_images + 1] int64, match_offsets [num_pairs + 1] int64, matches [num_matches, 2] int32 (a, b)
 * and match_scores [num_matches] fp32.  The rules:
 * 1. Vertices.  Row r of the keypoints is a vertex.  Keypoint a of image i has row r = kp_offsets[i] + a.  K = kp_offsets[N] =
 *    num_rows, where N = num_images.
 * 2. Edges.  Each match (a, b) of pair k = (i, j) whose match_scores value is > min_score joins row kp_offsets[i] + a to row
 *    kp_offsets[j] + b.  The comparison is in fp32, with min_score rounded to fp32, so a NaN score is never an edge.  Repeated
 *    pairs, reversed pairs and i == j pairs all just add edges.
 * 3. Components.  Take the connected components of that graph on the K rows.  A component has a conflict when two distinct rows
 *    in it belong to one image.  num_conflicting counts those components, whatever their size.
 * 4. Tracks.  A component is a track when it has at least min_length rows (an int, at least 2) and has no conflict.  With
 *    drop_conflicts = 0, conflicts are allowed, and the elements of a track may then repeat an image.
 * 5. Order.  Tracks are numbered in ascending order of their smallest row.  The elements of a track are in ascending row order,
 *    which is image ascending, then keypoint id ascending.  kp_track[r] is the track of row r, or -1.
 * 6. Determinism.  The result is bit-identical from run to run, and it depends on no timing.
 * Every match's ids are checked, 0 <= a < K_i and 0 <= b < K_j (K_i = kp_offsets[i + 1] - kp_offsets[i]), before any access that
 * depends on them; an out-of-range match sets RB_TRACKS_BAD_ID in info[0] and is skipped.  A walk of parent pointers longer than
 * K steps (which the invariant parent[r] <= r rules out) sets RB_TRACKS_WALK and stops.  The caller checks the offsets on the host:
 * both start at 0 and do not decrease, pairs hold image indices < N, num_rows < 2^31, num_matches = match_offsets[num_pairs].
 *
 * romab200_tracks_link: parent[r] = r, then a lock-free union-find over the matches (path halving; a link is
 * atomicCAS(&parent[larger root], larger root, smaller root), so the root of a component is its smallest row), then
 * parent[r] = root(r) and size[root] = the component's size (integer atomics).  kp_track [num_rows] is set to -1.  The rows of
 * components of at least 2 rows are counted per tile of RB_TRACKS_TILE rows into tile_scan [ceil(num_rows / RB_TRACKS_TILE) + 1]
 * and scanned; info [5] int64 = {status, kept rows, T, E, num_conflicting} receives the status and the kept rows.
 * romab200_tracks_build (after the caller has read info[0..1] and sized the buffers by num_kept = info[1] > 0): the kept rows in
 * ascending order as keys (root << 32 | row), a stable LSD radix sort on the ceil(log2 num_rows) bits of the root in 8-bit digits
 * (keys and keys_alt [num_kept] uint64, hist [256 * ceil(num_kept / RB_TRACKS_TILE) + 1] int32), the conflict flags (bit 31 of
 * size[root]), then track_offsets [T + 1] int64 (capacity num_kept / 2 + 1), elements [E, 2] int32 (image, keypoint id; capacity
 * num_kept) and kp_track, and info[2..4].  tile_scan is reused for the sorted tiles.  Workspace: 8 bytes per row (parent, size),
 * 16.25 bytes per kept row, 8 bytes per tile. */
#define RB_TRACKS_TILE 4096
#define RB_TRACKS_BAD_ID 1
#define RB_TRACKS_WALK 2
typedef struct {
    const int64_t* pairs; int32_t num_pairs, num_images;
    const int64_t* kp_offsets; int32_t num_rows;
    const int64_t* match_offsets; const int32_t* matches; const float* match_scores; int64_t num_matches;
    float min_score; int32_t min_length, drop_conflicts;
    int32_t* parent; int32_t* size; int64_t* tile_scan; int64_t* info; int32_t* kp_track;
    int64_t num_kept;                                                   /* build only: */
    uint64_t* keys; uint64_t* keys_alt; int32_t* hist;
    int64_t* track_offsets; int32_t* elements;
} rb_tracks_args;
int romab200_tracks_link(const rb_tracks_args* args, void* stream);
int romab200_tracks_build(const rb_tracks_args* args, void* stream);

/* ---- geometric verification of a match graph: a MAGSAC++ fundamental matrix per pair, only its inlier matches kept ----
 * Not in the reference.  The input is a match graph as consolidate_matches returns it (kp_offsets [num_images + 1] int64, keypoints
 * [K, 2] fp32, match_offsets [num_pairs + 1] int64, matches [num_matches, 2] int32, match_scores [num_matches] fp32) with the pairs
 * [num_pairs, 2] int64 it was built from.  The rules:
 * 1. Points.  Pair k = (i, j) has matches (a, b).  Its points are x0 = keypoints[kp_offsets[i] + a] and x1 = keypoints[kp_offsets[j] + b],
 *    widened exactly to float64, in match order.
 * 2. Estimate.  F, ok and the per-match mask are what find_fundamental_batched([x0], [x1], USAC_MAGSAC, threshold, confidence,
 *    max_iters, seed=seed) returns for that pair.  The Philox counter of fundamental.cu does not name the pair, so every pair draws
 *    the stream keyed by seed alone.  Pair k is therefore bit-identical to that single call, whatever the chunking and pair order.
 *    Pairs with fewer than 7 matches get ok = 0.
 * 3. Accept.  num_inliers[k] is the sum of the mask.  accepted[k] = ok[k] and num_inliers[k] >= min_inliers.
 * 4. Output.  For an accepted pair, keep the matches whose mask is 1, in their original order (ascending a), with their scores
 *    unchanged.  A rejected pair keeps no matches.  match_offsets keeps num_pairs + 1 entries, so pair indices do not change.
 * 5. No special cases.  i == j and repeated pairs get exactly what rule 2 gives.
 * 6. Determinism.  Integer work only outside the estimator.  The result is bit-identical from run to run, for any workspace_bytes
 *    and under any pair order.
 * Every match's ids are checked, 0 <= a < K_i and 0 <= b < K_j, before any access that depends on them; an out-of-range match sets
 * RB_VERIFY_BAD_ID in info[0].  The caller checks the offsets on the host (both start at 0 and do not decrease, pairs hold image
 * indices < num_images, num_matches = match_offsets[num_pairs]).
 *
 * romab200_verify_check: every match's ids; info [2] int64 = {status, kept matches} is zeroed first.  The caller reads info[0] and
 *   launches no estimator when it is set.
 * romab200_verify_gather: the pairs [pair_begin, pair_end) of one chunk, whose matches are [match_offsets[pair_begin],
 *   match_offsets[pair_end]): x0, x1 [max(total, 1), 2] float64 (rule 1; zero for a bad id) and chunk_offsets [pair_end - pair_begin
 *   + 1] int64, starting at 0: the x0 / x1 / offsets layout of rb_fund_args.  With pair_list set, [pair_begin, pair_end) index
 *   pair_list instead, and the listed pairs pair_list[pair_begin], ... are packed in list order in the same layout (their pair
 *   indices must lie in [0, num_pairs); a pair may be listed twice); with pair_list null the call is unchanged.  The estimator then runs on the chunk (romab200_fund_*).
 *   Its device bytes, with B pairs, total matches and S = max(1, ceil(max_n / RB_FUND_SLICE)) score slices (max_n the chunk's
 *   largest pair), are the buffers it allocates plus the gathered points:
 *     B (RB_VERIFY_PAIR_BYTES + RB_VERIFY_SLICE_BYTES S) + RB_VERIFY_POINT_BYTES max(total, 1) + RB_VERIFY_CHUNK_BYTES
 *   per pair norm 48, sample 28 672, nmod 4 096, F 221 184, state 32, best_F 72, best_loss 8, out_F 72, ok 1, chunk_offsets 8;
 *   per pair and slice counts 12 288 and losses 24 576; per match xn 32, mask 1, x0 16, x1 16; once running 4 and chunk_offsets 8.
 * romab200_verify_count (after every chunk's F, ok and mask are in the whole-call ok [num_pairs] uint8 and mask [num_matches]
 *   uint8): one CTA per pair sums its mask (integers) into num_inliers [num_pairs] int64 and sets accepted [num_pairs] uint8 (rule 3);
 *   out_offsets [num_pairs + 1] int64 becomes the exclusive scan of the kept counts (num_inliers where accepted, else 0), total
 *   last; the kept matches (mask set and pair accepted) are counted per tile of RB_VERIFY_TILE matches into tile_scan
 *   [ceil(num_matches / RB_VERIFY_TILE) + 1] and scanned; info[1] = the total.
 * romab200_verify_emit (after the caller has sized the outputs by num_kept = info[1] > 0): out_matches [num_kept, 2] int32 and
 *   out_scores [num_kept] fp32, the kept matches in their original order (rule 4). */
#define RB_VERIFY_TILE 4096
#define RB_VERIFY_BAD_ID 1
#define RB_VERIFY_PAIR_BYTES 254193
#define RB_VERIFY_SLICE_BYTES 36864
#define RB_VERIFY_POINT_BYTES 65
#define RB_VERIFY_CHUNK_BYTES 12
typedef struct {
    const int64_t* pairs; int32_t num_pairs, num_images;
    const int64_t* kp_offsets; const float* keypoints; int64_t num_rows;
    const int64_t* match_offsets; const int32_t* matches; const float* match_scores; int64_t num_matches;
    int64_t* info;
    int32_t pair_begin, pair_end;                                       /* gather only: */
    double* x0; double* x1; int64_t* chunk_offsets;
    const uint8_t* ok; const uint8_t* mask; int64_t min_inliers;        /* count and emit: */
    int64_t* num_inliers; uint8_t* accepted; int64_t* tile_scan; int64_t* out_offsets;
    int64_t num_kept; int32_t* out_matches; float* out_scores;          /* emit only */
    const int32_t* pair_list;                                           /* gather only: null, or the pairs to pack */
} rb_verify_args;
int romab200_verify_check(const rb_verify_args* args, void* stream);
int romab200_verify_gather(const rb_verify_args* args, void* stream);
int romab200_verify_count(const rb_verify_args* args, void* stream);
int romab200_verify_emit(const rb_verify_args* args, void* stream);

/* ---- triangulation of feature tracks with known cameras: two-view RANSAC over each track's observations, multi-view refinement,
 *      reprojection and angle filters ----
 * Not in the reference.  The input is a match graph's kp_offsets [num_images + 1] int64 and keypoints [K, 2] fp32, the tracks built
 * from it (track_offsets [num_tracks + 1] int64, elements [num_elements, 2] int32 (image, keypoint id)) and per image i a camera
 * x ~ K_i (R_i X + t_i) in pixels.  All arithmetic is float64.  The rules:
 * 1. Observations.  Element (i, a) of track k is observed at x = keypoints[kp_offsets[i] + a], widened to float64.  The host builds a
 *    float64 camera table once: P_i = K_i [R_i | t_i] and C_i = -R_i^T t_i.  An observation's depth is (R_i X + t_i)_z.
 * 2. Hypotheses.  Let the track have L elements.  If L (L - 1) / 2 <= max_hypotheses, take every pair p < q in lexicographic order.
 *    Otherwise take max_hypotheses pairs: pair h is the two distinct indices in [0, L) that ransac_draw<2> gives under key seed and
 *    counter (h, s, k, RB_TRI_CTR), s = 0, 1, ..., in the order drawn.  A pair whose two elements share an image is skipped but keeps
 *    its index h (this can only happen with drop_conflicts = 0).
 * 3. Two-view point.  Triangulate each pair by DLT: the point is the eigenvector of the smallest eigenvalue of the 4 x 4 A^T A, where
 *    A has rows x P^3 - P^1 and y P^3 - P^2 per observation (P^r row r of P), dehomogenised.  The hypothesis is skipped if the point
 *    is not finite or either depth is <= 0.
 * 4. Support.  Element e is an inlier of X when its depth is > 0 and |pi(P_i X) - x_e|^2 <= max_error^2 (pi(p) = (p_0 / p_2,
 *    p_1 / p_2)).  The best hypothesis has the most inliers, ties to the smallest h.  If no hypothesis has 2 inliers, the track is
 *    not ok.
 * 5. Refine.  A multi-view DLT over the best hypothesis's inliers (the same rows, summed over them; the hypothesis's own point is
 *    kept if it is not finite), then Gauss-Newton on their summed squared reprojection error: at most RB_TRI_GN_ITERS steps, a step
 *    kept only if it lowers the cost, stopping at the first rejected step.  Then the inlier set is recomputed once against the
 *    refined X by rule 4.
 * 6. Accept.  A track is ok when it has at least 2 inliers in distinct images and the largest angle between X - C_i and X - C_j over
 *    its inlier pairs in distinct images (atan2(|a x b|, a . b)) is >= min_angle (radians, min_angle_deg pi / 180 on the host).
 * 7. Determinism.  The result is bit-identical from run to run: no float atomics, every reduction in a fixed order.
 * Outputs, zero where the track is not ok: X [num_tracks, 3], num_inliers [num_tracks] int32, error [num_tracks] (the mean
 * reprojection error in px of the inliers), inlier [num_elements] uint8; ok [num_tracks] uint8.
 * Every element's ids are checked, 0 <= i < num_images and 0 <= a < K_i, before any access that depends on them; a bad element sets
 * RB_TRI_BAD_ID in info[0] (zeroed by the call) and its track is left not ok.  The caller checks on the host: track_offsets start at 0,
 * never decrease and end at num_elements < 2^31; kp_offsets likewise; the cameras are finite; max_error2 > 0; 1 <= max_hypotheses.
 *
 * romab200_triangulate: one warp per track.  The lanes split the hypotheses (lane l takes h = l, l + 32, ...), each solving its DLT
 * by cyclic Jacobi (10 sweeps); the best is the warp maximum of (count << 32) | ~h.  The refinement sums the 4 x 4 DLT matrix, the
 * 3 x 3 normal equations and the cost over the lanes (each lane its elements e = l, l + 32, ... in order, then a xor butterfly);
 * the lanes split the angle test over the inlier pairs.  Observations are read through global memory, so any L is supported.
 * cameras [num_images, RB_TRI_CAM] float64 per image: P (12, row-major), row 2 of R (3), t_z, C (3), and the exclusion flag: 0, or
 * 1 for an image that is not among the registered `images` of triangulate_tracks.  An element of an excluded image is not an
 * observation: a pair that contains it is skipped but keeps its index h (as a pair within one image is in rule 2), and it is never an
 * inlier.  The other entries of an excluded image's row are not read. */
#define RB_TRI_CTR 0x54524900u
#define RB_TRI_GN_ITERS 10
#define RB_TRI_CAM 20
#define RB_TRI_BAD_ID 1
typedef struct {
    int32_t num_tracks, num_images;
    const int64_t* track_offsets; const int32_t* elements; int64_t num_elements;
    const int64_t* kp_offsets; const float* keypoints; int64_t num_rows;
    const double* cameras;
    double max_error2, min_angle;
    int32_t max_hypotheses;
    uint64_t seed;
    int64_t* info;                                                      /* [1] status */
    double* X; uint8_t* ok; int32_t* num_inliers; double* error; uint8_t* inlier;
} rb_tri_args;
int romab200_triangulate(const rb_tri_args* args, void* stream);

/* ---- bundle adjustment: Levenberg-Marquardt over the cameras' poses and the tracks' points, with a Schur-reduced camera system ----
 * Not in the reference.  The input is what triangulation takes and gives: kp_offsets and keypoints of a match graph, the tracks
 * (track_offsets, elements), per track ok [num_tracks] uint8 and per element inlier [num_elements] uint8, the points X
 * [num_tracks, 3], and per image i a camera x ~ K_i (R_i X + t_i) in pixels; K stays fixed.  All arithmetic is float64.  The rules:
 * 1. Observations.  The used observations are the elements e with inlier[e] set, in tracks with ok set.  Element (i, a) of track k
 *    is observed at x_e = keypoints[kp_offsets[i] + a], widened to float64.  A track that is not ok is not touched: its X stays as
 *    given (zero).
 * 2. Residual and cost.  r_e = pi(K_i (R_i X_k + t_i)) - x_e in px, and s_e = |r_e|^2.  The cost is F = 1/2 sum_e rho(s_e).
 *    rho(s) = s without a loss scale.  Otherwise rho(s) = c^2 log(1 + s / c^2) with c the loss scale (Cauchy), which is scipy's
 *    loss="cauchy", f_scale=c cost.
 * 3. Linearisation.  Parameters are d_omega_i, d_t_i per camera and d_X_k per ok track.  The update is R_i <- Exp(d_omega_i) R_i,
 *    t_i <- t_i + d_t_i and X_k <- X_k + d_X_k.  Exp is Rodrigues in float64: with theta^2 = |w|^2 > 2^-52, Exp(w) = cos theta I +
 *    (1 - cos theta) k k^T + sin theta [k]x with k = w / theta; otherwise the small-angle branch Exp(w) = I + [w]x.  Each
 *    observation's Jacobian block is weighted by w_e = rho'(s_e) (1 without a loss scale, 1 / (1 + s_e / c^2) with one): this is
 *    IRLS, with no second-order corrector.  H = J^T W J and g = J^T W r.
 * 4. Gauge.  The cameras in fixed_poses get d_omega = d_t = 0.  The cameras in fixed_tx get d_t_x = 0: in the reduced system, that
 *    row and column become the identity and the right-hand side becomes 0.  This is COLMAP's default, which holds the first pose
 *    and the second camera's x-translation constant.
 * 5. Damped step.  D is the diagonal of H, each entry clamped to [1e-6, 1e32].  Solve (H + lambda D) d = -g by the Schur complement
 *    on the cameras.  V_k is the damped 3 x 3 block of track k.  S = U - W V^-1 W^T, restricted to free cameras, is factored by
 *    dense Cholesky.  Back-substitution then gives d_X_k.  A non-positive or non-finite pivot makes the trial a rejected step.
 * 6. Trial.  pred = 1/2 d^T (lambda D d - g) and rho = (F(x) - F(x + d)) / pred.  The step is kept when rho > 1e-3, F(x + d) is
 *    finite and every used observation has depth > 0 at x + d.  When kept: lambda <- lambda max(1/3, 1 - (2 rho - 1)^3) and
 *    nu <- 2.  When not kept: lambda <- lambda nu and nu <- 2 nu.  Start from lambda = 1e-4 and nu = 2.  This is Ceres'
 *    Levenberg-Marquardt with radius 1 / lambda.
 * 7. Stop.  Each trial counts against max_iterations.  The run also stops after a kept step that lowered F by at most
 *    function_tolerance F ("function_tolerance"), or when lambda > 1e32 ("no_progress").  With no used observations or no free
 *    parameters, it returns the inputs ("nothing_to_adjust").
 * 8. Determinism.  There are no float atomics and every reduction runs in a fixed order, so reruns are bit-identical.
 * A track whose used observations repeat an image (possible with drop_conflicts = 0) is refused: it sets RB_BA_REPEATED in info[0].
 * Every used element's ids are checked, 0 <= i < num_images and 0 <= a < K_i, before any access that depends on them; a bad one
 * sets RB_BA_BAD_ID in info[0].
 * The caller checks on the host: the offsets as for triangulation, the cameras and points finite.  It builds the compact index of
 * the free cameras (those not in fixed_poses): free_index [num_images] int32 (-1 for a fixed camera), free_cams [num_free] int32
 * (their images, ascending) and fixed_tx [num_free] uint8 (1 for a camera in fixed_tx).
 *
 * The host drives the loop of rules 6-7 and reads result [RB_BA_RESULT] once per trial: F(x + d), pred, the number of used
 * observations with depth <= 0 at x + d, and the pivot flag.  The cameras are cams [num_images, RB_BA_CAM] float64: R (9,
 * row-major), t (3), K (9, row-major).  One trial is linearize, cameras, cholesky, solve, step; an accepted trial swaps the
 * (cams, X) and (cams_trial, X_trial) buffers.
 * romab200_ba_setup: info [2] int64 = {status, used observations} is zeroed; a warp per track checks its used elements' ids and
 *   writes elem_track [num_elements] int32 and keys (image << 32 | e, image = num_images for an unused element) [num_elements];
 *   radix_sort_hi32 (common.cuh) sorts them stably by image (keys_alt, hist RADIX_DIGITS ceil(num_elements / RB_TRACKS_TILE) + 1 int32);
 *   obs_offsets [num_images + 1] int64 is the start of each image's observations in obs [num_elements] int32 (element ids in
 *   ascending order per image); info[1] = obs_offsets[num_images].
 * romab200_ba_linearize: a warp per track at lambda: track_sys [num_tracks, RB_BA_TRACK] = V^-1 of the damped block (00, 01, 02, 11,
 *   12, 22), g_X (3), D_X (3), the track's cost 1/2 sum rho(s_e); W [num_elements, 18] = w_e J_c^T J_X (6 x 3 row-major) of every
 *   used element.  result[0..3] are zeroed.
 * romab200_ba_cameras: a CTA per free camera fills the 6 rows of S [6 num_free, 6 num_free] (row-major, the blocks (i, j) with j <= i;
 *   the Cholesky reads the lower triangle), rhs [6 num_free] and cam_sys [num_free, 12] = g_c (6), D_c (6).
 * romab200_ba_cholesky: S = L L^T in place (lower triangle), right-looking with RB_BA_NB-wide panels: panel, triangular solve and
 *   trailing update kernels; a pivot that is not > 0 and finite sets result[3].  Then the forward and backward substitutions turn
 *   rhs into the camera step.
 * romab200_ba_step: the trial cameras cams_trial, cam_pred [num_images] (1/2 d_c^T (lambda D_c d_c - g_c)), then a warp per track:
 *   d_X, X_trial, track_part [num_tracks, 3] = the trial cost, 1/2 d_X^T (lambda D_X d_X - g_X), and the count of depths <= 0;
 *   then result[0..2] as fixed-order tree sums.  Without free cameras, pass num_free = 0 and skip cameras and cholesky.
 * romab200_ba_cost: result[0] = the sum of the tracks' costs in track_sys (after linearize), result[1] = 0.
 * romab200_ba_error: error [num_tracks] = the mean |r_e| of the used observations of every ok track (0 for the others).
 * Device bytes, with N images, F free cameras, T tracks and E elements (the buffers bundle.py allocates):
 *   RB_BA_ELEMENT_BYTES E + RB_BA_TRACK_BYTES T + RB_BA_IMAGE_BYTES N + RB_BA_FREE_BYTES F + 288 F^2
 *   + 1024 ceil(E / RB_TRACKS_TILE) + RB_BA_ONCE_BYTES
 *   per element keys 8, keys_alt 8, elem_track 4, obs 4, W 144, inlier 1; per track track_sys 104, X 24, X_trial 24, track_part 24,
 *   error 8, track_offsets 8, track_ok 1; per image cams 168, cams_trial 168, cam_pred 8, free_index 4, obs_offsets 8, kp_offsets 8;
 *   per free camera cam_sys 96, rhs 48, free_cams 4, fixed_tx 1; S 288 F^2; once hist 4, obs_offsets 8, kp_offsets 8, track_offsets
 *   8, info 16, result 32.  W is stored rather than recomputed by the camera kernel: 144 B per element is 576 MB at 4 M elements.
 *
 * Camera models.  camera_model = 0 is the PINHOLE model above, and a zero-initialised struct means it.  camera_model = 1 is
 * SIMPLE_RADIAL (see the keypoint undistortion below): cams rows are RB_BA_CAM1 doubles R (9), t (3), f, cx, cy, k, and each camera
 * also refines its focal length and radial coefficient, with the principal point fixed.  The rules change as follows:
 * 2'. Residual.  r_e = (f d x + cx, f d y + cy) - x_e with (x, y) = (p0, p1) / p2, p = R_i X_k + t_i, r^2 = x^2 + y^2 and
 *    d = 1 + k r^2, on the raw (distorted) keypoint widened to float64.
 * 3'. Parameters.  Camera i has the 8 parameters (d_omega, d_t, d_f, d_k); the update adds f <- f + d_f and k <- k + d_k.  Through
 *    (x, y): du/dx = f (d + 2 k x^2), du/dy = dv/dx = 2 f k x y, dv/dy = f (d + 2 k y^2).  Intrinsics: d(u, v)/df = d (x, y) and
 *    d(u, v)/dk = f r^2 (x, y).
 * 4'. Gauge as pinned rows.  fixed_tx is not read.  A camera is free (enters the reduced system) when any of its 8 parameters is
 *    free, and pin [num_free, 8] uint8 marks its pinned parameters: rows 0-5 for a camera whose pose is fixed, row 3 for a fixed
 *    t_x, row 6 for a fixed f, row 7 for a fixed k.  Each pinned row and column of S becomes the identity with a zero right-hand
 *    side, so its step is exactly 0, and the trial camera copies a pinned parameter (all of R when rows 0-2 are pinned).
 * 6'. Trial.  result[2] also counts the used observations whose camera's trial f is not > 0, so such a trial is rejected.  A free
 *    camera without used observations has a zero step.
 * Shapes for model 1: W [num_elements, 24] (8 x 3), cam_sys [num_free, 16] = g_c (8), D_c (8), S [8 num_free, 8 num_free], rhs
 * [8 num_free].  Device bytes: RB_BA_ELEMENT_BYTES1 E + RB_BA_TRACK_BYTES T + RB_BA_IMAGE_BYTES1 N + RB_BA_FREE_BYTES1 F + 512 F^2
 *   + 1024 ceil(E / RB_TRACKS_TILE) + RB_BA_ONCE_BYTES
 *   per element W 192 (the rest as above); per image cams 128, cams_trial 128; per free camera cam_sys 128, rhs 64, free_cams 4,
 *   pin 8 (no fixed_tx).
 *
 * Shared intrinsics (model 1, rb_ba_groups_args).  Each image belongs to a camera group, and the images of a group share f and k;
 * each keeps its own pose and the principal point stays fixed.  With J the per-image Jacobian above and P the 8F x n' matrix that
 * maps a free camera's pose rows to its own 6 parameters and its f, k rows to its group's, the shared Jacobian is J P.  Hence:
 * 4''. Gauge.  A camera is free when its pose is free or its group's intrinsics are.  pin keeps the pose pins of rule 4' and gives
 *    every member its group's f, k pins; group_pin [num_groups, 2] uint8 pins the group's (f, k) rows after the fold.  A free camera
 *    without observations (an image whose pose is pinned) gets its group's step.
 * 5''. Fold.  S' = P^T S P and b' = P^T b of order n' = 6F + 2G: the free cameras' pose rows at 6 fi, then group g's (f, k) rows at
 *    6F + 2g.  S and b are those of romab200_ba_cameras; the point blocks are unchanged, so the Schur reduction commutes with P.
 *    The group's damping is the sum of its members' clamped diagonals, sum_i clamp(U_i[f, f]) (Ceres clamps the sum; the two
 *    differ only for a member whose diagonal is below 1e-6).  A pinned group row and column become the identity with a zero
 *    right-hand side.  After the Cholesky solve, d = P d' (unfold) and romab200_ba_step runs unchanged; its per-member pred sums
 *    to the group's term up to rounding.
 * The G groups are those with a free camera, ascending by id; group_offsets [G + 1] int32 indexes group_members [F] int32, the
 * free camera indices (fi) of each group, ascending.  The groups path has its own argument struct, rb_ba_groups_args, whose S, rhs
 * and result are the rb_ba_args buffers of the same call; rb_ba_args is unchanged.  A trial is romab200_ba_cameras,
 * romab200_ba_fold, romab200_ba_groups_cholesky, romab200_ba_unfold, romab200_ba_step; without groups it is the model-1 trial above
 * and launches nothing new.
 * romab200_ba_fold: a thread per entry of S' in a pose column (pose-pose copies, group-pose sums over the members in list order)
 *   and of b'; then a CTA per group pair (g, h <= g), whose 2 x 2 block sums the |g| |h| member pairs in a fixed-order tree.
 *   Only the lower triangle of S and S' is read and written.
 * romab200_ba_groups_cholesky: the Cholesky factorisation and both substitutions of romab200_ba_cholesky (the same kernels), on
 *   S_groups and rhs_groups of order n'; a pivot that is not > 0 and finite sets result[3].
 * romab200_ba_unfold: a CTA per group writes rhs [8F] of its members from rhs_groups.
 * Device bytes of the groups path: those of model 1 plus 8 (6F + 2G)^2 + 8 (6F + 2G) + 4 (G + 1) + 4 F + 2 G (S_groups,
 *   rhs_groups, group_offsets, group_members, group_pin). */
#define RB_BA_BAD_ID 1
#define RB_BA_REPEATED 2
#define RB_BA_CAM 21
#define RB_BA_TRACK 13
#define RB_BA_RESULT 4
#define RB_BA_NB 32
#define RB_BA_ELEMENT_BYTES 169
#define RB_BA_TRACK_BYTES 193
#define RB_BA_IMAGE_BYTES 364
#define RB_BA_FREE_BYTES 149
#define RB_BA_ONCE_BYTES 76
#define RB_BA_CAM1 16
#define RB_BA_ELEMENT_BYTES1 217
#define RB_BA_IMAGE_BYTES1 284
#define RB_BA_FREE_BYTES1 204
typedef struct {
    int32_t num_tracks, num_images, num_free;
    const int64_t* track_offsets; const int32_t* elements; int64_t num_elements;
    const int64_t* kp_offsets; const float* keypoints; int64_t num_rows;
    const uint8_t* track_ok; const uint8_t* inlier;
    const int32_t* free_index; const int32_t* free_cams; const uint8_t* fixed_tx;
    double loss_scale2;                                                 /* c^2, or 0 for the squared loss */
    double lambda;
    int64_t* info;                                                      /* [2] status, used observations */
    int32_t* elem_track; uint64_t* keys; uint64_t* keys_alt; int32_t* hist; int64_t* obs_offsets; int32_t* obs;
    const double* cams; const double* X;                                /* the current state */
    double* cams_trial; double* X_trial;
    double* W; double* track_sys; double* cam_sys; double* S; double* rhs;
    double* cam_pred; double* track_part; double* result;
    double* error;
    int32_t camera_model;                                               /* 0 PINHOLE, 1 SIMPLE_RADIAL */
    const uint8_t* pin;                                                 /* [num_free, 8], model 1 */
} rb_ba_args;
int romab200_ba_setup(const rb_ba_args* args, void* stream);
int romab200_ba_linearize(const rb_ba_args* args, void* stream);
int romab200_ba_cameras(const rb_ba_args* args, void* stream);
int romab200_ba_cholesky(const rb_ba_args* args, void* stream);
int romab200_ba_step(const rb_ba_args* args, void* stream);
int romab200_ba_cost(const rb_ba_args* args, void* stream);
int romab200_ba_error(const rb_ba_args* args, void* stream);
typedef struct {
    int32_t num_free, num_groups;                                       /* F free cameras, G groups with a free camera */
    const int32_t* group_offsets; const int32_t* group_members;         /* [G + 1], [F] */
    const uint8_t* group_pin;                                           /* [G, 2] */
    const double* S; double* rhs;                                       /* rb_ba_args' S [8F, 8F] and rhs [8F] */
    double* S_groups; double* rhs_groups;                               /* [n', n'], [n'], n' = 6F + 2G */
    double* result;                                                     /* rb_ba_args' result: [3] is the pivot flag */
} rb_ba_groups_args;
int romab200_ba_fold(const rb_ba_groups_args* args, void* stream);
int romab200_ba_groups_cholesky(const rb_ba_groups_args* args, void* stream);
int romab200_ba_unfold(const rb_ba_groups_args* args, void* stream);

/* ---- absolute pose: batched P3P RANSAC and Gauss-Newton refinement (COLMAP's EstimateAbsolutePose + RefineAbsolutePose) ----
 * Not in the reference.  B items with ragged point counts, packed: item b owns points [offsets[b], offsets[b+1]), each a pixel x
 * [total, 2] and a world point X [total, 3], and its intrinsics K [batch, 3, 3], with the camera model x ~ K (R X + t).  All
 * arithmetic is float64.  The rules:
 * 1. Bearings.  For each point, f = normalise(K^-1 [x, y, 1]), K^-1 by cofactors over the determinant.
 * 2. Samples.  Hypothesis h draws 3 distinct indices with ransac_draw<3> (geometry.cuh) under key seed and counter
 *    (h, s, 0, RB_ABS_CTR), s = 0, 1, ...  The counter does not name the item, so item b is bit-identical to a call on that item
 *    alone, whatever the batch and its order.
 * 3. Minimal solver.  Lambda Twist P3P (Persson & Nordberg, ECCV 2018) on the three bearings f_i and world points X_i: with
 *    a_ij = |X_i - X_j|^2 and b_ij = f_i . f_j, D1 = a23 M12 - a12 M23 and D2 = a23 M13 - a13 M23 (M_ij the quadratic form of
 *    l_i^2 + l_j^2 - 2 b_ij l_i l_j), of the real roots g of det(D1 + g D2) = 0 (Cardano or the trigonometric form, two Newton
 *    steps each; descending) whose D0 = D1 + g D2 is indefinite (cyclic Jacobi; its two eigenvalues of largest magnitude have
 *    opposite signs), the one with the largest ratio of their magnitudes is used, the first on a tie: it keeps clear of a
 *    semidefinite D0, whose lines are complex.  Let sigma1 > 0 > sigma2 be those eigenvalues, with eigenvectors u1, u2 signed so that
 *    their first largest-magnitude entry is positive.  Its lines n = u1 - s u2, then u1 + s u2 (s = sqrt(-sigma2 / sigma1)) give
 *    l1 = w0 l2 + w1 l3 (w = -(n1, n2) / n0); on each, the roots tau > 0 of the quadratic v^T D2 v, v = (w0 + w1 tau, 1, tau), in
 *    ascending order, give l2 = sqrt(a23 / (tau^2 - 2 b23 tau + 1)), l3 = tau l2, kept when l1 > 0.  The depths are then polished
 *    by at most RB_ABS_POLISH_ITERS Newton steps on the three residuals l_i^2 + l_j^2 - 2 b_ij l_i l_j - a_ij (a step kept only if
 *    it lowers their sum of squares), and with Y_i = l_i f_i, R = [Y1 - Y2, Y1 - Y3, (Y1 - Y2) x (Y1 - Y3)] [X1 - X2, X1 - X3,
 *    (X1 - X2) x (X1 - X3)]^-1 and t = Y1 - R X1.  A solution that is not finite is dropped; every other one is a model, so a
 *    sample gives up to RB_ABS_MAX_SOL models.  The 4th-point disambiguation of OpenCV's P3P is not used.
 * 4. Support.  Point j is an inlier of (R, t) when its depth (R X_j + t)_z > 0 and |pi(K (R X_j + t)) - x_j|^2 <= max_error2
 *    (pi(p) = (p_0 / p_2, p_1 / p_2)).  The best model has the most inliers, and at least 3; ties go to the smallest
 *    (h, solution index).  The loop is OpenCV's: the best changes iff count > max(best, 2), then niters =
 *    RANSACUpdateNumIters(conf, (n - count) / n, 3, niters) (ransac_update_num_iters<3>), and it stops at h >= niters; it is
 *    replayed one hypothesis at a time, so the stopping point does not depend on the round size.
 * 5. Refine.  Over the best model's inliers, at most RB_ABS_GN_ITERS Gauss-Newton steps on their summed squared reprojection
 *    error: the update is R <- Exp(d_omega) R, t <- t + d_t, with Exp as in bundle rule 3, and (J^T J) d = -J^T r is solved by
 *    Cholesky.  A step is kept only if it lowers the cost and every used depth stays > 0; the first rejected step (or a pivot that
 *    is not > 0 and finite) stops.  Then the inlier set is recomputed once against the refined pose by rule 4.
 * 6. Output.  ok[b] = 1 when a model exists; an item with fewer than 3 points has none.  R [batch, 3, 3], t [batch, 3], num_inliers
 *    [batch] int64 and mask [total] uint8 are zero where ok is 0.
 * 7. Determinism.  Integer counts, no float atomics, and every reduction in a fixed order, so reruns are byte-identical.
 *   romab200_abspose_hypotheses  one thread per hypothesis of round `round`: rules 1-3.
 *   romab200_abspose_score       thread = (hypothesis, solution slot), the model in registers, the item's points streamed through
 *                                shared memory; grid.y cuts the points into slices whose integer partial counts `select` adds.
 *   romab200_abspose_select      one thread per item replays rule 4's loop over the round and sets running[0] when an item needs
 *                                another round.
 *   romab200_abspose_refine      one CTA per item: rule 5, the 6 x 6 normal equations and the cost summed by cta_sum (a fixed
 *                                order), then rule 6.
 * The caller zero-fills `state` before round 0 and calls hypotheses / score / select for rounds 0, 1, ... while running[0] != 0 and
 * round * RB_ABS_ROUND < max_iters, then refine once.  With max_iters <= RB_ABS_ROUND nothing is read back. */
#define RB_ABS_ROUND 256
#define RB_ABS_MAX_SOL 4
#define RB_ABS_MAX_SPLITS 16
#define RB_ABS_SLICE 1024
#define RB_ABS_GN_ITERS 10
#define RB_ABS_POLISH_ITERS 5
#define RB_ABS_CTR 0x41425300u
#define RB_ABS_MAX_BATCH 16383  /* the score's grid.z holds batch * RB_ABS_MAX_SOL */
#define RB_ABS_STATE 8        /* state[b, :]: iter, niters, best count, best hypothesis, best solution, running, n, unused */
typedef struct {
    int32_t batch;
    const double* x;                      /* [total, 2] pixels */
    const double* X;                      /* [total, 3] world points */
    const int64_t* offsets;               /* [batch + 1] */
    const double* K;                      /* [batch, 3, 3] */
    int64_t max_n;                        /* largest item (sizes the point slices of the score) */
    double max_error2, conf;
    int32_t max_iters, round;
    uint64_t seed;
    int32_t* sample;                      /* [batch, RB_ABS_ROUND, 3] drawn indices of the round */
    double* models;                       /* [batch, RB_ABS_ROUND, RB_ABS_MAX_SOL, 12] R (row-major), t of the round */
    int32_t* nsol;                        /* [batch, RB_ABS_ROUND] */
    int32_t* counts;                      /* [batch, splits, RB_ABS_MAX_SOL, RB_ABS_ROUND] partial inlier counts, splits =
                                             max(1, min(RB_ABS_MAX_SPLITS, ceil(max_n / RB_ABS_SLICE))) */
    int32_t* state;                       /* [batch, RB_ABS_STATE] */
    double* best;                         /* [batch, 12] the best model of the loop */
    int32_t* running;                     /* [1] */
    double* R; double* t;                 /* [batch, 3, 3], [batch, 3] */
    uint8_t* ok;                          /* [batch] */
    int64_t* num_inliers;                 /* [batch] */
    uint8_t* mask;                        /* [total] */
} rb_abspose_args;
int romab200_abspose_hypotheses(const rb_abspose_args* args, void* stream);
int romab200_abspose_score(const rb_abspose_args* args, void* stream);
int romab200_abspose_select(const rb_abspose_args* args, void* stream);
int romab200_abspose_refine(const rb_abspose_args* args, void* stream);

/* ---- image registration: the correspondences of listed images against triangulated tracks, gathered for the absolute-pose
 *      estimator ----
 * Not in the reference.  The input is a match graph's kp_offsets [num_images + 1] int64 and keypoints [K, 2] fp32, the tracks
 * (track_offsets, elements) and per track ok [num_tracks] uint8 and X [num_tracks, 3] float64.  The correspondences of image i are the
 * elements (i, a) of tracks k with ok[k], in element order; each has x = keypoints[kp_offsets[i] + a] widened to float64 and X = X[k].
 * Every element's ids are checked, 0 <= i < num_images and 0 <= a < K_i, and a bad one sets RB_REG_BAD_ID in info[0]; the caller reads
 * it before any kernel indexes with the ids.
 * romab200_register_setup: info [1] int64 is zeroed; a warp per track checks its elements and writes keys (image << 32 | e, image =
 *   num_images for an element of a track that is not ok or of a bad id) [num_elements]; radix_sort_hi32 (common.cuh) sorts them stably
 *   by image (keys_alt, hist RADIX_DIGITS ceil(num_elements / RB_TRACKS_TILE) + 1 int32); image_offsets [num_images + 1] int64 is the
 *   start of each image's correspondences, elem [num_elements] int32 the element ids in sorted order and track [num_elements] int32
 *   the track of every element (by element id).
 * romab200_register_gather: for the chunk's images `images` [num_list] int32, packed at out_offsets [num_list + 1] int64 (the host's
 *   exclusive scan of their counts), x [total, 2] and X [total, 3] float64: the x / X / offsets layout of rb_abspose_args.
 * Device bytes of one estimator chunk of B images with `total` correspondences and S = max(1, min(RB_ABS_MAX_SPLITS,
 * ceil(max_n / RB_ABS_SLICE))) score slices (max_n its largest image), the buffers register.py allocates per chunk:
 *   B (RB_REG_ITEM_BYTES + RB_REG_SLICE_BYTES S) + RB_REG_POINT_BYTES max(total, 1) + RB_REG_CHUNK_BYTES
 *   per item sample 3 072, models 98 304, nsol 1 024, state 32, best 96, R 72, t 24, ok 1, num_inliers 8, K 72, images 4, offsets 8;
 *   per item and slice counts 4 096; per point x 16, X 24, mask 1; once running 4 and offsets 8. */
#define RB_REG_BAD_ID 1
#define RB_REG_ITEM_BYTES 102717
#define RB_REG_SLICE_BYTES 4096
#define RB_REG_POINT_BYTES 41
#define RB_REG_CHUNK_BYTES 12
typedef struct {
    int32_t num_tracks, num_images;
    const int64_t* track_offsets; const int32_t* elements; int64_t num_elements;
    const int64_t* kp_offsets; const float* keypoints; int64_t num_rows;
    const uint8_t* track_ok; const double* points;                     /* [num_tracks], [num_tracks, 3] */
    int64_t* info;                                                      /* [1] status */
    uint64_t* keys; uint64_t* keys_alt; int32_t* hist;
    int64_t* image_offsets; int32_t* elem; int32_t* track;
    int32_t num_list; const int32_t* images; const int64_t* out_offsets;  /* gather only: */
    double* x; double* X;
} rb_register_args;
int romab200_register_setup(const rb_register_args* args, void* stream);
int romab200_register_gather(const rb_register_args* args, void* stream);

/* ---- two-view initialisation: statistics of a candidate pair's relative pose (COLMAP's EstimateInitialTwoViewGeometry) ----
 * Not in the reference.  It runs after the relative-pose estimator (romab200_pose_*) on a batch of candidate pairs and reads that
 * call's buffers: offsets [batch + 1], xn [total, 4] (the normalised points the estimator wrote), mask [total], R [batch, 3, 3],
 * t [batch, 3] (unit length), ok [batch] and K [batch, 2, 3, 3], with the gathered pixels x0, x1 [total, 2].  All arithmetic is
 * float64.  The rules:
 * 1. Points.  Only the matches with mask set are used: the RANSAC inliers that passed recoverPose's chirality test.  Each is
 *    triangulated by the DLT of the chirality test (dlt_two_view, geometry.cuh) with P0 = [I | 0] and P1 = [R | t] on xn: the
 *    homogeneous Q, and X = Q.xyz / Q.w.
 * 2. Good point.  A point is good when Q.w != 0 and X is finite, X.z > 0 and (R X + t).z > 0, and the squared reprojection error in
 *    pixels is <= max_error2 in both images: |pi(K_0 X) - x0|^2 and |pi(K_1 (R X + t)) - x1|^2, pi(p) = (p_0 / p_2, p_1 / p_2).
 * 3. Angle.  The triangulation angle of a good point is atan2(|a x b|, a . b) with a = X - C0 = X and b = X - C1, C1 = -R^T t
 *    (triangulation rule 6's formula), in degrees (times 180 / pi).
 * 4. Outputs per candidate.  num_good [batch] int64, median_angle [batch] float64 degrees and forward [batch] = |t_z|.
 *    median_angle is the median of the good points' angles: the mean of the two middle values for an even count (numpy's and
 *    COLMAP's Median), and 0 when there are none.  A candidate with ok = 0 has no masked matches, so num_good = 0 there.
 * 5. Median without a sort.  The k-th smallest angle is found exactly by a radix select on its IEEE-754 bits: the angles are
 *    non-negative, so their bit patterns order like their values.  8-bit digits from the top, one shared-memory histogram of
 *    integer counts per digit over the per-point scratch angle [max(total, 1)] float64 that the first pass writes (-1 for a point
 *    that is not good).
 * 6. Determinism.  No float atomics and integer counts only, so reruns are byte-identical.
 * romab200_twoview_score: one CTA of 256 threads per candidate. */
typedef struct {
    int32_t batch;
    const int64_t* offsets;               /* [batch + 1] */
    const double* x0; const double* x1;   /* [total, 2] pixels */
    const double* xn;                     /* [total, 4] */
    const uint8_t* mask;                  /* [total] */
    const double* K;                      /* [batch, 2, 3, 3] */
    const double* R; const double* t;     /* [batch, 3, 3], [batch, 3] */
    const uint8_t* ok;                    /* [batch] */
    double max_error2;
    double* angle;                        /* [max(total, 1)] scratch */
    int64_t* num_good; double* median_angle; double* forward;   /* [batch] */
} rb_twoview_args;
int romab200_twoview_score(const rb_twoview_args* args, void* stream);

/* ---- keypoint undistortion under SIMPLE_RADIAL cameras (COLMAP's camera model 2) ----
 * Not in the reference.  Camera i has intrinsics [num_images, 4] float64 (f, cx, cy, k) and maps a camera-frame point p to
 * x = p0 / p2, y = p1 / p2, r^2 = x^2 + y^2, d = 1 + k r^2, u = f d x + cx, v = f d y + cy.  Each keypoint (u, v) of image i,
 * keypoints[kp_offsets[i] .. kp_offsets[i + 1]), is mapped to the pixel of the same camera without distortion.  All arithmetic is
 * float64 on the keypoint widened from fp32.  The rules:
 * 1. Normalise.  (dx, dy) = (u - cx, v - cy) and rho_d = sqrt(dx^2 + dy^2) / f.
 * 2. Solve rho (1 + k rho^2) = rho_d by Newton from rho = rho_d: step = (rho (1 + k rho^2) - rho_d) / (1 + 3 k rho^2), rho -= step,
 *    at most RB_UNDISTORT_ITERS steps, stopping after a step that is exactly 0.  g(rho) = rho (1 + k rho^2) - rho_d is convex on
 *    rho > 0 for k > 0 and concave for k < 0, so the iterates move monotonically towards the root from rho_d.
 * 3. Output (cx + dx s, cy + dy s) with s = rho / rho_d, rounded to fp32.  With k = 0 or rho_d = 0 the keypoint is copied bit for bit.
 * 4. For k < 0, g has no root at or beyond rho_d >= 2 / (3 sqrt(-3 k)), the image of the turning radius 1 / sqrt(-3 k).  Such a
 *    keypoint gets rho = 1 / sqrt(-3 k) (clamped in its own direction) and counts in clamped[0].  No output is NaN.
 * The caller checks on the host that every f is finite and > 0 and every cx, cy, k finite.
 * romab200_undistort_keypoints: a thread per keypoint; clamped [1] int64 is zeroed and counted with integer atomics. */
#define RB_UNDISTORT_ITERS 20
typedef struct {
    int32_t num_images;
    int64_t num_rows;
    const int64_t* kp_offsets;            /* [num_images + 1] */
    const float* keypoints;               /* [num_rows, 2] */
    const double* intrinsics;             /* [num_images, 4] */
    float* out;                           /* [num_rows, 2] */
    int64_t* clamped;                     /* [1] */
} rb_undistort_args;
int romab200_undistort_keypoints(const rb_undistort_args* args, void* stream);

/* ---- dense reconstruction: per-image depth maps triangulated from dense warps, fused into a point cloud ----
 * Not in the reference.  The input is what match_pairs returns for the rows first_pair .. first_pair + chunk of pairs [num_pairs, 2]
 * int64: warp [chunk, H, 2W, 4] and certainty [chunk, H, 2W] fp32, symmetric.  Element (r, c) of the left half is grid pixel (r, c)
 * of image pairs[k][0], matched at warp[..., 2:4] in image pairs[k][1]; element (r, W + c) of the right half is grid pixel (r, c) of
 * image pairs[k][1], matched at warp[..., 0:2] in image pairs[k][0].  k = first_pair + row is the global pair index, half 0 / 1 the
 * side, g = 2 k + half names the element's pair-half.  image_sizes [num_images, 2] int32 (H_img, W_img) is the pixel frame of the
 * cameras; cameras [num_images, RB_DENSE_CAM] float64 per image: K (9, row-major), K^-1 (9, computed on the host), R (9), t (3),
 * SIMPLE_RADIAL (f, cx, cy, k) (4), 2 unused; x ~ K (R X + t).  All geometry is float64.  The rules of one element:
 * 1. Grid side.  x = W_img (c + 0.5) / W, y = H_img (r + 0.5) / H in the grid image's frame, evaluated left to right.
 * 2. Match side.  (u, v) read from the warp; x = (W_img / 2) * (u + 1), y = (H_img / 2) * (v + 1), each operation rounded to fp32
 *    (consolidate_matches' rule), then widened.
 * 3. Rejection, in this order, the first failure being the element's reason: 1 certainty <= min_certainty or any of the certainty,
 *    u, v not finite; 2 u or v outside [-1, 1]; 3 either image not registered; 4 (radial only) either position clamped by the
 *    undistortion; 5 the point not in front of both cameras (Q_w = 0, or either depth not > 0, NaN included); 6 the squared
 *    reprojection error in px in either image > max_error2; 7 the triangulation angle < min_angle (radians).  Reason 0 is accepted.
 * 4. Normalised coordinates.  Pinhole: h = K^-1 (x, y, 1), (h0 / h2, h1 / h2).  radial = 1: (dx, dy) = (x - cx, y - cy), rho_d =
 *    |(dx, dy)| / f and (dx s / f, dy s / f) with s = rho / rho_d from the Newton loop of the keypoint undistortion below (s = 1 when
 *    k = 0 or rho_d = 0); clamped positions are reason 4.
 * 5. Triangulation.  dlt_two_view (geometry.cuh) with the relative pose R_m R_g^T, t_m - R_m R_g^T t_g (g the grid image, m the match
 *    image) gives Q; X = Q.xyz / Q.w in the grid camera's frame and X_m = R_rel X + t_rel.  Reprojection: pinhole pi(K X), radial
 *    the forward model (f d x + cx, f d y + cy), each against the position of rule 1 / 2 (the raw, distorted pixel).  Angle:
 *    atan2(|a x b|, a . b) with a = X and b = X - C_m, C_m = -R_rel^T t_rel.  The depth is X.z rounded to fp32.
 * 6. Winner.  A grid pixel keeps the accepted element with the largest certainty, ties to the smallest g: the 64-bit integer maximum
 *    of key = (certainty bits << 32) | ~g (uint32), over every call that accumulates into the same maps, so the maps do not depend on
 *    chunking, pair order or arrival order.  depth, score [num_images, H, W] fp32 and source [num_images, H, W] int64 hold the winner's
 *    depth, certainty and g (0, 0, -1 where none).
 * romab200_dense_triangulate: source and score of the listed images `images` [num_list] int32 (every image the chunk references, each
 *   once) are packed into keys in place (source holds key, 0 for none); one thread per (pair-half, pixel) with grid.y = 2 row + half
 *   classifies its element, writes elem_depth [chunk, 2, H, W] (0 unless accepted) and takes the atomicMax of its key; the reason
 *   counts go through warp reductions into partial [2 chunk, RB_DENSE_MAX_CTAS, RB_DENSE_REASONS] int32, and one more kernel adds them
 *   per pair in a fixed order to pair_counts [num_pairs, RB_DENSE_REASONS] int64 (row k: accepted, then reasons 1-7).
 * romab200_dense_resolve (same arguments, after triangulate): every accepted element whose key won writes its depth, then the listed
 *   images' keys are unpacked back to source and score.  Between the two calls source holds keys.
 *
 * Fusion.  Neighbours of image i: nbrs[nbr_offsets[i] .. nbr_offsets[i + 1]) int32, the registered images sharing a pair with i in
 * ascending order (built on the host).  For grid pixel p = (r, c) of a registered image i with depth d > 0:
 * F1. X = R_i^T (d (a, b, 1) - t_i) with (a, b) the normalised coordinates (rule 4) of p's position (rule 1); a clamped p is skipped.
 * F2. Per neighbour j in order: X_j = R_j X + t_j; skip unless X_j.z > 0; (u, v) its pixel, q = (floor(v H / H_j), floor(u W / W_j));
 *     q agrees when it lies inside the grid, d_q = depth_j(q) > 0, |d_q - X_j.z| <= max_depth_error X_j.z, q's position is not
 *     clamped, and Y = R_j^T (d_q (a', b', 1) - t_j) (F1 for q) has R_i Y + t_i in front of i and projects within max_reproj_error
 *     (squared: max_reproj_error2) of p's position.
 * F3. p is kept when at least min_num_views - 1 neighbours agree, and emitted when also no agreeing neighbour has an index < i.  The
 *     point is (X + the agreeing Y in neighbour order) / (1 + agreeing), num_views = 1 + agreeing, score = score_i(p), image i,
 *     pixel r W + c, colour the pixel (((2 r + 1) H_c) / (2 H), ((2 c + 1) W_c) / (2 W)) (integer division) of image i's colour
 *     image [H_c, W_c, 3] uint8 at colors + color_offsets[i] (color_sizes [num_images, 2] int32, color_bytes the buffer's size), or
 *     128 grey when colors is null.
 * romab200_dense_fuse_count: one CTA per tile of RB_DENSE_TILE pixels of one image (tiles = ceil(H W / RB_DENSE_TILE) per image,
 *   image-major) counts its emitted pixels into tile_scan [num_images tiles + 1] int64, then scans it (exclusive, total last).
 * romab200_dense_fuse_emit (after the caller has read the total into num_points): the same CTAs write points [num_points, 3] float64,
 *   rgb [num_points, 3] uint8, image int32, pixel int64, num_views int32 and point_score fp32 at their offsets, pixels in order. */
#define RB_DENSE_CAM 36
#define RB_DENSE_REASONS 8
#define RB_DENSE_MAX_CTAS 256
#define RB_DENSE_TILE 256
typedef struct {
    const int64_t* pairs; int32_t num_pairs, num_images;
    int32_t first_pair, chunk, H, W;
    const float* warp; const float* certainty;
    const int32_t* image_sizes; const double* cameras; const uint8_t* registered; int32_t radial;
    float min_certainty; double max_error2, min_angle;
    const int32_t* images; int32_t num_list;
    float* depth; float* score; int64_t* source;
    float* elem_depth; int32_t* partial; int64_t* pair_counts;
} rb_dense_tri_args;
int romab200_dense_triangulate(const rb_dense_tri_args* args, void* stream);
int romab200_dense_resolve(const rb_dense_tri_args* args, void* stream);

typedef struct {
    int32_t num_images, H, W;
    const int32_t* image_sizes; const double* cameras; const uint8_t* registered; int32_t radial;
    const int64_t* nbr_offsets; const int32_t* nbrs;
    const float* depth; const float* score;
    double max_reproj_error2, max_depth_error; int32_t min_num_views;
    const uint8_t* colors; const int64_t* color_offsets; const int32_t* color_sizes; int64_t color_bytes;
    int64_t* tile_scan;
    int64_t num_points;                                                 /* emit only: */
    double* points; uint8_t* rgb; int32_t* image; int64_t* pixel; int32_t* num_views; float* point_score;
} rb_dense_fuse_args;
int romab200_dense_fuse_count(const rb_dense_fuse_args* args, void* stream);
int romab200_dense_fuse_emit(const rb_dense_fuse_args* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ROMAB200_H */
