"""Parity mode on the tensor cores: RB_F16S (split fp16 pair) operands through the tensor-core back-end of romab200_gemm must
reproduce an fp32 GEMM (error at the fp32 rounding level against a float64 reference), and every kernel that produces or
passes on an RB_F16S matrix must reproduce the value it was given to ~2^-22.

RB_F16S: hi = fp16(x), lo = fp16((x - hi) * 2^11), value = hi + lo * 2^-11 (include/romab200.h)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from roma_b200 import cabi  # noqa: E402
from roma_b200.cabi import call  # noqa: E402
from roma_b200.packing import Split, split_f16s  # noqa: E402

DEV = "cuda"
F32, F16S = cabi.RB_F32, cabi.RB_F16S


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def dev_split(x, rows, cols, ld, row_norm=None):
    hi = torch.full((rows, ld), 7.0, dtype=torch.float16, device=DEV)
    lo = torch.full((rows, ld), 7.0, dtype=torch.float16, device=DEV)
    call("romab200_split_f16s", "rb_split_pair_args", x=x, hi=hi, lo=lo, rows=rows, cols=cols, ldx=x.stride(0), ldd=ld, row_norm=row_norm)
    return Split(hi, lo)


def sgemm(A: Split, B: Split, C, M, N, K, lda, ldb, ldc, **kw):
    args = dict(A=A.hi, A_lo=A.lo, B=B.hi, B_lo=B.lo, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, dtype_ab=F16S,
                batch0=1, batch1=1, ntaps=1, alpha=1.0, backend=cabi.BACKEND_TCGEN05)
    if isinstance(C, Split):
        args.update(C=C.hi, C_lo=C.lo, dtype_c=F16S)
    else:
        args.update(C=C, dtype_c=F32)
    args.update(kw)
    call("romab200_gemm", "rb_gemm_args", **args)


def rel_err(got, ref):
    return ((got.double().cpu() - ref.double().cpu()).abs().max() / ref.double().abs().max()).item()


@pytest.mark.parametrize("scale", [1.0, 1e-3, 200.0])
def test_split_kernel_roundtrip(scale):
    """value -> (hi, lo) on the device equals the host twin and reconstructs x to 2^-21 relative (2^-36 absolute floor)."""
    rows, cols, ld = 301, 1377, 1384
    x = rnd(rows, ld, seed=1, scale=scale)
    x[0, :4] = torch.tensor([0.0, 65000.0, -1e-7, 3e-5], device=DEV)
    s = dev_split(x, rows, cols, ld)
    hi, lo = split_f16s(x[:, :cols].cpu())
    assert torch.equal(s.hi[:, :cols].cpu(), hi) and torch.equal(s.lo[:, :cols].cpu(), lo)
    back = s.join()[:, :cols]
    err = (back - x[:, :cols]).abs()
    assert (err <= x[:, :cols].abs() * 2.0 ** -21 + 2.0 ** -36).all()
    # odd geometry takes the scalar kernel
    y = rnd(17, 13, seed=2)
    s2 = dev_split(y, 17, 13, 16)
    assert torch.equal(s2.hi[:, :13].cpu(), split_f16s(y.cpu())[0])
    nrm = y.norm(dim=1).contiguous()
    s3 = dev_split(y, 17, 13, 16, row_norm=nrm)
    assert (s3.join()[:, :13] - y / nrm[:, None]).abs().max() < 1e-6


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (300, 200, 136), (1000, 24, 24), (257, 4097, 1024), (130, 64, 592), (3200, 1377, 1384),
                                   (500, 9, 64), (20000, 144, 144), (19000, 569, 569), (9000, 1137, 1137), (19000, 130, 72), (19000, 192, 200),
                                   (3202, 1024, 4096), (3202, 3072, 1024)])
def test_split_gemm_is_fp32_class(M, N, K):
    """Every tile width / accumulator schedule of the SPLIT kernel against float64: the error must sit at the level of an
    fp32 GEMM.  The operand representation contributes 2^-22; what remains is the tensor core's own fp32 accumulation, which
    truncates on every accumulator update (one per 16 k), so the bound grows with K / 16 updates of 2^-24 each (measured:
    K = 4096 -> 6e-6 relative to the largest output against 2.8e-6 for cuBLAS fp32)."""
    lda = (K + 7) // 8 * 8
    A, B = rnd(M, lda, seed=1), rnd(N, lda, seed=2, scale=0.05)
    ldc = (N + 3) // 4 * 4
    C = torch.full((M, ldc), 3.0, device=DEV)
    sgemm(dev_split(A, M, K, lda), dev_split(B, N, K, lda), C, M, N, K, lda, lda, ldc)
    ref = A[:, :K].double() @ B[:, :K].double().t()
    e_split = rel_err(C[:, :N], ref)
    e_f32 = rel_err(A[:, :K] @ B[:, :K].t(), ref)
    assert e_split <= e_f32 + 2.0 ** -20 + 0.5 * (K / 16) * 2.0 ** -24, (e_split, e_f32)
    if ldc > N:       # pad columns: untouched beyond the 16-byte granule of the row tail (TMA clipping granularity), zeros or untouched inside it
        gran = (N + 3) // 4 * 4
        assert (C[:, gran:] == 3.0).all() and ((C[:, N:gran] == 3.0) | (C[:, N:gran] == 0.0)).all()


def test_split_gemm_small_magnitudes():
    """The 2^11-scaled low plane keeps full precision for small operands (an unscaled fp16 low part would underflow)."""
    M, N, K = 512, 256, 512
    A, B = rnd(M, K, seed=1, scale=1e-3), rnd(N, K, seed=2, scale=1e-3)
    C = torch.zeros(M, N, device=DEV)
    sgemm(dev_split(A, M, K, K), dev_split(B, N, K, K), C, M, N, K, K, K, N)
    ref = A.double() @ B.double().t()
    assert rel_err(C, ref) < 2e-6


def test_split_gemm_epilogues_and_split_output():
    M, N, K = 391, 264, 320
    A, B = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.1)
    bias, gamma, X = rnd(N, seed=3), rnd(N, seed=4), rnd(M, N, seed=5)
    sa, sb = dev_split(A, M, K, K), dev_split(B, N, K, K)
    base = (A.double() @ B.double().t() + bias.double())
    out = Split(torch.zeros(M, N, dtype=torch.float16, device=DEV), torch.zeros(M, N, dtype=torch.float16, device=DEV))
    sgemm(sa, sb, out, M, N, K, K, K, N, bias=bias, act=cabi.ACT_GELU)
    assert rel_err(out.join(), F.gelu(base)) < 3e-6
    sgemm(sa, sb, out, M, N, K, K, K, N, bias=bias, act=cabi.ACT_RELU)
    assert rel_err(out.join(), F.relu(base)) < 3e-6
    ref = X.double() + base * gamma.double()
    sgemm(sa, sb, X, M, N, K, K, K, N, bias=bias, col_scale=gamma, R=X, ldr=N, dtype_r=F32)
    assert rel_err(X, ref) < 3e-6
    # ragged split output (N not a multiple of 8, pitch padded): the scalar tail path
    N2 = 251
    out2 = Split(torch.full((M, 256), 5.0, dtype=torch.float16, device=DEV), torch.full((M, 256), 5.0, dtype=torch.float16, device=DEV))
    sgemm(sa, Split(sb.hi[:N2], sb.lo[:N2]), out2, M, N2, K, K, K, 256, alpha=0.5)
    assert rel_err(out2.join()[:, :N2], 0.5 * (A.double() @ B[:N2].double().t())) < 3e-6
    gran = (N2 + 7) // 8 * 8            # 16-byte granule of the fp16 planes
    assert (out2.hi[:, gran:] == 5.0).all() and (out2.lo[:, gran:] == 5.0).all()


@pytest.mark.parametrize("d,N", [(64, 203), (128, 160), (64, 1601)])
def test_split_attention_chain(d, N):
    """QK^T (batched, strided) -> softmax written as a pair -> PV with the MN-major B operand, all on RB_F16S operands."""
    Bn, H = 2, 3
    dim = H * d
    qkv32 = rnd(Bn * N, 3 * dim, seed=1, scale=0.7)
    qkv = dev_split(qkv32, Bn * N, 3 * dim, 3 * dim)
    npad = (N + 7) // 8 * 8
    S = torch.zeros(Bn, H, N, npad, device=DEV)
    ld = 3 * dim
    sgemm(qkv, qkv.at(dim), S, N, N, d, ld, ld, npad, batch0=Bn, batch1=H, alpha=1.0 / math.sqrt(d),
          sa0=N * ld, sa1=d, sb0=N * ld, sb1=d, sc0=H * N * npad, sc1=N * npad)
    q, k, v = qkv32.double().reshape(Bn, N, 3, H, d).unbind(2)
    ref = torch.einsum("bnhd,bmhd->bhnm", q, k) / math.sqrt(d)
    assert rel_err(S[..., :N], ref) < 2e-6
    P = Split(torch.zeros(Bn, H, N, npad, dtype=torch.float16, device=DEV), torch.zeros(Bn, H, N, npad, dtype=torch.float16, device=DEV))
    call("romab200_softmax_rows", "rb_softmax_args", s=S, rows=Bn * H * N, cols=N, lds=npad, dtype=F32, scale=1.0, out_hi=P.hi, out_lo=P.lo, ldo=npad)
    pref = torch.softmax(ref, dim=-1)
    assert (P.join()[..., :N].double().cpu() - pref.cpu()).abs().max() < 5e-7
    O = Split(torch.zeros(Bn * N, dim, dtype=torch.float16, device=DEV), torch.zeros(Bn * N, dim, dtype=torch.float16, device=DEV))
    sgemm(P, qkv.at(2 * dim), O, N, d, N, npad, ld, dim, trans_b=1, batch0=Bn, batch1=H,
          sa0=H * N * npad, sa1=N * npad, sb0=N * ld, sb1=d, sc0=N * dim, sc1=d)
    ref_o = torch.einsum("bhnm,bmhd->bnhd", pref, v).reshape(Bn * N, dim)
    assert rel_err(O.join(), ref_o) < 3e-6


@pytest.mark.parametrize("halves", [1, 2])
@pytest.mark.parametrize("N,scale", [(203, 0.7), (1601, 0.7), (128, 3.0), (64, 0.05), (1, 1.0), (33, 1.0), (97, 0.7)])
def test_split_flash_attention(N, scale, halves):
    """Fused split-fp16 attention (head_dim 64) against float64 SDPA: fp32-class, incl. ragged last key tile (N = 1, 33, 97
    leave most of a 64-key tile empty), peaked (scale 3) and flat (scale 0.05) score distributions.  halves = 2 runs the
    two-image batch as two one-image calls on offset views of the same buffers (tensor maps and outputs not at the base)."""
    Bn, H, d = 2, 3, 64
    dim = H * d
    qkv32 = rnd(Bn * N, 3 * dim, seed=1, scale=scale)
    qkv = dev_split(qkv32, Bn * N, 3 * dim, 3 * dim)
    O = Split(torch.full((Bn * N, dim), 9.0, dtype=torch.float16, device=DEV), torch.full((Bn * N, dim), 9.0, dtype=torch.float16, device=DEV))
    per_call = Bn if halves == 1 else 1
    for i in range(0, Bn, per_call):
        r = slice(i * N, (i + per_call) * N)
        call("romab200_flash_attn", "rb_flash_attn_args", qkv=qkv.hi[r], qkv_lo=qkv.lo[r], out=O.hi[r], out_lo=O.lo[r], ld_qkv=3 * dim, ld_out=dim,
             batch=per_call, n_tokens=N, heads=H, head_dim=d, dtype=F16S)
    q, k, v = qkv32.double().reshape(Bn, N, 3, H, d).unbind(2)
    ref = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2).reshape(Bn * N, dim)
    f32 = F.scaled_dot_product_attention(q.float().transpose(1, 2), k.float().transpose(1, 2), v.float().transpose(1, 2)).transpose(1, 2).reshape(Bn * N, dim)
    e_split, e_f32 = rel_err(O.join(), ref), rel_err(f32, ref)
    print(f"flash split N={N}: rel err {e_split:.2e} (torch fp32 SDPA: {e_f32:.2e})")
    # ~N/16 truncating accumulator updates per output (the tensor core's fp32 accumulation rounds toward zero): 6e-6 at N = 1601
    assert e_split <= max(4 * e_f32, 2e-6 + N * 3e-9), (e_split, e_f32)


@pytest.mark.parametrize("cin,cout,H,W", [(64, 64, 20, 36), (128, 256, 9, 13)])
def test_split_conv3x3_taps_maxpool(cin, cout, H, W):
    """VGG layer in the parity mode: 9-tap GEMM on a zero-padded RB_F16S map -> RB_F16S map, then the pair-wise max-pool."""
    E = 2
    x, w, b = rnd(E, cin, H, W, seed=1), rnd(cout, cin, 3, 3, seed=2, scale=0.1), rnd(cout, seed=3)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    xp = torch.zeros(E, H + 2, W + 2, cin, device=DEV)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    rows = E * (H + 2) * (W + 2)
    xs = dev_split(xp.view(rows, cin), rows, cin, cin)
    wm = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    ws = dev_split(wm, cout, 9 * cin, 9 * cin)
    out = Split(torch.zeros(E, H + 2, W + 2, cout, dtype=torch.float16, device=DEV), torch.zeros(E, H + 2, W + 2, cout, dtype=torch.float16, device=DEV))
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    sgemm(xs, ws, out, rows, cout, 9 * cin, cin, 9 * cin, cout, ntaps=9, tap_rows=taps, a_rows=rows, bias=b,
          act=cabi.ACT_RELU, rowmap=cabi.ROWMAP_PAD_KEEP, pad_h=H + 2, pad_w=W + 2)
    got = out.join()
    assert rel_err(got[:, 1:-1, 1:-1], ref) < 3e-6
    assert (got[:, 0] == 0).all() and (got[:, :, -1] == 0).all()
    if H % 2 == 0 and W % 2 == 0:
        pooled = Split(torch.zeros(E, H // 2 + 2, W // 2 + 2, cout, dtype=torch.float16, device=DEV),
                       torch.zeros(E, H // 2 + 2, W // 2 + 2, cout, dtype=torch.float16, device=DEV))
        call("romab200_maxpool2x2_padded", "rb_maxpool_args", **{"in": out.hi}, in_lo=out.lo, out=pooled.hi, out_lo=pooled.lo,
             batch=E, height=H, width=W, channels=cout, dtype=F16S)
        refp = F.max_pool2d(got[:, 1:-1, 1:-1].permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
        assert torch.equal(pooled.join()[:, 1:-1, 1:-1], refp)          # pairs are passed through unchanged
        assert (pooled.join()[:, 0] == 0).all()


def test_split_producers_layernorm_convfirst_dwconv():
    # LayerNorm -> pair (vector path: 1024 columns; generic path: 520)
    for cols in (1024, 520):
        x, g, b = rnd(77, cols, seed=1, scale=3.0), rnd(cols, seed=2), rnd(cols, seed=3)
        y = Split(torch.zeros(77, cols, dtype=torch.float16, device=DEV), torch.zeros(77, cols, dtype=torch.float16, device=DEV))
        call("romab200_layernorm", "rb_layernorm_args", x=x, y=y.hi, y_lo=y.lo, gamma=g, beta=b, rows=77, cols=cols, ldx=cols, ldy=cols,
             dtype_x=F32, dtype_y=F16S, eps=1e-6)
        ref = F.layer_norm(x.double(), (cols,), g.double(), b.double(), 1e-6)
        assert (y.join().double() - ref).abs().max() < 2e-5
        y32 = torch.zeros(77, cols, device=DEV)
        call("romab200_layernorm", "rb_layernorm_args", x=x, y=y32, gamma=g, beta=b, rows=77, cols=cols, ldx=cols, ldy=cols,
             dtype_x=F32, dtype_y=F32, eps=1e-6)
        assert (y.join() - y32).abs().max() <= y32.abs().max() * 2.0 ** -21     # the pair carries the fp32 result
    # first VGG conv -> pair
    E, H, W = 2, 12, 20
    img, w, b = rnd(E, 3, H, W, seed=4), rnd(64, 27, seed=5, scale=0.2), rnd(64, seed=6)
    o = Split(torch.zeros(E, H + 2, W + 2, 64, dtype=torch.float16, device=DEV), torch.zeros(E, H + 2, W + 2, 64, dtype=torch.float16, device=DEV))
    call("romab200_conv3x3_first", "rb_conv_first_args", image=img, out=o.hi, out_lo=o.lo, weight=w, bias=b, batch=E, height=H, width=W, cout=64, dtype_out=F16S)
    ref = F.relu(F.conv2d(img.double(), w.double().view(64, 3, 3, 3), b.double(), padding=1)).permute(0, 2, 3, 1)
    assert rel_err(o.join()[:, 1:-1, 1:-1], ref) < 1e-6 and (o.join()[:, 0] == 0).all()
    # depthwise 5x5 (fp32 map) -> pair
    D, h, w_, c, cp = 2, 13, 21, 569, 576
    x = rnd(D, h, w_, cp, seed=7)
    wt, bb = rnd(25, cp, seed=8, scale=0.2), rnd(c, seed=9)
    t = Split(torch.zeros(D * h * w_, cp, dtype=torch.float16, device=DEV), torch.zeros(D * h * w_, cp, dtype=torch.float16, device=DEV))
    call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": x}, out=t.hi, out_lo=t.lo, ldi=cp, ldo=cp, weight=wt, ldw=cp, bias=bb,
         batch=D, h=h, w=w_, c=c, dtype=F32)
    wk = wt[:, :c].t().reshape(c, 1, 5, 5).double()
    ref = F.relu(F.conv2d(x[..., :c].permute(0, 3, 1, 2).double(), wk, bb.double(), padding=2, groups=c)).permute(0, 2, 3, 1)
    assert rel_err(t.join().view(D, h, w_, cp)[..., :c], ref) < 2e-6


def test_split_coskernel_matrix():
    """All-pairs CosKernel from RB_F16S pairs of the L2-normalised rows: fp32-class against float64 (SURVEY Appendix A)."""
    n, c = 1600, 512
    g = torch.Generator().manual_seed(0)
    base = torch.randn(8, c, generator=g)
    x = (torch.randn(n, 8, generator=g) @ base + 0.5 * torch.randn(n, c, generator=g)).to(DEV)
    y = (torch.randn(n, 8, generator=g) @ base + 0.5 * torch.randn(n, c, generator=g)).to(DEV)
    nx, ny = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    call("romab200_row_norms", "rb_rownorm_args", x=x, out=nx, rows=n, cols=c, ldx=c, dtype=F32)
    call("romab200_row_norms", "rb_rownorm_args", x=y, out=ny, rows=n, cols=c, ldx=c, dtype=F32)
    xs, ys = dev_split(x, n, c, c, row_norm=nx), dev_split(y, n, c, c, row_norm=ny)
    K = torch.zeros(n, n, device=DEV)
    sgemm(xs, ys, K, n, n, c, c, c, n, epi=cabi.EPI_COSKERNEL, norm_a=nx, norm_b=ny, eps=1e-6, inv_t=5.0, diag_add=0.1, cos_normalized=1)
    xd, yd = x.double(), y.double()
    cos = (xd @ yd.t()) / (xd.norm(dim=1)[:, None] * yd.norm(dim=1)[None] + 1e-6)
    ref = torch.exp((cos - 1) * 5.0) + 0.1 * torch.eye(n, device=DEV, dtype=torch.float64)
    assert (K.double() - ref).abs().max() < 1.5e-5        # cosine error x 5 (1/T) through the exponential
    Kp = Split(torch.zeros(n, n, dtype=torch.float16, device=DEV), torch.zeros(n, n, dtype=torch.float16, device=DEV))
    sgemm(xs, ys, Kp, n, n, c, c, c, n, epi=cabi.EPI_COSKERNEL, norm_a=nx, norm_b=ny, eps=1e-6, inv_t=5.0, diag_add=0.0, cos_normalized=1)
    assert (Kp.join().double() - (ref - 0.1 * torch.eye(n, device=DEV, dtype=torch.float64))).abs().max() < 1.5e-5


@pytest.mark.parametrize("B,H,W", [(2, 37, 50), (1, 16, 16), (2, 5, 3)])
def test_refiner_block_small_fp32_host_tensors(B, H, W):
    """Fused thin-map block (DW5x5 + ReLU + PW, C = 24) on fp32 maps: fp32 FFMA throughout, against conv2d in float64."""
    C = 24
    x = rnd(B, C, H, W, seed=1)
    dw, db = rnd(C, 1, 5, 5, seed=2, scale=0.3), rnd(C, seed=3)
    pw, pb = rnd(C, C, seed=4, scale=0.3), rnd(C, seed=5)
    mid = F.relu(F.conv2d(x.double(), dw.double(), db.double(), padding=2, groups=C))
    ref = (torch.einsum("bchw,oc->bohw", mid, pw.double()) + pb.double()[None, :, None, None]).permute(0, 2, 3, 1)
    xi = x.permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(B, H, W, C, device=DEV)
    dwt = dw.reshape(C, 25).t().contiguous()
    pw_host, pb_host = pw.cpu().contiguous(), pb.cpu().contiguous()       # host arrays: they travel as kernel parameters
    call("romab200_refiner_block_small", "rb_refiner_block_small_args", **{"in": xi}, out=out, ld=C, dw_weight=dwt, ldw=C, dw_bias=db,
         pw_weight_host=pw_host, pw_bias_host=pb_host, batch=B, h=H, w=W, c=C, dtype=F32)
    assert rel_err(out, ref) < 2e-6


@pytest.mark.parametrize("B,C,H,W", [(2, 150, 19, 37), (1, 64, 8, 16), (2, 569, 54, 54), (1, 70, 5, 3), (2, 24, 33, 20), (1, 144, 40, 48)])
def test_dwconv_fp32_tma_split_out(B, C, H, W):
    """TMA-fed depthwise 5x5 + ReLU on fp32 maps with the RB_F16S result (ragged 16x16 tiles, channel tail, zero-filled
    borders) against conv2d in float64."""
    x = rnd(B, C, H, W, seed=1)
    w, b = rnd(C, 1, 5, 5, seed=2, scale=0.3), rnd(C, seed=3)
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), padding=2, groups=C)).permute(0, 2, 3, 1)
    ld = (C + 7) // 8 * 8
    xi = torch.zeros(B, H, W, ld, device=DEV)
    xi[..., :C] = x.permute(0, 2, 3, 1)
    wt = torch.zeros(25, ld, device=DEV)
    wt[:, :C] = w.reshape(C, 25).t()
    t = Split(torch.full((B, H, W, ld), 7.0, dtype=torch.float16, device=DEV), torch.full((B, H, W, ld), 7.0, dtype=torch.float16, device=DEV))
    call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": xi}, out=t.hi, out_lo=t.lo, ldi=ld, ldo=ld, weight=wt, ldw=ld, bias=b,
         batch=B, h=H, w=W, c=C, dtype=F32)
    assert rel_err(t.join()[..., :C], ref) < 2e-6
