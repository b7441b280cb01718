"""Tensor-core (wgmma) / TMA back-end of romab200_gemm against torch matmul on the same 16-bit-rounded operands."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from roma_b200 import cabi  # noqa: E402
from roma_b200.cabi import call  # noqa: E402
from roma_b200.packing import at  # noqa: E402

DEV = "cuda"
CODE = cabi.DTYPE_CODE


def rnd(*shape, seed=0, scale=1.0, dtype=torch.float16):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def gemm(A, B, C, M, N, K, lda, ldb, ldc, dt, dtc, **kw):
    args = dict(A=A, B=B, C=C, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, dtype_ab=CODE[dt], dtype_c=CODE[dtc],
                batch0=1, batch1=1, ntaps=1, alpha=1.0, backend=cabi.BACKEND_TCGEN05)
    args.update(kw)
    call("romab200_gemm", "rb_gemm_args", **args)


def close(a, b, tol):
    err = (a.float().cpu() - b.float().cpu()).abs().max().item()
    assert err <= tol, f"max abs err {err} > {tol}"


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (300, 200, 136), (1000, 24, 24), (257, 4097, 1024), (130, 64, 592), (3200, 1377, 1384), (500, 9, 64),
                                   (20000, 144, 144), (19000, 569, 569), (19000, 1137, 1137), (19000, 130, 72), (19000, 192, 200)])
def test_tc_plain_f32_out(dt, M, N, K):
    lda = (K + 7) // 8 * 8
    A, B = rnd(M, lda, seed=1, dtype=dt), rnd(N, lda, seed=2, dtype=dt)
    ldc = (N + 3) // 4 * 4
    C = torch.full((M, ldc), 3.0, device=DEV)
    gemm(A, B, C, M, N, K, lda, lda, ldc, dt, torch.float32)
    ref = A[:, :K].double() @ B[:, :K].double().t()
    close(C[:, :N], ref, 2e-3 * math.sqrt(K) / 8 + 1e-3)
    if ldc > N:       # pad columns: untouched beyond the 16-byte granule of the row tail (TMA clipping granularity), zeros or untouched inside it
        gran = (N + 3) // 4 * 4
        assert (C[:, gran:] == 3.0).all() and ((C[:, N:gran] == 3.0) | (C[:, N:gran] == 0.0)).all()


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_tc_epilogues_16bit_out(dt):
    M, N, K = 391, 264, 320
    A, B = rnd(M, K, seed=1, dtype=dt), rnd(N, K, seed=2, dtype=dt, scale=0.1)
    bias = rnd(N, seed=3, dtype=torch.float32)
    gamma = rnd(N, seed=4, dtype=torch.float32)
    X = rnd(M, N, seed=5, dtype=torch.float32)
    base = A.float() @ B.float().t() + bias
    C = torch.zeros(M, N, dtype=dt, device=DEV)
    gemm(A, B, C, M, N, K, K, K, N, dt, dt, bias=bias, act=cabi.ACT_GELU)
    close(C, F.gelu(base), 3e-2 if dt == torch.bfloat16 else 4e-3)
    gemm(A, B, C, M, N, K, K, K, N, dt, dt, bias=bias, act=cabi.ACT_RELU)
    close(C, F.relu(base), 6e-2 if dt == torch.bfloat16 else 8e-3)
    ref = X + base * gamma
    gemm(A, B, X, M, N, K, K, K, N, dt, torch.float32, bias=bias, col_scale=gamma, R=X, ldr=N, dtype_r=cabi.RB_F32)
    close(X, ref, 2e-3)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("d,N", [(64, 203), (128, 160)])
def test_tc_attention_shapes_qkv_views(dt, d, N):
    Bn, H = 2, 3
    dim = H * d
    qkv = rnd(Bn, N, 3 * dim, seed=1, dtype=dt, scale=0.5)
    npad = (N + 7) // 8 * 8
    S = torch.zeros(Bn, H, N, npad, dtype=dt, device=DEV)
    gemm(qkv, at(qkv, dim), S, N, N, d, 3 * dim, 3 * dim, npad, dt, dt, batch0=Bn, batch1=H,
         alpha=1.0 / math.sqrt(d), sa0=N * 3 * dim, sa1=d, sb0=N * 3 * dim, sb1=d, sc0=H * N * npad, sc1=N * npad)
    q, k, v = qkv.float().reshape(Bn, N, 3, H, d).unbind(2)
    ref = torch.einsum("bnhd,bmhd->bhnm", q, k) / math.sqrt(d)
    close(S[..., :N], ref, 5e-2 if dt == torch.bfloat16 else 6e-3)
    call("romab200_softmax_rows", "rb_softmax_args", s=S, rows=Bn * H * N, cols=N, lds=npad, dtype=CODE[dt], scale=1.0)
    P = S[..., :N].float()
    O = torch.zeros(Bn, N, dim, dtype=dt, device=DEV)
    gemm(S, at(qkv, 2 * dim), O, N, d, N, npad, 3 * dim, dim, dt, dt, trans_b=1, batch0=Bn, batch1=H,
         sa0=H * N * npad, sa1=N * npad, sb0=N * 3 * dim, sb1=d, sc0=N * dim, sc1=d)
    ref_o = torch.einsum("bhnm,bmhd->bnhd", P, v).reshape(Bn, N, dim)
    close(O, ref_o, 2e-2 if dt == torch.bfloat16 else 3e-3)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("cin,cout,H,W", [(64, 64, 20, 36), (128, 256, 9, 13)])
def test_tc_conv3x3_taps(dt, cin, cout, H, W):
    E = 2
    x = rnd(E, cin, H, W, seed=1, dtype=dt)
    w = rnd(cout, cin, 3, 3, seed=2, scale=0.1, dtype=dt)
    b = rnd(cout, seed=3, dtype=torch.float32)
    ref = F.relu(F.conv2d(x.float(), w.float(), b, padding=1)).permute(0, 2, 3, 1)
    xp = torch.zeros(E, H + 2, W + 2, cin, dtype=dt, device=DEV)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    wm = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    out = torch.full((E, H + 2, W + 2, cout), -5.0, dtype=dt, device=DEV)
    rows = E * (H + 2) * (W + 2)
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    gemm(xp, wm, out, rows, cout, 9 * cin, cin, 9 * cin, cout, dt, dt, ntaps=9, tap_rows=taps, a_rows=rows, bias=b,
         act=cabi.ACT_RELU, rowmap=cabi.ROWMAP_PAD_KEEP, pad_h=H + 2, pad_w=W + 2)
    close(out[:, 1:-1, 1:-1], ref, 8e-2 if dt == torch.bfloat16 else 1e-2)
    # border rows of a padded map: left alone (direct stores) or rewritten with the zeros they hold on the path (TMA-store epilogue)
    border = torch.cat((out[:, 0].flatten(), out[:, -1].flatten(), out[:, :, 0].flatten(), out[:, :, -1].flatten()))
    assert ((border == -5.0) | (border == 0.0)).all()


def test_tc_coskernel_split_f16x3_is_fp32_class():
    """All-pairs CosKernel on the f16 tensor pipe with hi/lo operand splitting: error vs float64 must be at
    the fp32 level (SURVEY Appendix A: single-pass fp16/TF32 gives 3e-4 on the GP output, bf16 2e-3)."""
    n, c = 1600, 512
    g = torch.Generator().manual_seed(0)
    base = torch.randn(8, c, generator=g)
    x = (torch.randn(n, 8, generator=g) @ base + 0.5 * torch.randn(n, c, generator=g)).to(DEV)
    y = (torch.randn(n, 8, generator=g) @ base + 0.5 * torch.randn(n, c, generator=g)).to(DEV)
    nx, ny = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    call("romab200_row_norms", "rb_rownorm_args", x=x, out=nx, rows=n, cols=c, ldx=c, dtype=cabi.RB_F32)
    call("romab200_row_norms", "rb_rownorm_args", x=y, out=ny, rows=n, cols=c, ldx=c, dtype=cabi.RB_F32)
    xa = torch.zeros(n, 3 * c, dtype=torch.float16, device=DEV)
    yb = torch.zeros(n, 3 * c, dtype=torch.float16, device=DEV)
    call("romab200_split_f16x3", "rb_split_args", x=x, dst=xa, rows=n, cols=c, ldx=c, ldd=3 * c, row_norm=nx, layout_b=0)
    call("romab200_split_f16x3", "rb_split_args", x=y, dst=yb, rows=n, cols=c, ldx=c, ldd=3 * c, row_norm=ny, layout_b=1)
    K = torch.zeros(n, n, device=DEV)
    gemm(xa, yb, K, n, n, 3 * c, 3 * c, 3 * c, n, torch.float16, torch.float32, epi=cabi.EPI_COSKERNEL, norm_a=nx, norm_b=ny,
         eps=1e-6, inv_t=5.0, diag_add=0.0, cos_normalized=1)
    xd, yd = x.double().cpu(), y.double().cpu()
    cos = (xd @ yd.t()) / (xd.norm(dim=-1)[:, None] * yd.norm(dim=-1)[None] + 1e-6)
    ref = ((cos - 1) / 0.2).exp()
    err = (K.double().cpu() - ref).abs().max().item()
    print("coskernel split-f16x3 max abs err vs fp64:", err)
    assert err < 3e-5      # fp32 CUDA-core path: ~2e-6; single-pass fp16/TF32 operands: ~5e-4


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_refiner_block_small_fused_vs_unfused_host_tensors(dt):
    """Fused thin-map block (DW5x5+ReLU+PW, C=24) against conv2d on the same 16-bit-rounded tensors."""
    B, C, H, W = 2, 24, 37, 50
    x = rnd(B, C, H, W, seed=1, dtype=dt)
    dw, db = rnd(C, 1, 5, 5, seed=2, scale=0.3, dtype=torch.float32), rnd(C, seed=3, dtype=torch.float32)
    pw, pb = rnd(C, C, seed=4, scale=0.3, dtype=dt), rnd(C, seed=5, dtype=torch.float32)
    mid = F.relu(F.conv2d(x.float(), dw, db, padding=2, groups=C)).to(dt).float()
    ref = (torch.einsum("bchw,oc->bohw", mid, pw.float()) + pb[None, :, None, None]).permute(0, 2, 3, 1)
    xi = x.permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(B, H, W, C, dtype=dt, device=DEV)
    dwt = dw.reshape(C, 25).t().contiguous()
    pw_host, pb_host = pw.float().cpu().contiguous(), pb.cpu().contiguous()       # host arrays: they travel as kernel parameters
    call("romab200_refiner_block_small", "rb_refiner_block_small_args", **{"in": xi}, out=out, ld=C, dw_weight=dwt, ldw=C, dw_bias=db,
         pw_weight_host=pw_host, pw_bias_host=pb_host, batch=B, h=H, w=W, c=C, dtype=CODE[dt])
    close(out, ref, 6e-2 if dt == torch.bfloat16 else 8e-3)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("H,d,N,Bn", [(16, 64, 1601, 2), (8, 128, 1600, 2), (3, 64, 77, 1), (2, 128, 300, 3), (2, 64, 128, 1)])
def test_flash_attn(dt, H, d, N, Bn):
    dim = H * d
    qkv = rnd(Bn, N, 3 * dim, seed=1, dtype=dt, scale=1.0)
    out = torch.full((Bn, N, dim), 9.0, dtype=dt, device=DEV)
    call("romab200_flash_attn", "rb_flash_attn_args", qkv=qkv, out=out, ld_qkv=3 * dim, ld_out=dim, batch=Bn, n_tokens=N, heads=H,
         head_dim=d, dtype=CODE[dt])
    torch.cuda.synchronize()
    q, k, v = qkv.float().reshape(Bn, N, 3, H, d).unbind(2)
    ref = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2).reshape(Bn, N, dim)
    close(out, ref, 2.5e-2 if dt == torch.bfloat16 else 4e-3)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,W", [(2, 37, 50), (1, 8, 16), (2, 84, 84)])
def test_refiner_block_c144_fused(dt, B, H, W):
    """Fused stride-2 block (DW5x5+ReLU on CUDA cores -> wgmma PW 144x144) against conv2d on the same rounded tensors."""
    C = 144
    x = rnd(B, C, H, W, seed=1, dtype=dt)
    dw, db = rnd(C, 1, 5, 5, seed=2, scale=0.3, dtype=torch.float32), rnd(C, seed=3, dtype=torch.float32)
    pw, pb = rnd(C, C, seed=4, scale=0.1, dtype=dt), rnd(C, seed=5, dtype=torch.float32)
    mid = F.relu(F.conv2d(x.float(), dw, db, padding=2, groups=C)).to(dt).float()
    ref = (torch.einsum("bchw,oc->bohw", mid, pw.float()) + pb[None, :, None, None]).permute(0, 2, 3, 1)
    xi = x.permute(0, 2, 3, 1).contiguous()
    out = torch.full((B, H, W, C), 7.0, dtype=dt, device=DEV)
    dwt = dw.reshape(C, 25).t().contiguous()
    call("romab200_refiner_block_c144", "rb_refiner_block_c144_args", **{"in": xi}, out=out, ld=C, dw_weight=dwt, ldw=C, dw_bias=db,
         pw_weight=pw.contiguous(), ld_pw=C, pw_bias=pb, batch=B, h=H, w=W, c=C, dtype=CODE[dt])
    torch.cuda.synchronize()
    close(out, ref, 1.5e-1 if dt == torch.bfloat16 else 2e-2)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,C,H,W", [(2, 150, 19, 37), (1, 64, 8, 16), (2, 569, 54, 54), (1, 70, 5, 3)])
def test_dwconv_16bit_tma(dt, B, C, H, W):
    """TMA-fed depthwise 5x5 + ReLU on 16-bit maps (ragged tiles, channel tail, zero-filled borders) against conv2d."""
    x = rnd(B, C, H, W, seed=1, dtype=dt)
    w, b = rnd(C, 1, 5, 5, seed=2, scale=0.3, dtype=torch.float32), rnd(C, seed=3, dtype=torch.float32)
    ref = F.relu(F.conv2d(x.float(), w, b, padding=2, groups=C)).permute(0, 2, 3, 1)
    ld = (C + 7) // 8 * 8
    xi = torch.zeros(B, H, W, ld, dtype=dt, device=DEV)
    xi[..., :C] = x.permute(0, 2, 3, 1)
    wt = torch.zeros(25, ld, device=DEV)
    wt[:, :C] = w.reshape(C, 25).t()
    out = torch.full((B, H, W, ld), 7.0, dtype=dt, device=DEV)
    call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": xi}, out=out, ldi=ld, ldo=ld, weight=wt, ldw=ld, bias=b, batch=B, h=H, w=W, c=C,
         dtype=CODE[dt])
    torch.cuda.synchronize()
    close(out[..., :C], ref, 6e-2 if dt == torch.bfloat16 else 8e-3)


@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,C,H,W", [(2, 64, 14, 22), (1, 128, 6, 4), (2, 72, 8, 8)])
def test_maxpool_16bit_vector(dt, B, C, H, W):
    """2x2 max-pool between zero-padded channels-last maps, 16-byte vector kernel: exact (a max is a selection)."""
    x = rnd(B, H, W, C, seed=1, dtype=dt)
    xin = torch.zeros(B, H + 2, W + 2, C, dtype=dt, device=DEV)
    xin[:, 1:-1, 1:-1] = x
    out = torch.zeros(B, H // 2 + 2, W // 2 + 2, C, dtype=dt, device=DEV)
    call("romab200_maxpool2x2_padded", "rb_maxpool_args", **{"in": xin}, out=out, batch=B, height=H, width=W, channels=C, dtype=CODE[dt])
    ref = F.max_pool2d(x.permute(0, 3, 1, 2).float(), 2).permute(0, 2, 3, 1)
    assert torch.equal(out[:, 1:-1, 1:-1].float().cpu(), ref.cpu())
    assert out[:, 0].abs().max() == 0 and out[:, :, 0].abs().max() == 0 and out[:, -1].abs().max() == 0 and out[:, :, -1].abs().max() == 0
