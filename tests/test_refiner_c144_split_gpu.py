"""Parity-mode fused refiner block at C = 144 (romab200_refiner_block_c144_split) against the two launches it replaces:
romab200_dwconv5x5_relu (fp32 map -> RB_F16S pair) then the split-fp16 romab200_gemm (+ bias, fp32 out).  The results must be
equal bit for bit (torch.equal: +0 and -0 compare equal, NaN never does); outputs are NaN-filled first, so an element a kernel
fails to write shows up."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from roma_b200 import cabi  # noqa: E402
from roma_b200.cabi import call  # noqa: E402

C = 144


def rnd(*shape, seed, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).cuda()


def make_block(ld, seed):
    """Depthwise taps [25][ld] + bias, pointwise RB_F16S planes [144][ld] (pad columns zero, as packed) + bias."""
    dw = torch.zeros(25, ld, device="cuda")
    dw[:, :C] = rnd(25, C, seed=seed, scale=0.2)
    pw = rnd(C, C, seed=seed + 1, scale=C ** -0.5)
    hi = torch.zeros(C, ld, dtype=torch.float16, device="cuda")
    lo = torch.zeros(C, ld, dtype=torch.float16, device="cuda")
    hi[:, :C] = pw.half()
    lo[:, :C] = ((pw - hi[:, :C].float()) * 2048.0).half()
    return dict(dw=dw, db=rnd(C, seed=seed + 2, scale=0.1), hi=hi, lo=lo, pb=rnd(C, seed=seed + 3, scale=0.1))


def unfused(x, y, blk, B, H, W, ld):
    """y = the two-launch block of the parity mode on x."""
    rows = B * H * W
    ts_hi = torch.full((rows, ld), float("nan"), dtype=torch.float16, device="cuda")
    ts_lo = torch.full((rows, ld), float("nan"), dtype=torch.float16, device="cuda")
    call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": x}, out=ts_hi, out_lo=ts_lo, ldi=ld, ldo=ld, weight=blk["dw"], ldw=ld,
         bias=blk["db"], batch=B, h=H, w=W, c=C, dtype=cabi.RB_F32)
    call("romab200_gemm", "rb_gemm_args", A=ts_hi, A_lo=ts_lo, B=blk["hi"], B_lo=blk["lo"], C=y, M=rows, N=C, K=C, lda=ld, ldb=ld, ldc=ld,
         batch0=1, batch1=1, ntaps=1, alpha=1.0, bias=blk["pb"], dtype_ab=cabi.RB_F16S, dtype_c=cabi.RB_F32)


def fused(x, y, blk, B, H, W, ld):
    call("romab200_refiner_block_c144_split", "rb_refiner_block_c144_split_args", **{"in": x}, out=y, ld=ld, dw_weight=blk["dw"], ldw=ld,
         dw_bias=blk["db"], pw_weight=blk["hi"], pw_weight_lo=blk["lo"], ld_pw=ld, pw_bias=blk["pb"], batch=B, h=H, w=W, c=C)


def input_map(B, H, W, ld, seed):
    """fp32 map [B*H*W, ld]; the pad columns hold NaN (neither path may read them)."""
    x = torch.full((B * H * W, ld), float("nan"), device="cuda")
    x[:, :C] = rnd(B * H * W, C, seed=seed)
    return x


def assert_same(a, b, ld):
    assert torch.equal(a[:, :C], b[:, :C]), f"{(a[:, :C] != b[:, :C]).sum().item()} elements differ"
    if ld > C:
        assert torch.isnan(a[:, C:]).all() and torch.isnan(b[:, C:]).all(), "pad columns were written"


@pytest.mark.parametrize("B,H,W,ld", [(2, 432, 432, 144), (2, 280, 280, 144), (3, 13, 37, 144), (2, 40, 50, 152)])
def test_block_bit_identical(B, H, W, ld):
    x = input_map(B, H, W, ld, seed=1)
    blk = make_block(ld, seed=10)
    ref = torch.full_like(x, float("nan"))
    out = torch.full_like(x, float("nan"))
    unfused(x, ref, blk, B, H, W, ld)
    fused(x, out, blk, B, H, W, ld)
    torch.cuda.synchronize()
    assert torch.isfinite(ref[:, :C]).all()
    assert_same(out, ref, ld)


def test_chain_of_nine_blocks_bit_identical():
    """The 9-block chain as the engine runs it: fused blocks ping-pong two buffers, the un-fused ones update the map in place."""
    B, H, W, ld = 2, 280, 280, C
    blocks = [make_block(ld, seed=100 + 10 * i) for i in range(9)]
    d_ref = input_map(B, H, W, ld, seed=2)
    d, t = d_ref.clone(), torch.full_like(d_ref, float("nan"))
    for blk in blocks:
        unfused(d_ref, d_ref, blk, B, H, W, ld)
        fused(d, t, blk, B, H, W, ld)
        d, t = t, d
    torch.cuda.synchronize()
    assert torch.isfinite(d_ref).all()
    assert_same(d, d_ref, ld)


def test_rejects_bad_arguments():
    B, H, W, ld = 1, 8, 16, C
    x = input_map(B, H, W, ld, seed=3)
    blk = make_block(ld, seed=20)
    with pytest.raises(RuntimeError, match="differ"):
        fused(x, x, blk, B, H, W, ld)
    y = torch.empty_like(x)
    with pytest.raises(RuntimeError, match="C must be 144"):
        call("romab200_refiner_block_c144_split", "rb_refiner_block_c144_split_args", **{"in": x}, out=y, ld=ld, dw_weight=blk["dw"],
             ldw=ld, dw_bias=blk["db"], pw_weight=blk["hi"], pw_weight_lo=blk["lo"], ld_pw=ld, pw_bias=blk["pb"], batch=B, h=H, w=W, c=128)
    x2 = torch.zeros(B * H * W, 148, device="cuda")
    with pytest.raises(RuntimeError, match="activation layout"):
        fused(x2, torch.empty_like(x2), blk, B, H, W, 148)
