"""Tile order of the tensor-core GEMM (gemm_tc.cu): launches whose A operand is too big to stay in L2 walk their tiles in bands of
M-tiles instead of m-fastest.  Each launch here is chosen to take the banded order and is compared bit for bit with the same
product computed as column slices no wider than 128: a slice has one N-tile, so its order is m-fastest whatever the rule, and
every output element has the same k order in both.  Outputs start as a sentinel, so a tile the scheduler skips shows up."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from roma_b200 import cabi, packing  # noqa: E402
from roma_b200.cabi import call  # noqa: E402

DEV = "cuda"
SENT = -7.0


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def split(x):
    """fp32 -> (hi, lo) fp16 planes, x ~ hi + lo * 2^-11 (the RB_F16S format)."""
    hi = x.half()
    return hi, ((x - hi.float()) * 2048.0).half()


def gemm(**kw):
    args = dict(batch0=1, batch1=1, ntaps=1, alpha=1.0, backend=cabi.BACKEND_TCGEN05, dtype_ab=cabi.RB_F16S)
    args.update(kw)
    call("romab200_gemm", "rb_gemm_args", **args)


def at(t, elems):
    """Flat view of tensor t from element `elems` on (None stays None)."""
    return None if t is None else packing.at(t, elems)


def full_and_sliced(A, B, outs, N, ldb, ldc, bias=None, col_scale=None, residual=False, **kw):
    """Runs the launch once over all N columns and once as slices of at most 128 columns, each on its own copy of the output
    planes `outs` (C, or C and C_lo).  residual: the output is also the residual R (updated in place)."""
    (Ah, Al), (Bh, Bl) = A, B
    full = [o.clone() for o in outs]
    sliced = [o.clone() for o in outs]

    def run(C, n0, w):
        extra = dict(R=at(C[0], n0), ldr=ldc, dtype_r=kw["dtype_c"]) if residual else {}
        gemm(A=Ah, A_lo=Al, B=at(Bh, n0 * ldb), B_lo=at(Bl, n0 * ldb), C=at(C[0], n0), C_lo=at(C[1], n0) if len(C) > 1 else None,
             N=w, ldb=ldb, ldc=ldc, bias=at(bias, n0), col_scale=at(col_scale, n0), **extra, **kw)

    run(full, 0, N)
    for n0 in range(0, N, 128):
        run(sliced, n0, min(128, N - n0))
    torch.cuda.synchronize()
    return full, sliced


def assert_banded(M, k_extent, N, K):
    """The launch is on the banded side of the rule on this device: A (both planes) is more than half the L2, B at most half."""
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    assert 2 * M * k_extent * 4 > l2 and 2 * N * K * 4 <= l2, (M, k_extent, N, K, l2)


@pytest.mark.parametrize("M", [40000, 38017])          # 313 / 298 M-tiles: the last band is short for every band height here
@pytest.mark.parametrize("C,max_ctas", [(569, 0), (1137, 0), (569, 40)])
def test_refiner_pointwise_bands_vs_slice_views(M, C, max_ctas):
    """The refiner's pointwise 1x1 convolution: split operands, fp32 output + bias, N = K = C (4 or 9 N-tiles); max_ctas caps the
    grid and with it the band height."""
    assert_banded(M, C, C, C)
    ld = (C + 7) // 8 * 8
    A, B = rnd(M, ld, seed=1), rnd(C, ld, seed=2, scale=0.05)
    A[:, C:] = 0
    B[:, C:] = 0
    bias = rnd(C, seed=3)
    out = torch.full((M, ld), SENT, device=DEV)
    (full,), (sliced,) = full_and_sliced(split(A), split(B), [out], C, ld, ld, bias=bias, M=M, K=C, lda=ld, dtype_c=cabi.RB_F32,
                                         max_ctas=max_ctas)
    assert not (full[:, :C] == SENT).any(), "every tile is computed"
    assert torch.equal(full, sliced)


def test_conv3x3_taps_pad_keep_bands_vs_slice_views():
    """A 9-tap 3x3 convolution on a zero-padded channels-last map (the VGG pattern): split output, bias + ReLU, PAD_KEEP rows.
    The tap shifts of +-(W + 3) rows reach into neighbouring M-tiles of the same band."""
    E, H, W, cin, cout = 2, 128, 128, 256, 512
    rows = E * (H + 2) * (W + 2)
    assert_banded(rows, cin, cout, 9 * cin)
    x = torch.zeros(E, H + 2, W + 2, cin, device=DEV)
    x[:, 1:-1, 1:-1] = rnd(E, H, W, cin, seed=1)
    w = rnd(cout, 9 * cin, seed=2, scale=0.05)
    bias = rnd(cout, seed=3)
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    outs = [torch.full((rows, cout), SENT, dtype=torch.float16, device=DEV) for _ in range(2)]
    full, sliced = full_and_sliced(split(x.view(rows, cin)), split(w), outs, cout, 9 * cin, cout, bias=bias, M=rows, K=9 * cin,
                                   lda=cin, dtype_c=cabi.RB_F16S, ntaps=9, tap_rows=taps, a_rows=rows, act=cabi.ACT_RELU,
                                   rowmap=cabi.ROWMAP_PAD_KEEP, pad_h=H + 2, pad_w=W + 2)
    inner = full[0].view(E, H + 2, W + 2, cout)[:, 1:-1, 1:-1]
    assert not (inner == SENT).any(), "every tile is computed"
    assert (full[0].view(E, H + 2, W + 2, cout)[:, 0] == SENT).all(), "PAD_KEEP border rows are not stored"
    assert torch.equal(full[0], sliced[0]) and torch.equal(full[1], sliced[1])


def test_residual_in_place_col_scale_bands_vs_slice_views():
    """X += (A B^T + bias) * gamma with R == C (the ViT fc2 pattern: M = 3202 tokens, K = 4096, N = 1024)."""
    M, N, K = 3202, 1024, 4096
    assert_banded(M, K, N, K)
    A, B = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.02)
    bias, gamma = rnd(N, seed=3), rnd(N, seed=4)
    X = rnd(M, N, seed=5)
    (full,), (sliced,) = full_and_sliced(split(A), split(B), [X], N, K, N, bias=bias, col_scale=gamma, residual=True, M=M, K=K,
                                         lda=K, dtype_c=cabi.RB_F32)
    assert not torch.equal(full, X), "the residual is updated"
    assert torch.equal(full, sliced)


def test_batched_bands_vs_slice_views():
    """Two independent products in one launch (batch0 = 2): bands run inside each z, z outermost."""
    Z, M, N, K = 2, 20000, 569, 576
    assert_banded(M, K, N, K)
    A, B = rnd(Z * M, K, seed=1), rnd(Z * N, K, seed=2, scale=0.05)
    bias = rnd(N, seed=3)
    out = torch.full((Z * M, K), SENT, device=DEV)
    (full,), (sliced,) = full_and_sliced(split(A), split(B), [out], N, K, K, bias=bias, M=M, K=K, lda=K, dtype_c=cabi.RB_F32,
                                         batch0=Z, sa0=M * K, sb0=N * K, sc0=M * K)
    assert not (full[:, :N] == SENT).any(), "every tile of every z is computed"
    assert torch.equal(full, sliced)
