"""Epilogue of the tensor-core GEMM (gemm_tc.cu): every output dtype x row map at ragged shapes against float64, sentinel-filled
outputs (pad columns past the 16-byte granule and PAD_KEEP border rows stay untouched), in-place residuals, and the 144-wide split
tiles against the same problem computed as column slices no wider than 128."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from roma_b200 import cabi  # noqa: E402
from roma_b200.cabi import call  # noqa: E402
from roma_b200.packing import at  # noqa: E402

DEV = "cuda"
SENT = -7.0
PAD_H, PAD_W, IMGS = 50, 61, 4                     # 12200 rows: enough tiles for the 256-wide fp16 tiles
SEG_IN, SEG_OUT, SEG_OFF = 1000, 1013, 5


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def split(x):
    """fp32 -> (hi, lo) fp16 planes, x ~ hi + lo * 2^-11 (the RB_F16S format)."""
    hi = x.half()
    return hi, ((x - hi.float()) * 2048.0).half()


def joined(hi, lo):
    return hi.double() + lo.double() / 2048.0


def gemm(**kw):
    args = dict(batch0=1, batch1=1, ntaps=1, alpha=1.0, backend=cabi.BACKEND_TCGEN05)
    args.update(kw)
    call("romab200_gemm", "rb_gemm_args", **args)


def stored_rows(rowmap, M):
    """(logical rows that are stored, their stored rows, number of rows of the output)."""
    m = torch.arange(M)
    if rowmap == cabi.ROWMAP_NONE:
        return m, m, M
    if rowmap == cabi.ROWMAP_SEGMENT:
        o = m // SEG_IN * SEG_OUT + m % SEG_IN + SEG_OFF
        return m, o, int(o.max()) + 1
    rem = m % (PAD_H * PAD_W)
    yp, xp = rem // PAD_W, rem % PAD_W
    inner = (yp > 0) & (xp > 0) & (yp < PAD_H - 1) & (xp < PAD_W - 1)
    if rowmap == cabi.ROWMAP_PAD_KEEP:
        return m[inner], m[inner], M
    o = m // (PAD_H * PAD_W) * (PAD_H - 2) * (PAD_W - 2) + (yp - 1) * (PAD_W - 2) + (xp - 1)
    return m[inner], o[inner], IMGS * (PAD_H - 2) * (PAD_W - 2)


OUT = {"f32": cabi.RB_F32, "f16": cabi.RB_F16, "bf16": cabi.RB_BF16, "f16s": cabi.RB_F16S}
TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16, "f16s": torch.float16}
REL = {"f32": 2e-6, "f16": 2.0 ** -11, "bf16": 2.0 ** -8, "f16s": 2e-6}     # output rounding on top of fp32 accumulation
MAPS = {"none": cabi.ROWMAP_NONE, "pad_keep": cabi.ROWMAP_PAD_KEEP, "pad_to_compact": cabi.ROWMAP_PAD_TO_COMPACT, "segment": cabi.ROWMAP_SEGMENT}


@pytest.mark.parametrize("operands", ["f16", "f16s"])
@pytest.mark.parametrize("out", list(OUT))
@pytest.mark.parametrize("rowmap", list(MAPS))
@pytest.mark.parametrize("pitch", ["aligned", "odd"])
def test_epilogue_dtype_rowmap(operands, out, rowmap, pitch):
    """bias + GELU, then col_scale + a bf16 residual, at N = 203 (not a multiple of 8, 32 or any tile width) on every row map; the
    output starts as a sentinel, which must survive outside the stored rows and past the zeroed pad granule."""
    rm = MAPS[rowmap]
    M = IMGS * PAD_H * PAD_W
    N, K = 203, 200
    A32, B32 = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.1)
    if operands == "f16":
        Ah, Bh = A32.half(), B32.half()
        Ad, Bd = Ah.double(), Bh.double()
        ops = dict(A=Ah, B=Bh, dtype_ab=cabi.RB_F16)
    else:
        (Ah, Al), (Bh, Bl) = split(A32), split(B32)
        Ad, Bd = joined(Ah, Al), joined(Bh, Bl)
        ops = dict(A=Ah, A_lo=Al, B=Bh, B_lo=Bl, dtype_ab=cabi.RB_F16S)
    bias, gamma = rnd(N, seed=3), rnd(N, seed=4)
    ms, orows, rows_out = stored_rows(rm, M)
    ldc = 208 if pitch == "aligned" else 211
    rmk = dict(rowmap=rm, pad_h=PAD_H, pad_w=PAD_W, seg_in=SEG_IN, seg_out=SEG_OUT, seg_off=SEG_OFF)
    es = 4 if out == "f32" else 2
    gran = 16 // es

    def new_out():
        C = torch.full((rows_out, ldc), SENT, dtype=TORCH[out], device=DEV)
        C_lo = torch.full((rows_out, ldc), SENT, dtype=torch.float16, device=DEV) if out == "f16s" else None
        return C, C_lo

    def value(C, C_lo):
        return joined(C, C_lo) if out == "f16s" else C.double()

    def check(C, C_lo, ref, zero_pad):
        got = value(C, C_lo).cpu()
        exp = torch.full((rows_out, ldc), float("nan"), dtype=torch.float64)
        exp[orows, :N] = ref.cpu()[ms]
        sel = ~torch.isnan(exp)
        err = (got[sel] - exp[sel]).abs()
        tol = REL[out] * exp[sel].abs() + 2e-5
        assert (err <= tol).all(), f"max err {err.max().item()} (out {out}, rowmap {rowmap}, pitch {pitch})"
        untouched = torch.ones(rows_out, ldc, dtype=torch.bool)
        untouched[orows, :N] = False
        nz = (N + gran - 1) // gran * gran if zero_pad else N
        if zero_pad:
            assert (got[orows][:, N:nz] == 0).all(), "pad columns inside the row's last 16-byte granule are zeroed"
            untouched[orows, N:nz] = False
        for plane in (C, C_lo) if C_lo is not None else (C,):
            p = plane.float().cpu()
            assert (p[untouched] == SENT).all(), "rows and columns that are not stored keep their contents"

    acc = Ad @ Bd.t()
    C, C_lo = new_out()
    gemm(**ops, C=C, C_lo=C_lo, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, dtype_c=OUT[out], bias=bias, act=cabi.ACT_GELU, **rmk)
    zero_pad = pitch == "aligned" and rm in (cabi.ROWMAP_NONE, cabi.ROWMAP_PAD_KEEP)
    check(C, C_lo, torch.nn.functional.gelu(acc + bias.double()), zero_pad)

    R = torch.zeros(rows_out, ldc, dtype=torch.bfloat16, device=DEV)
    R[:, :N] = rnd(rows_out, N, seed=5).bfloat16()
    Rm = torch.zeros(M, N, dtype=torch.float64)
    Rm[ms] = R.double().cpu()[orows, :N]
    C, C_lo = new_out()
    gemm(**ops, C=C, C_lo=C_lo, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, dtype_c=OUT[out], bias=bias, col_scale=gamma, R=R, ldr=ldc,
         dtype_r=cabi.RB_BF16, **rmk)
    check(C, C_lo, (acc + bias.double()) * gamma.double() + Rm.to(DEV), zero_pad=False)


@pytest.mark.parametrize("out", ["f32", "bf16"])
def test_epilogue_residual_in_place_split(out):
    """C = C + (A B^T + bias) * gamma with R == C (the ViT proj / fc2 pattern) on split operands at a ragged N."""
    M, N, K = 3001, 1037, 304
    (Ah, Al), (Bh, Bl) = split(rnd(M, K, seed=1)), split(rnd(N, K, seed=2, scale=0.1))
    bias, gamma = rnd(N, seed=3), rnd(N, seed=4)
    ldc = 1040
    X = rnd(M, ldc, seed=5).to(TORCH[out])
    x0 = X.double()
    gemm(A=Ah, A_lo=Al, B=Bh, B_lo=Bl, dtype_ab=cabi.RB_F16S, C=X, M=M, N=N, K=K, lda=K, ldb=K, ldc=ldc, dtype_c=OUT[out],
         bias=bias, col_scale=gamma, R=X, ldr=ldc, dtype_r=OUT[out])
    ref = x0[:, :N] + (joined(Ah, Al) @ joined(Bh, Bl).t() + bias.double()) * gamma.double()
    err = (X[:, :N].double() - ref).abs()
    assert (err <= REL[out] * ref.abs() + 1e-4).all(), err.max().item()
    assert torch.equal(X[:, N:].double(), x0[:, N:]), "columns past N (the residual disables the pad-granule zeroing) are untouched"


@pytest.mark.parametrize("N", [144, 569])
def test_split_144_tiles_match_narrow_slice_views(N):
    """N = 144 and 569 run on 144-wide split tiles; the same problem as launches over column slices of at most 128 (128-, 64- and
    32-wide tiles) has the same k order per output, so the results are bit-equal."""
    M, K = 12000, N                                   # enough tiles that the width rule does not fall back to 128 for occupancy
    lda = (K + 7) // 8 * 8
    A = torch.zeros(M, lda, device=DEV)
    B = torch.zeros(N, lda, device=DEV)
    A[:, :K], B[:, :K] = rnd(M, K, seed=1), rnd(N, K, seed=2, scale=0.1)
    (Ah, Al), (Bh, Bl) = split(A), split(B)
    bias = rnd(N, seed=3)
    ldc = (N + 3) // 4 * 4
    full = torch.full((M, ldc), SENT, device=DEV)
    gemm(A=Ah, A_lo=Al, B=Bh, B_lo=Bl, dtype_ab=cabi.RB_F16S, C=full, M=M, N=N, K=K, lda=lda, ldb=lda, ldc=ldc, dtype_c=cabi.RB_F32,
         bias=bias, act=cabi.ACT_RELU)
    sliced = torch.full((M, ldc), SENT, device=DEV)
    for n0 in range(0, N, 128):
        w = min(128, N - n0)
        gemm(A=Ah, A_lo=Al, B=at(Bh, n0 * lda), B_lo=at(Bl, n0 * lda), dtype_ab=cabi.RB_F16S,
             C=at(sliced, n0), M=M, N=w, K=K, lda=lda, ldb=lda, ldc=ldc, dtype_c=cabi.RB_F32, bias=at(bias, n0),
             act=cabi.ACT_RELU)
    torch.cuda.synchronize()
    ref = torch.relu(joined(Ah, Al) @ joined(Bh, Bl).t() + bias.double())
    assert ((full[:, :N].double() - ref).abs() <= 2e-6 * ref.abs() + 1e-5).all()
    assert torch.equal(full[:, :N], sliced[:, :N])
