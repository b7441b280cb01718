"""Per-kernel parity tests of the C ABI (fp32 back-ends) against plain PyTorch fp32 / the CPU oracle.

Every test calls through `roma_b200.cabi.call`, i.e. through the `extern "C"` entry points.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from roma_b200 import cabi  # noqa: E402
from roma_b200.cabi import call  # noqa: E402
from roma_b200.packing import at  # noqa: E402

DEV = "cuda"
F32 = cabi.RB_F32


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(DEV)


def gemm(A, B, C, M, N, K, lda, ldb, ldc, **kw):
    args = dict(A=A, B=B, C=C, M=M, N=N, K=K, lda=lda, ldb=ldb, ldc=ldc, dtype_ab=F32, dtype_c=F32,
                batch0=1, batch1=1, ntaps=1, alpha=1.0)
    args.update(kw)
    call("romab200_gemm", "rb_gemm_args", **args)


def close(a, b, tol):
    err = (a.float().cpu() - b.float().cpu()).abs().max().item()
    assert err <= tol, f"max abs err {err} > {tol}"


# ----------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("M,N,K", [(300, 70, 52), (129, 24, 24), (1000, 9, 64), (257, 4097, 1024), (64, 200, 588), (500, 3, 36)])
def test_gemm_plain(M, N, K):
    A, B = rnd(M, K, seed=1), rnd(N, K, seed=2)
    C = torch.zeros(M, N, device=DEV)
    gemm(A, B, C, M, N, K, K, K, N)
    close(C, A.double() @ B.double().t(), 2e-4 * math.sqrt(K))


def test_gemm_pitched_bias_relu_gelu():
    M, N, K, lda, ldb, ldc = 200, 90, 100, 104, 112, 96
    A, B = rnd(M, lda, seed=1), rnd(N, ldb, seed=2)
    bias = rnd(N, seed=3)
    for act, fn in ((cabi.ACT_RELU, torch.relu), (cabi.ACT_GELU, F.gelu), (cabi.ACT_NONE, lambda x: x)):
        C = torch.full((M, ldc), 7.0, device=DEV)
        gemm(A, B, C, M, N, K, lda, ldb, ldc, bias=bias, act=act)
        ref = fn(A[:, :K] @ B[:, :K].t() + bias)
        close(C[:, :N], ref, 1e-4)
        assert (C[:, N:] == 7.0).all()


def test_gemm_layerscale_residual_inplace():
    M, N, K = 130, 128, 256
    A, B, bias, gamma = rnd(M, K, seed=1), rnd(N, K, seed=2), rnd(N, seed=3), rnd(N, seed=4)
    X = rnd(M, N, seed=5)
    ref = X + (A @ B.t() + bias) * gamma
    gemm(A, B, X, M, N, K, K, K, N, bias=bias, col_scale=gamma, R=X, ldr=N, dtype_r=F32)
    close(X, ref, 2e-4)


def test_gemm_trans_b_and_batched_heads_qkv_views():
    Bn, H, N, d = 2, 3, 70, 16
    dim = H * d
    qkv = rnd(Bn, N, 3 * dim, seed=1)
    npad = 72
    S = torch.zeros(Bn, H, N, npad, device=DEV)
    gemm(qkv, at(qkv, dim), S, N, N, d, 3 * dim, 3 * dim, npad, batch0=Bn, batch1=H,
         sa0=N * 3 * dim, sa1=d, sb0=N * 3 * dim, sb1=d, sc0=H * N * npad, sc1=N * npad)
    q, k, v = qkv.reshape(Bn, N, 3, H, d).unbind(2)
    ref = torch.einsum("bnhd,bmhd->bhnm", q, k)
    close(S[..., :N], ref, 1e-4)
    call("romab200_softmax_rows", "rb_softmax_args", s=S, rows=Bn * H * N, cols=N, lds=npad, dtype=F32, scale=0.25)
    close(S[..., :N], (ref * 0.25).softmax(-1), 1e-5)
    O = torch.zeros(Bn, N, dim, device=DEV)
    gemm(S, at(qkv, 2 * dim), O, N, d, N, npad, 3 * dim, dim, trans_b=1, batch0=Bn, batch1=H,
         sa0=H * N * npad, sa1=N * npad, sb0=N * 3 * dim, sb1=d, sc0=N * dim, sc1=d)
    ref_o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)).transpose(1, 2).reshape(Bn, N, dim)
    close(O, ref_o, 1e-4)


@pytest.mark.parametrize("cin,cout,H,W", [(16, 32, 9, 13), (64, 64, 20, 36)])
def test_gemm_conv3x3_taps(cin, cout, H, W):
    E = 2
    x = rnd(E, cin, H, W, seed=1)
    w = rnd(cout, cin, 3, 3, seed=2, scale=0.2)
    b = rnd(cout, seed=3)
    ref = F.relu(F.conv2d(x, w, b, padding=1)).permute(0, 2, 3, 1)
    xp = torch.zeros(E, H + 2, W + 2, cin, device=DEV)
    xp[:, 1:-1, 1:-1] = x.permute(0, 2, 3, 1)
    wm = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin).contiguous()
    out = torch.full((E, H + 2, W + 2, cout), -5.0, device=DEV)
    rows = E * (H + 2) * (W + 2)
    taps = [(ky - 1) * (W + 2) + (kx - 1) for ky in range(3) for kx in range(3)]
    gemm(xp, wm, out, rows, cout, 9 * cin, cin, 9 * cin, cout, ntaps=9, tap_rows=taps, a_rows=rows, bias=b,
         act=cabi.ACT_RELU, rowmap=cabi.ROWMAP_PAD_KEEP, pad_h=H + 2, pad_w=W + 2)
    close(out[:, 1:-1, 1:-1], ref, 2e-4)
    assert (out[:, 0] == -5.0).all() and (out[:, :, 0] == -5.0).all() and (out[:, -1] == -5.0).all() and (out[:, :, -1] == -5.0).all()
    # compact row map (used by proj on padded taps)
    w1 = rnd(24, cin, seed=4)
    comp = torch.zeros(E, H, W, 24, device=DEV)
    gemm(xp, w1, comp, rows, 24, cin, cin, cin, 24, rowmap=cabi.ROWMAP_PAD_TO_COMPACT, pad_h=H + 2, pad_w=W + 2)
    close(comp, x.permute(0, 2, 3, 1) @ w1.t(), 1e-4)


def test_gemm_segment_rowmap():
    M, N, K = 12, 8, 8
    A, B = rnd(M, K, seed=1), rnd(N, K, seed=2)
    out = torch.zeros(3 * 5, N, device=DEV)
    gemm(A, B, out, M, N, K, K, K, N, rowmap=cabi.ROWMAP_SEGMENT, seg_in=4, seg_out=5, seg_off=1)
    ref = (A @ B.t()).reshape(3, 4, N)
    close(out.reshape(3, 5, N)[:, 1:], ref, 1e-5)


def test_gemm_coskernel_epilogue():
    from oracle.roma_oracle import RomaOracle
    n, c, Bz = 100, 64, 2
    x, y = rnd(Bz, n, c, seed=1), rnd(Bz, n, c, seed=2)
    nx = torch.empty(Bz * n, device=DEV)
    ny = torch.empty(Bz * n, device=DEV)
    call("romab200_row_norms", "rb_rownorm_args", x=x, out=nx, rows=Bz * n, cols=c, ldx=c, dtype=F32)
    call("romab200_row_norms", "rb_rownorm_args", x=y, out=ny, rows=Bz * n, cols=c, ldx=c, dtype=F32)
    close(nx, x.norm(dim=-1).reshape(-1), 1e-5)
    K = torch.zeros(Bz, n, 104, device=DEV)
    gemm(x, y, K, n, n, c, c, c, 104, batch0=Bz, sa0=n * c, sb0=n * c, sc0=n * 104, epi=cabi.EPI_COSKERNEL, norm_a=nx, norm_b=ny,
         sna0=n, snb0=n, eps=1e-6, inv_t=5.0, diag_add=0.1, cos_normalized=0)
    ref = RomaOracle.cos_kernel(x.cpu(), y.cpu()) + 0.1 * torch.eye(n)
    close(K[..., :n], ref, 2e-6)


# ----------------------------------------------------------------------------------------------- row-wise
@pytest.mark.parametrize("rows,cols,out_dt", [(37, 1024, torch.float32), (3202, 1024, torch.float16), (5, 1024, torch.bfloat16),
                                              (37, 200, torch.float32), (9, 1000, torch.float16)])
def test_layernorm(rows, cols, out_dt):
    """cols == 1024 takes the row-in-registers kernel, everything else the generic warp-per-row one."""
    x, g, b = rnd(rows, cols, seed=1, scale=3.0), rnd(cols, seed=2), rnd(cols, seed=3)
    ldy = (cols + 7) // 8 * 8
    y = torch.zeros(rows, ldy, dtype=out_dt, device=DEV)
    code = {torch.float32: F32, torch.float16: cabi.RB_F16, torch.bfloat16: cabi.RB_BF16}[out_dt]
    call("romab200_layernorm", "rb_layernorm_args", x=x, y=y, gamma=g, beta=b, rows=rows, cols=cols, ldx=cols, ldy=ldy,
         dtype_x=F32, dtype_y=code, eps=1e-6)
    ref = F.layer_norm(x, (cols,), g, b, 1e-6)
    tol = {torch.float32: 2e-5, torch.float16: 1e-2, torch.bfloat16: 8e-2}[out_dt]
    close(y[:, :cols], ref, tol)


@pytest.mark.parametrize("cols", [1600, 2047, 2048, 2049, 2240, 2304, 4100])
@pytest.mark.parametrize("extra", [0, 12])
def test_softmax_split_rows(cols, extra):
    """Softmax of fp32 scores written as an RB_F16S pair (the parity mode's attention probabilities), up to 2048 columns by the
    warp-per-row kernel, beyond by the block-per-row one (decoders of coarse grids with more than 2048 tokens); `extra` makes
    the pitches ragged.  hi + lo 2^-11 against fp64, the pad columns of the last 4-element group zero and the rest of the pitch
    untouched, and bit for bit the in-place fp32 softmax of the same scores, split."""
    rows, c4 = 37, (cols + 3) // 4 * 4
    lds, ldo = c4 + extra, c4 + 2 * extra
    s = rnd(rows, lds, seed=cols, scale=3.0)
    hi = torch.full((rows, ldo), 7.0, dtype=torch.float16, device=DEV)
    lo = torch.full((rows, ldo), 7.0, dtype=torch.float16, device=DEV)
    call("romab200_softmax_rows", "rb_softmax_args", s=s, rows=rows, cols=cols, lds=lds, dtype=F32, scale=1.0, out_hi=hi, out_lo=lo, ldo=ldo)
    ref = torch.softmax(s[:, :cols].double(), -1).cpu()
    got = (hi[:, :cols].double() + lo[:, :cols].double() * 2.0 ** -11).cpu()
    err = ((got - ref).abs() - (2.0 ** -19 * ref + 2.0 ** -34)).max().item()
    assert err <= 0, f"split softmax off fp64 by {err:.3e} beyond the bar"
    for plane in (hi, lo):
        assert (plane[:, cols:c4] == 0).all() and (plane[:, c4:] == 7.0).all()
    inplace = s.clone()
    call("romab200_softmax_rows", "rb_softmax_args", s=inplace, rows=rows, cols=cols, lds=lds, dtype=F32, scale=1.0)
    p = inplace[:, :cols]
    p_hi = p.half()
    p_lo = ((p - p_hi.float()) * 2048.0).half()
    assert torch.equal(hi[:, :cols], p_hi) and torch.equal(lo[:, :cols], p_lo)


def test_copy_split_transpose_tokens_im2col():
    x = rnd(33, 20, seed=1)
    d = torch.zeros(33, 24, dtype=torch.float16, device=DEV)
    call("romab200_copy2d", "rb_copy2d_args", src=x, dst=d, rows=33, cols=20, lds=20, ldd=24, dtype_src=F32, dtype_dst=cabi.RB_F16)
    assert torch.equal(d[:, :20], x.half())
    nrm = x.norm(dim=-1).contiguous()
    sp = torch.zeros(33, 64, dtype=torch.float16, device=DEV)
    call("romab200_split_f16x3", "rb_split_args", x=x, dst=sp, rows=33, cols=20, ldx=20, ldd=64, row_norm=nrm, layout_b=0)
    xn = x / nrm[:, None]
    hi = xn.half()
    lo = (xn - hi.float()).half()
    assert torch.equal(sp[:, :20], hi) and torch.equal(sp[:, 20:40], lo) and torch.equal(sp[:, 40:60], hi)
    close(hi.float() + lo.float(), xn, 2e-7)
    t = rnd(2, 3, 45, 70, seed=2)
    o = torch.zeros(2, 3, 70, 48, device=DEV)
    call("romab200_transpose", "rb_transpose_args", src=t, dst=o, rows=45, cols=70, lds=70, ldd=48, batch0=2, batch1=3,
         ss0=3 * 45 * 70, ss1=45 * 70, sd0=3 * 70 * 48, sd1=70 * 48, dtype=F32)
    assert torch.equal(o[..., :45], t.transpose(-1, -2))
    img = rnd(2, 3, 28, 42, seed=3)
    cols = torch.zeros(2 * 2 * 3, 592, device=DEV)
    call("romab200_im2col_patch", "rb_im2col_args", image=img, out=cols, batch=2, height=28, width=42, patch=14, ldo=592, dtype_out=F32)
    w = rnd(8, 3, 14, 14, seed=4)
    ref = F.conv2d(img, w, stride=14).flatten(2).transpose(1, 2).reshape(-1, 8)
    close(cols[:, :588] @ w.flatten(1).t(), ref, 1e-4)
    patch, cls, pos = rnd(2 * 6, 16, seed=5), rnd(16, seed=6), rnd(7, 16, seed=7)
    tok = torch.zeros(2, 7, 16, device=DEV)
    call("romab200_assemble_tokens", "rb_tokens_args", patch=patch, cls=cls, pos=pos, tokens=tok, batch=2, npatch=6, dim=16)
    ref = torch.cat((cls.expand(2, 1, 16), patch.reshape(2, 6, 16)), 1) + pos
    assert torch.equal(tok, ref)


# ----------------------------------------------------------------------------------------------- VGG pieces
def test_conv_first_and_maxpool():
    E, H, W = 2, 14, 150
    img = rnd(E, 3, H, W, seed=1)
    w, b = rnd(64, 3, 3, 3, seed=2, scale=0.3), rnd(64, seed=3)
    out = torch.zeros(E, H + 2, W + 2, 64, device=DEV)
    call("romab200_conv3x3_first", "rb_conv_first_args", image=img, out=out, weight=w.reshape(64, 27).contiguous(), bias=b,
         batch=E, height=H, width=W, cout=64, dtype_out=F32)
    ref = F.relu(F.conv2d(img, w, b, padding=1)).permute(0, 2, 3, 1)
    close(out[:, 1:-1, 1:-1], ref, 1e-5)
    assert out[:, 0].abs().max() == 0 and out[:, :, -1].abs().max() == 0
    pooled = torch.zeros(E, H // 2 + 2, W // 2 + 2, 64, device=DEV)
    call("romab200_maxpool2x2_padded", "rb_maxpool_args", **{"in": out}, out=pooled, batch=E, height=H, width=W, channels=64, dtype=F32)
    refp = F.max_pool2d(out[:, 1:-1, 1:-1].permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)
    assert torch.equal(pooled[:, 1:-1, 1:-1], refp)
    assert pooled[:, 0].abs().max() == 0 and pooled[:, :, 0].abs().max() == 0


# ----------------------------------------------------------------------------------------------- GP solve
@pytest.mark.parametrize("algo", [0, 1, 2, 3])
@pytest.mark.parametrize("n,nrhs,batch", [(64, 40, 2), (100, 512, 1), (1600, 512, 2), (224, 70, 3), (1408, 512, 2), (1600, 512, 5)])
def test_gp_solve(n, nrhs, batch, algo):
    g = torch.Generator().manual_seed(n)
    feats = torch.randn(batch, n, 48, generator=g)
    feats = feats / feats.norm(dim=-1, keepdim=True)
    Kyy = ((feats @ feats.transpose(1, 2) - 1) / 0.2).exp() + 0.1 * torch.eye(n)
    Fm = torch.cos(torch.randn(n, nrhs, generator=g) * 3)
    ref = torch.cholesky_solve(Fm[None].expand(batch, n, nrhs).double(), torch.linalg.cholesky(Kyy.double()))
    ldw = (n + 7) // 8 * 8
    Wk = torch.zeros(batch, n + nrhs, ldw)
    Wk[:, :n, :n] = Kyy
    Wk[:, n:, :n] = Fm.t()
    Wk = Wk.to(DEV)
    ws_floats = max(batch * ((n + 31) // 32) * 1024 + 1, batch * ((n + 127) // 128) * 16384)
    if algo == 3:         # block inverses + split-fp16 scratch pairs of the tensor-core variant (include/romab200.h)
        ws_floats = batch * (((n + 127) // 128) * 16384 + max((n + nrhs) * 128 + 16384, nrhs * 128 + 16384 + 128 * ldw))
    ws = torch.empty(ws_floats, device=DEV)
    call("romab200_gp_solve", "rb_gp_solve_args", W=Wk, n=n, nrhs=nrhs, batch=batch, ldw=ldw, stride=(n + nrhs) * ldw,
         workspace=ws if algo else None, workspace_bytes=ws_floats * 4 if algo else 0, algo=algo)
    torch.cuda.synchronize()
    alpha_t = Wk[:, n:, :n].cpu()
    err = (alpha_t.transpose(1, 2).double() - ref).abs().max().item()
    assert err < 5e-4 * ref.abs().max().item(), err
    if algo != 1:            # in-place variants (0, 2, 3): the lower triangle now holds the Cholesky factor
        L = torch.tril(Wk[:, :n, :n].cpu().double())
        close((L @ L.transpose(1, 2)).float(), Kyy, 1e-5)


# ----------------------------------------------------------------------------------------------- decoder pieces
def test_cls_to_flow_refine():
    from oracle.roma_oracle import RomaOracle
    B, hh, ww = 2, 5, 6
    cls = rnd(B, 4097, hh, ww, seed=1, scale=4.0)
    cls[0, :4096, 0, 0] = 0.0                      # all-equal logits: argmax = 0, clamp duplicates
    cls[0, 4095, 0, 1] = 100.0                     # mode at the last anchor (clamped +1/+64)
    cls[0, 63, 0, 2] = 100.0                       # +1 wraps to the next row
    ref = RomaOracle.cls_to_flow_refine(cls[:, :4096].cpu())
    logits = torch.zeros(B * hh * ww, 4104, device=DEV)
    logits[:, :4097] = cls.permute(0, 2, 3, 1).reshape(-1, 4097)
    state = torch.zeros(B * hh * ww, 3, device=DEV)
    call("romab200_cls_to_flow_refine", "rb_cls_args", logits=logits, state=state, rows=B * hh * ww, ldl=4104, res=64, dtype=F32)
    close(state[:, :2].reshape(B, hh, ww, 2), ref, 2e-6)
    close(state[:, 2].reshape(B, hh, ww), cls[:, 4096], 0)


def _windows(r, h, w):
    return (torch.linspace(-2 * r / w, 2 * r / w, 2 * r + 1).to(DEV), torch.linspace(-2 * r / h, 2 * r / h, 2 * r + 1).to(DEV))


@pytest.mark.parametrize("r,c,h,w", [(7, 512, 10, 12), (3, 512, 14, 14), (2, 256, 21, 17), (2, 64, 9, 9)])
def test_local_corr(r, c, h, w):
    from oracle.roma_oracle import RomaOracle
    B = 2
    f0, f1 = rnd(B, c, h, w, seed=1), rnd(B, c, h, w, seed=2)
    flow = (torch.rand(B, 2, h, w, generator=torch.Generator().manual_seed(3)) * 2.6 - 1.3)     # includes out-of-image
    ref = RomaOracle.local_correlation(f0.cpu(), f1.cpu(), r, flow)
    K = (2 * r + 1) ** 2
    f0c, f1c = f0.permute(0, 2, 3, 1).contiguous(), f1.permute(0, 2, 3, 1).contiguous()
    fl = flow.permute(0, 2, 3, 1).contiguous().to(DEV)
    out = torch.zeros(B, h, w, K, device=DEV)
    wx, wy = _windows(r, h, w)
    call("romab200_local_corr", "rb_local_corr_args", f0=f0c, f1=f1c, ldf0=c, ldf1=c, f0_img_stride=h * w * c, f1_img_stride=h * w * c,
         flow=fl, ldflow=2, out=out, ldo=K, batch=B, h=h, w=w, c=c, radius=r, scale=1.0 / math.sqrt(c), dtype_f=F32, dtype_out=F32,
         n_img=B, y_shift=0, win_x=wx, win_y=wy)
    close(out.permute(0, 3, 1, 2), ref, 3e-5)


@pytest.mark.parametrize("s", [16, 8, 4, 2, 1])
def test_refiner_prologue_blocks_tail(weights, s):
    """prologue + 9 x (dwconv, pointwise GEMM) + tail against the oracle's refiner on the same inputs."""
    from oracle.roma_oracle import RomaOracle
    from roma_b200 import arch
    from roma_b200.packing import PackedWeights, pad8
    spec = arch.REFINERS[s]
    h, w = (6, 7) if s >= 4 else (12, 10)
    E = D = 2
    orc = RomaOracle(weights[0], weights[1])
    feat = rnd(E, spec.feat, h, w, seed=s)
    flow = (torch.rand(D, 2, h, w, generator=torch.Generator().manual_seed(s + 1)) * 2.2 - 1.1)
    cert = torch.randn(D, 1, h, w, generator=torch.Generator().manual_seed(s + 2))
    fc = feat.cpu()
    x, y = fc, torch.cat((fc[1:], fc[:1]))
    sf = 1.3
    d_ref = orc.refiner_input(s, x, y, flow, sf)
    out_ref = orc.refiner_blocks(s, d_ref)
    # --- ours
    pw = _packed(weights)
    R = pw.refiner[s]
    cp, c = R["cp"], R["c"]
    ldf = pad8(spec.feat)
    featc = torch.zeros(E, h, w, ldf, device=DEV)
    featc[..., :spec.feat] = feat.permute(0, 2, 3, 1)
    state = torch.cat((flow, cert), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    state0 = state.clone()
    d = torch.zeros(D * h * w, cp, device=DEV)
    t = torch.zeros(D * h * w, cp, device=DEV)
    gx = torch.linspace(-1 + 1 / w, 1 - 1 / w, w).to(DEV)
    gy = torch.linspace(-1 + 1 / h, 1 - 1 / h, h).to(DEV)
    r = spec.radius
    wx, wy = _windows(r, h, w) if r else (None, None)
    call("romab200_refiner_prologue", "rb_refiner_prologue_args", feat=featc, ldf=ldf, n_img=E, y_shift=1, state=state, d=d, ldd=cp,
         D=D, h=h, w=w, cf=spec.feat, emb=spec.emb, radius=r, dtype=F32, emb_weight=R["emb_w"], emb_bias=R["emb_b"],
         disp_scale=float(torch.tensor(40 / 32 * sf, dtype=torch.float32)), grid_x=gx, grid_y=gy, win_x=wx, win_y=wy)
    close(d.view(D, h, w, cp)[..., :c].permute(0, 3, 1, 2), d_ref, 5e-5)
    for blk in R["blocks"]:
        call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": d}, out=t, ldi=cp, ldo=cp, weight=blk["dw_w"], ldw=cp, bias=blk["dw_b"],
             batch=D, h=h, w=w, c=c, dtype=F32)
        gemm(t, blk["pw_w"], d, D * h * w, c, c, cp, cp, cp, bias=blk["pw_b"])
    delta = torch.zeros(D * h * w, 3, device=DEV)
    call("romab200_refiner_tail", "rb_refiner_tail_args", d=d, ldd=cp, weight=R["out_w"], ldw=cp, bias=R["out_b"], state=state,
         rows=D * h * w, c=c, scale_x=0.5, scale_y=0.25, dtype=F32, delta_out=delta)
    tol = 2e-3 if s in (8, 4) else 5e-4          # O(10) activations through 9 blocks
    close(delta.view(D, h, w, 3).permute(0, 3, 1, 2), out_ref, tol)
    exp_state = state0 + delta.view(D, h, w, 3) * torch.tensor([0.5, 0.25, 1.0], device=DEV)
    close(state, exp_state, 1e-6)


@pytest.mark.parametrize("s,h,w,kind", [(16, 12, 10, "smooth"), (16, 9, 14, "shift"), (8, 20, 27, "smooth"), (8, 17, 24, "shift"), (8, 16, 16, "mixed"),
                                        (4, 23, 30, "smooth"), (4, 16, 24, "mixed"), (4, 40, 33, "random")])
def test_refiner_prologue_tile_pass(weights, s, h, w, kind):
    """refiner_prologue_tile_kernel<R> (one CTA per tile of pixels, the union of their windows staged in shared memory) against the
    oracle's refiner input and against the per-pixel kernel, on coherent flow (identity + sub-pixel noise; shifted so that windows
    leave the image), on flow that is coherent in one half only (the other half falls back to the per-pixel kernel) and on random flow."""
    from oracle.roma_oracle import RomaOracle
    from roma_b200 import arch
    from roma_b200.packing import pad8
    spec = arch.REFINERS[s]
    E = D = 2
    orc = RomaOracle(weights[0], weights[1])
    g = torch.Generator().manual_seed(100 * s + h)
    feat = rnd(E, spec.feat, h, w, seed=s + 7)
    ys, xs = torch.linspace(-1 + 1 / h, 1 - 1 / h, h), torch.linspace(-1 + 1 / w, 1 - 1 / w, w)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    ident = torch.stack((gx, gy))[None].expand(D, 2, h, w)
    noise = torch.randn(D, 2, h, w, generator=g) * torch.tensor([1.0 / w, 1.0 / h]).view(1, 2, 1, 1)          # 0.5 pixel
    if kind == "smooth":
        flow = ident + noise
    elif kind == "shift":                                  # windows of the border tiles leave the image on two sides
        flow = ident * 1.05 + noise + torch.tensor([0.35, -0.4]).view(1, 2, 1, 1)
    elif kind == "mixed":
        flow = ident + noise
        rnd_flow = torch.rand(D, 2, h, w, generator=g) * 2.2 - 1.1
        flow[:, :, :, w // 2:] = rnd_flow[:, :, :, w // 2:]
    else:
        flow = torch.rand(D, 2, h, w, generator=g) * 2.2 - 1.1
    cert = torch.zeros(D, 1, h, w)
    fc = feat.cpu()
    sf = 1.3
    d_ref = orc.refiner_input(s, fc, torch.cat((fc[1:], fc[:1])), flow, sf)
    R = _packed(weights).refiner[s]
    cp, c = R["cp"], R["c"]
    ldf = pad8(spec.feat)
    featc = torch.zeros(E, h, w, ldf, device=DEV)
    featc[..., :spec.feat] = feat.permute(0, 2, 3, 1)
    state = torch.cat((flow, cert), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    r = spec.radius
    ntiles = D * cabi.prologue_tiles(r, h, w)
    wx, wy = _windows(r, h, w)
    outs = []
    for tiles in (torch.full((ntiles,), 7, dtype=torch.uint8, device=DEV), None):
        d = torch.zeros(D * h * w, cp, device=DEV)
        call("romab200_refiner_prologue", "rb_refiner_prologue_args", feat=featc, ldf=ldf, n_img=E, y_shift=1, state=state, d=d, ldd=cp,
             D=D, h=h, w=w, cf=spec.feat, emb=spec.emb, radius=r, dtype=F32, emb_weight=R["emb_w"], emb_bias=R["emb_b"],
             disp_scale=float(torch.tensor(40 / 32 * sf, dtype=torch.float32)), grid_x=xs.to(DEV), grid_y=ys.to(DEV), win_x=wx, win_y=wy,
             tile_done=tiles, tile_done_len=ntiles if tiles is not None else 0)
        outs.append(d)
        if tiles is not None:
            done = tiles.cpu()
            assert ((done == 0) | (done == 1)).all()                   # every tile reports
            frac = done.float().mean().item()
            if kind in ("smooth", "shift"):
                assert frac == 1.0, frac
            elif kind == "mixed":
                assert 0.0 < frac < 1.0, frac
            else:
                assert frac < 0.5, frac
    close(outs[0].view(D, h, w, cp)[..., :c].permute(0, 3, 1, 2), d_ref, 5e-5)
    close(outs[0], outs[1], 2e-5)
    assert (outs[0][:, c:] == 0).all()                                  # the zero padding of the rows is left alone


@pytest.mark.parametrize("h,w", [(12, 10), (7, 9)])
def test_refiner_prologue_corr_table(weights, h, w):
    """Stride-16 prologue with the window dot products gathered from an all-pairs table (rb_refiner_prologue_args.corr_table) built by
    romab200_gemm from split-fp16 pairs, against the oracle's refiner input."""
    from oracle.roma_oracle import RomaOracle
    from roma_b200 import arch
    from roma_b200.packing import pad8
    s = 16
    spec = arch.REFINERS[s]
    E = D = 2
    n = h * w
    orc = RomaOracle(weights[0], weights[1])
    feat = rnd(E, spec.feat, h, w, seed=3)
    flow = (torch.rand(D, 2, h, w, generator=torch.Generator().manual_seed(5)) * 2.2 - 1.1)
    fc = feat.cpu()
    sf = 1.0
    d_ref = orc.refiner_input(s, fc, torch.cat((fc[1:], fc[:1])), flow, sf)
    R = _packed(weights).refiner[s]
    cp, c = R["cp"], R["c"]
    cf = spec.feat
    featc = feat.permute(0, 2, 3, 1).contiguous().to(DEV)                       # [E, h, w, 512]
    hi = torch.empty(E * n, cf, dtype=torch.float16, device=DEV)
    lo = torch.empty(E * n, cf, dtype=torch.float16, device=DEV)
    call("romab200_split_f16s", "rb_split_pair_args", x=featc, hi=hi, lo=lo, rows=E * n, cols=cf, ldx=cf, ldd=cf)
    ldt = pad8(n)
    table = torch.zeros(D, n, ldt, device=DEV)
    for i0, y0 in ((0, 1), (1, 0)):
        call("romab200_gemm", "rb_gemm_args", A=hi[i0 * n:], A_lo=lo[i0 * n:], B=hi[y0 * n:], B_lo=lo[y0 * n:], C=table[i0], M=n, N=n, K=cf, lda=cf, ldb=cf,
             ldc=ldt, dtype_ab=cabi.RB_F16S, dtype_c=F32, batch0=1, batch1=1, ntaps=1, alpha=float(torch.rsqrt(torch.tensor(float(cf)))))
    ref_tab = torch.einsum("bpc,bqc->bpq", featc.view(E, n, cf).double(), featc.view(E, n, cf).double()[[1, 0]]) / math.sqrt(cf)
    close(table[:, :, :n], ref_tab.float(), 2e-5)
    state = torch.cat((flow, torch.zeros(D, 1, h, w)), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    xs, ys = torch.linspace(-1 + 1 / w, 1 - 1 / w, w), torch.linspace(-1 + 1 / h, 1 - 1 / h, h)
    wx, wy = _windows(spec.radius, h, w)
    d = torch.zeros(D * n, cp, device=DEV)
    call("romab200_refiner_prologue", "rb_refiner_prologue_args", feat=featc, ldf=cf, n_img=E, y_shift=1, state=state, d=d, ldd=cp,
         D=D, h=h, w=w, cf=cf, emb=spec.emb, radius=spec.radius, dtype=F32, emb_weight=R["emb_w"], emb_bias=R["emb_b"],
         disp_scale=float(torch.tensor(40 / 32 * sf, dtype=torch.float32)), grid_x=xs.to(DEV), grid_y=ys.to(DEV), win_x=wx, win_y=wy,
         corr_table=table, ld_corr_table=ldt)
    close(d.view(D, h, w, cp)[..., :c].permute(0, 3, 1, 2), d_ref, 5e-5)


_PACKED = {}


def _packed(weights):
    from roma_b200.packing import PackedWeights
    if "w" not in _PACKED:
        _PACKED["w"] = PackedWeights(weights[0], weights[1], torch.device(DEV), torch.float32)
    return _PACKED["w"]


def test_dwconv_matches_conv2d():
    B, C, H, W = 2, 50, 19, 37
    x = rnd(B, C, H, W, seed=1)
    w, b = rnd(C, 1, 5, 5, seed=2, scale=0.3), rnd(C, seed=3)
    ref = F.relu(F.conv2d(x, w, b, padding=2, groups=C)).permute(0, 2, 3, 1)
    ld = 56
    xi = torch.zeros(B, H, W, ld, device=DEV)
    xi[..., :C] = x.permute(0, 2, 3, 1)
    wt = torch.zeros(25, ld, device=DEV)
    wt[:, :C] = w.reshape(C, 25).t()
    out = torch.zeros(B, H, W, ld, device=DEV)
    call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": xi}, out=out, ldi=ld, ldo=ld, weight=wt, ldw=ld, bias=b, batch=B, h=H, w=W, c=C, dtype=F32)
    close(out[..., :C], ref, 1e-5)


@pytest.mark.parametrize("hi,wi,ho,wo", [(8, 8, 14, 14), (40, 40, 70, 70), (56, 56, 21, 21), (7, 9, 13, 5)])
def test_bilinear_resize(hi, wi, ho, wo):
    x = rnd(2, 3, hi, wi, seed=1)
    ref = F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
    xi = x.permute(0, 2, 3, 1).contiguous()
    out = torch.zeros(2, ho, wo, 3, device=DEV)
    call("romab200_bilinear_resize", "rb_resize_args", **{"in": xi}, out=out, batch=2, hi=hi, wi=wi, ho=ho, wo=wo, c=3)
    close(out, ref, 2e-6)


@pytest.mark.parametrize("symmetric", [True, False])
def test_match_epilogue(symmetric):
    b, H, W, hc, wc = 2, 12, 10, 3, 4
    D = 2 * b if symmetric else b
    g = torch.Generator().manual_seed(5)
    flow = torch.rand(D, 2, H, W, generator=g) * 2.4 - 1.2
    cert = torch.randn(D, 1, H, W, generator=g) * 2
    c16 = torch.randn(D, 1, hc, wc, generator=g) * 2
    # reference semantics (matcher.py:839-850, 891-927)
    low = F.interpolate(c16, size=(H, W), align_corners=False, mode="bilinear")
    low = 0.5 * low * (low < 0)
    fl = flow.permute(0, 2, 3, 1)
    ce = (cert - low).sigmoid()
    ce[((fl.abs() > 1).sum(-1) > 0)[:, None]] = 0
    fl = fl.clamp(-1, 1)
    ys, xs = torch.linspace(-1 + 1 / H, 1 - 1 / H, H), torch.linspace(-1 + 1 / W, 1 - 1 / W, W)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    grid = torch.stack((gx, gy), -1)[None].expand(b, H, W, 2)
    if symmetric:
        a2b, b2a = fl.chunk(2)
        ref_w = torch.cat((torch.cat((grid, a2b), -1), torch.cat((b2a, grid), -1)), dim=2)
        ref_c = torch.cat(ce.chunk(2), dim=3)[:, 0]
    else:
        ref_w, ref_c = torch.cat((grid, fl), -1), ce[:, 0]
    state = torch.cat((flow, cert), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    cstate = torch.cat((torch.zeros(D, 2, hc, wc), c16), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    Wout = 2 * W if symmetric else W
    warp = torch.zeros(b, H, Wout, 4, device=DEV)
    co = torch.zeros(b, H, Wout, device=DEV)
    call("romab200_match_epilogue", "rb_match_epilogue_args", state=state, coarse_state=cstate, hc=hc, wc=wc, warp=warp, cert=co,
         b=b, H=H, W=W, symmetric=int(symmetric), grid_x=xs.to(DEV), grid_y=ys.to(DEV))
    close(warp, ref_w, 1e-6)
    close(co, ref_c, 2e-6)


def test_kde_density():
    from oracle.roma_oracle import RomaOracle
    n = 3000
    x = (torch.rand(n, 4, generator=torch.Generator().manual_seed(1)) * 2 - 1) * 0.7
    ref = RomaOracle.kde(x).float()
    out = torch.zeros(n, device=DEV)
    call("romab200_kde_density", "rb_kde_args", x=x.to(DEV), density=out, n=n, std=0.1, half=1)
    rel = ((out.cpu() - ref).abs() / ref.clamp_min(1.0)).max().item()
    assert rel < 0.02, rel
    out32 = torch.zeros(n, device=DEV)
    call("romab200_kde_density", "rb_kde_args", x=x.to(DEV), density=out32, n=n, std=0.1, half=0)
    ref32 = (-torch.cdist(x.double(), x.double()) ** 2 / (2 * 0.1 ** 2)).exp().sum(-1)
    close(out32, ref32.float(), 2e-3)
    # j range cut into splits summed in a fixed order (what sample() uses for its 40000 points): same densities up to the fp32 summation order
    for splits in (2, 5, 64):
        ws = torch.zeros(splits * n, device=DEV)
        outs = torch.zeros(n, device=DEV)
        call("romab200_kde_density", "rb_kde_args", x=x.to(DEV), density=outs, n=n, std=0.1, half=1, workspace=ws, splits=splits)
        ulp = (out.abs() * 2.0 ** -10).clamp_min(2.0 ** -14)               # one fp16 ulp of the rounded density
        assert ((outs - out).abs() <= ulp).all() and ((outs - out).abs() > 0).float().mean().item() < 0.02
        outs32 = torch.zeros(n, device=DEV)
        call("romab200_kde_density", "rb_kde_args", x=x.to(DEV), density=outs32, n=n, std=0.1, half=0, workspace=ws, splits=splits)
        close(outs32, out32, 1e-4)
    # symmetric schedule (every pair of 256-point blocks once, row and column sums credited): n = 3000 is 11.7 blocks (ragged last block)
    for nn, splits in ((n, 1), (n, 3), (n, 64), (700, 2), (256, 4), (257, 2)):
        xs = x[:nn].contiguous().to(DEV)
        ref_n = torch.zeros(nn, device=DEV)
        call("romab200_kde_density", "rb_kde_args", x=xs, density=ref_n, n=nn, std=0.1, half=1)
        nws = (splits + (nn + 255) // 256) * nn
        ws = torch.full((nws,), float("nan"), device=DEV)                   # every entry that is read must have been written
        outs = torch.zeros(nn, device=DEV)
        call("romab200_kde_density", "rb_kde_args", x=xs, density=outs, n=nn, std=0.1, half=1, workspace=ws, splits=splits, symmetric=1, workspace_floats=nws)
        assert torch.isfinite(outs).all()
        ulp = (ref_n.abs() * 2.0 ** -10).clamp_min(2.0 ** -14)
        assert ((outs - ref_n).abs() <= 2 * ulp).all(), ((outs - ref_n).abs() / ulp).max().item()
        assert ((outs - ref_n).abs() > 0).float().mean().item() < 0.05
        refo = RomaOracle.kde(x[:nn]).float()
        assert (((outs.cpu() - refo).abs() / refo.clamp_min(1.0)).max().item()) < 0.02
    with pytest.raises(RuntimeError):
        call("romab200_kde_density", "rb_kde_args", x=x.to(DEV), density=out, n=n, std=0.1, half=1, workspace=ws, splits=2, symmetric=1, workspace_floats=10)


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_local_corr_warp_wheel_signature(mode):
    """`romab200_local_corr_warp` = the fused-local-corr wheel's operator (local_correlation.py:22-35): arbitrary (non-lattice)
    warps incl. samples outside the image, against F.grid_sample + dot product."""
    B, C, H, W, K = 2, 48, 9, 11, 7
    f0, f1 = rnd(B, H * W, C, seed=1), rnd(B, H, W, C, seed=2)
    warp = (rnd(B, H * W, K, 2, seed=3) * 0.7).clamp(-1.3, 1.3).contiguous()
    out = torch.zeros(B, H * W, K, device=DEV)
    call("romab200_local_corr_warp", "rb_local_corr_warp_args", f0=f0, f1=f1, ldf0=C, ldf1=C, warp=warp, out=out, batch=B, h=H, w=W, c=C, k=K,
         mode=0 if mode == "bilinear" else 1)
    samp = F.grid_sample(f1.permute(0, 3, 1, 2), warp.reshape(B, H * W, K, 2), mode=mode, padding_mode="zeros", align_corners=False)   # [B,C,HW,K]
    ref = torch.einsum("bpc,bcpk->bpk", f0, samp)
    close(out, ref, 2e-5)


# ----------------------------------------------------------------------------------------------- 16-bit instantiations
# The fast mode runs the __half / bf16 instantiations of the kernels below; each is pinned here against the oracle evaluated on the
# SAME 16-bit-rounded inputs, so that only the kernel's own arithmetic (fp32 accumulation, one rounding at the store) is judged.
DT16 = [torch.float16, torch.bfloat16]
CODE16 = {torch.float16: cabi.RB_F16, torch.bfloat16: cabi.RB_BF16}
EPS16 = {torch.float16: 2.0 ** -10, torch.bfloat16: 2.0 ** -7}        # relative spacing of the storage format (x2 margin below)


@pytest.mark.parametrize("dt", DT16)
@pytest.mark.parametrize("r,c,h,w", [(7, 512, 10, 12), (3, 512, 14, 14), (2, 256, 21, 17)])
def test_local_corr_16bit(dt, r, c, h, w):
    """local_corr_kernel<__half / bf16>: 16-bit features, fp32 accumulation; fp32 and 16-bit results."""
    from oracle.roma_oracle import RomaOracle
    B = 2
    f0, f1 = rnd(B, c, h, w, seed=1).to(dt), rnd(B, c, h, w, seed=2).to(dt)
    flow = (torch.rand(B, 2, h, w, generator=torch.Generator().manual_seed(3)) * 2.6 - 1.3)
    ref = RomaOracle.local_correlation(f0.float().cpu(), f1.float().cpu(), r, flow)
    K = (2 * r + 1) ** 2
    f0c, f1c = f0.permute(0, 2, 3, 1).contiguous(), f1.permute(0, 2, 3, 1).contiguous()
    fl = flow.permute(0, 2, 3, 1).contiguous().to(DEV)
    wx, wy = _windows(r, h, w)
    for out_dt, code in ((torch.float32, F32), (dt, CODE16[dt])):
        out = torch.zeros(B, h, w, K, dtype=out_dt, device=DEV)
        call("romab200_local_corr", "rb_local_corr_args", f0=f0c, f1=f1c, ldf0=c, ldf1=c, f0_img_stride=h * w * c, f1_img_stride=h * w * c,
             flow=fl, ldflow=2, out=out, ldo=K, batch=B, h=h, w=w, c=c, radius=r, scale=1.0 / math.sqrt(c), dtype_f=CODE16[dt], dtype_out=code,
             n_img=B, y_shift=0, win_x=wx, win_y=wy)
        tol = 5e-5 if out_dt == torch.float32 else 2 * EPS16[dt] * ref.abs().max().item()
        close(out.permute(0, 3, 1, 2), ref, tol)


@pytest.mark.parametrize("dt", DT16)
@pytest.mark.parametrize("s", [16, 8, 4, 2, 1])
def test_refiner_prologue_and_tail_16bit(weights, dt, s):
    """refiner_prologue_kernel<T, R> (x copy, grid_sample, displacement embedding, local correlation) and refiner_tail_kernel<T> on
    16-bit maps against the oracle on the rounded features."""
    from oracle.roma_oracle import RomaOracle
    from roma_b200 import arch
    from roma_b200.packing import pad8
    spec = arch.REFINERS[s]
    h, w = (6, 7) if s >= 4 else (12, 10)
    E = D = 2
    orc = RomaOracle(weights[0], weights[1])
    feat = rnd(E, spec.feat, h, w, seed=s).to(dt)
    flow = (torch.rand(D, 2, h, w, generator=torch.Generator().manual_seed(s + 1)) * 2.2 - 1.1)
    cert = torch.randn(D, 1, h, w, generator=torch.Generator().manual_seed(s + 2))
    fc = feat.float().cpu()
    sf = 1.3
    d_ref = orc.refiner_input(s, fc, torch.cat((fc[1:], fc[:1])), flow, sf)
    R = _packed(weights).refiner[s]
    cp, c = R["cp"], R["c"]
    ldf = pad8(spec.feat)
    featc = torch.zeros(E, h, w, ldf, dtype=dt, device=DEV)
    featc[..., :spec.feat] = feat.permute(0, 2, 3, 1)
    state = torch.cat((flow, cert), 1).permute(0, 2, 3, 1).contiguous().to(DEV)
    state0 = state.clone()
    d = torch.zeros(D * h * w, cp, dtype=dt, device=DEV)
    gx = torch.linspace(-1 + 1 / w, 1 - 1 / w, w).to(DEV)
    gy = torch.linspace(-1 + 1 / h, 1 - 1 / h, h).to(DEV)
    r = spec.radius
    wx, wy = _windows(r, h, w) if r else (None, None)
    call("romab200_refiner_prologue", "rb_refiner_prologue_args", feat=featc, ldf=ldf, n_img=E, y_shift=1, state=state, d=d, ldd=cp,
         D=D, h=h, w=w, cf=spec.feat, emb=spec.emb, radius=r, dtype=CODE16[dt], emb_weight=R["emb_w"], emb_bias=R["emb_b"],
         disp_scale=float(torch.tensor(40 / 32 * sf, dtype=torch.float32)), grid_x=gx, grid_y=gy, win_x=wx, win_y=wy)
    got = d.view(D, h, w, cp)[..., :c].permute(0, 3, 1, 2).float().cpu()
    err = (got - d_ref).abs()
    assert (err <= 2 * EPS16[dt] * d_ref.abs() + 1e-4).all(), err.max().item()        # one rounding of an fp32-accurate value
    # tail: fp32 head on the 16-bit map
    delta = torch.zeros(D * h * w, 3, device=DEV)
    call("romab200_refiner_tail", "rb_refiner_tail_args", d=d, ldd=cp, weight=R["out_w"], ldw=cp, bias=R["out_b"], state=state,
         rows=D * h * w, c=c, scale_x=0.5, scale_y=0.25, dtype=CODE16[dt], delta_out=delta)
    ref_delta = d[:, :c].double() @ R["out_w"][:, :c].double().t() + R["out_b"].double()
    close(delta, ref_delta, 2e-5 * max(1.0, ref_delta.abs().max().item()))
    close(state, state0 + delta.view(D, h, w, 3) * torch.tensor([0.5, 0.25, 1.0], device=DEV), 1e-6)


@pytest.mark.parametrize("dt", DT16)
def test_cls_to_flow_refine_16bit(dt):
    """cls_to_flow_kernel<__half / bf16>: softmax / argmax / 5-neighbour soft-argmax on 16-bit logits (fp32 inside)."""
    from oracle.roma_oracle import RomaOracle
    B, hh, ww = 2, 5, 6
    cls = rnd(B, 4097, hh, ww, seed=1, scale=4.0).to(dt)
    cls[0, :4096, 0, 0] = 0.0
    cls[0, 4095, 0, 1] = 100.0
    cls[0, 63, 0, 2] = 100.0
    ref = RomaOracle.cls_to_flow_refine(cls[:, :4096].float().cpu())
    logits = torch.zeros(B * hh * ww, 4104, dtype=dt, device=DEV)
    logits[:, :4097] = cls.permute(0, 2, 3, 1).reshape(-1, 4097)
    state = torch.zeros(B * hh * ww, 3, device=DEV)
    call("romab200_cls_to_flow_refine", "rb_cls_args", logits=logits, state=state, rows=B * hh * ww, ldl=4104, res=64, dtype=CODE16[dt])
    close(state[:, :2].reshape(B, hh, ww, 2), ref, 5e-6)
    close(state[:, 2].reshape(B, hh, ww), cls[:, 4096].float(), 0)


# ----------------------------------------------------------------------------------------------- device-side sampling
def test_weighted_sample_kernel_is_a_draw_without_replacement():
    """romab200_weighted_sample: k distinct indices, never an item of zero weight while positive ones remain, inclusion frequencies
    proportional to the weights (for k << n), the three weight transforms, batching, determinism under the seed (ties included)."""
    n, k, B = 20000, 500, 3
    g = torch.Generator().manual_seed(0)
    vals = torch.rand(B, n, generator=g)
    vals[:, ::7] = 0.0                                     # zero weights are never drawn
    vals = vals.to(DEV).contiguous()

    def draw(seed, transform=cabi.SAMPLE_IDENTITY, param=0.0, values=vals, kk=k):
        idx = torch.full((values.shape[0], kk), -1, dtype=torch.int32, device=DEV)
        w = torch.zeros(values.shape[0], kk, device=DEV)
        keys = torch.empty(values.shape[0] * values.shape[1], device=DEV)
        scratch = torch.empty(values.shape[0] * 2056, dtype=torch.int32, device=DEV)
        call("romab200_weighted_sample", "rb_sample_args", values=values, n=values.shape[1], k=kk, batch=values.shape[0], stride=values.shape[1],
             seed=seed, transform=transform, param=param, out_idx=idx, out_weights=w, keys=keys, scratch=scratch)
        return idx.long(), w
    idx, w = draw(1)
    for b in range(B):
        assert idx[b].min() >= 0 and idx[b].unique().numel() == k
        assert (vals[b][idx[b]] > 0).all() and torch.equal(w[b], vals[b][idx[b]])
    assert torch.equal(draw(1)[0].sort(-1).values, idx.sort(-1).values) and not torch.equal(draw(2)[0].sort(-1).values, idx.sort(-1).values)
    assert not torch.equal(idx[0].sort().values, idx[1].sort().values)          # batch items use different streams
    # inclusion frequency ~ weight: items of weight in [0.9, 1] are drawn ~9.5x as often as items in [0.05, 0.15]
    hi = ((vals[0] >= 0.9)).float()
    lo = ((vals[0] > 0.05) & (vals[0] <= 0.15)).float()
    cnt = torch.zeros(n, device=DEV)
    for s in range(200):
        cnt[draw(100 + s)[0][0]] += 1
    ratio = ((cnt * hi).sum() / hi.sum()) / ((cnt * lo).sum() / lo.sum())
    assert 8.0 < ratio.item() < 11.0, ratio.item()
    # transforms: thresholding makes everything above the threshold equally likely; balancing implements 1/(d+1) with the d < 10 floor
    idx_t, w_t = draw(3, cabi.SAMPLE_THRESHOLD, 0.05)
    assert ((w_t[0] == 1.0) | (w_t[0] <= 0.05)).all() and (w_t[0] == 1.0).float().mean() > 0.95
    dens = torch.cat((torch.full((1, 5000), 3.0), torch.full((1, 5000), 50.0), torch.full((1, 5000), 500.0)), 1).to(DEV)
    idx_b, _ = draw(4, cabi.SAMPLE_BALANCE, 0.0, values=dens, kk=1000)
    frac = [(idx_b[0] // 5000 == j).float().mean().item() for j in range(3)]
    assert frac[0] < 0.01 and 0.85 < frac[1] < 0.95 and 0.05 < frac[2] < 0.15, frac          # 1e-7 : 1/51 : 1/501
    # k == n returns every index once; more draws than positive weights falls back to zero-weight items
    small = torch.tensor([[0.0, 1.0, 2.0, 0.0, 3.0]], device=DEV)
    all_idx, _ = draw(5, values=small, kk=5)
    assert sorted(all_idx[0].tolist()) == [0, 1, 2, 3, 4]
    three, _ = draw(6, values=small, kk=3)
    assert sorted(three[0].tolist()) == [1, 2, 4]
    # ties at the cut (here the +inf keys of the zero weights) are drawn by index, so a draw depends on the seed only
    for s in range(20):
        assert sorted(draw(7 + s, values=small, kk=4)[0][0].tolist()) == [0, 1, 2, 4]
    assert all(torch.equal(draw(3, cabi.SAMPLE_THRESHOLD, 0.05)[0].sort(-1).values, idx_t.sort(-1).values) for _ in range(5))
