"""The GP posterior solve (`romab200_gp_solve`, all four schedules) against fp64 at the sizes where its blocked schedules have
ragged edges: the last 128-block and the last 32-panel of odd, ragged and full size (n = 1 ... 2240, the coarse grids
9 x 13 = 117, 41 x 41 = 1681 and 40 x 56 = 2240 among them), on the engine's layout (ldw = pad8(n), stride = (n + nrhs) ldw).

Two kinds of K_yy: random 48-d features (cos ~ 0 off the diagonal, well conditioned) and spatially smooth ones with a block of
identical rows, which push cond(K_yy + 0.1 I) towards its bound 10 n + 1 the way real DINOv2 projections do.

The bars are the error of the reference's own arithmetic on the same matrix (fp32 `torch.linalg.cholesky` + `cholesky_solve`,
matcher.py:307-308) times ERR_FACTOR = 8: the schedules run the same algorithm in fp32 with other summation orders (a factor of up
to 2 between two fp32 orders), and algo 3 contracts split-fp16 operand pairs, whose products are fp32-class at 2^-22 rather than
fp32's 2^-24 (a factor of 4).  The floor 2^-23 keeps the bar meaningful where fp32 happens to be exact (n = 1)."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from roma_b200.cabi import call  # noqa: E402

DEV = "cuda"
SIZES = [1, 3, 17, 81, 117, 127, 129, 255, 1681, 2240]
ERR_FACTOR, ERR_FLOOR = 8.0, 2.0 ** -23
SIGMA = 0.1
NAN_WORD = 0x7FC07FC0          # an fp32 NaN whose two halves are fp16 NaNs too (the split-fp16 scratch of algo 3)


def features(kind, n, batch, seed):
    """[batch, n, 48] unit rows (K_yy's features) and [batch, 64, 48] query rows (K_xy's)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "random":
        y, x = torch.randn(batch, n, 48, generator=g, dtype=torch.float64), torch.randn(batch, 64, 48, generator=g, dtype=torch.float64)
    else:
        # low-frequency functions of the token's grid position around one common direction: neighbouring tokens are nearly parallel
        w = max(1, math.ceil(math.sqrt(n)))
        freq = torch.randint(0, 3, (2, 47), generator=g).double()
        phase = torch.rand(batch, 1, 47, generator=g, dtype=torch.float64) * 2 * math.pi

        def smooth(py, px):
            arg = math.pi * (py[None, :, None] * freq[0] + px[None, :, None] * freq[1]) + phase
            return torch.cat((torch.ones(batch, py.numel(), 1, dtype=torch.float64), 0.04 * torch.cos(arg)), -1)
        i = torch.arange(n, dtype=torch.float64)
        y = smooth(torch.div(i, w, rounding_mode="floor") / w, (i % w) / w)
        q = torch.rand(2, 64, generator=g, dtype=torch.float64)
        x = smooth(q[0], q[1])
        b0, cnt = n // 3, min(8, n // 4)
        y[:, b0:b0 + cnt] = y[:, b0:b0 + 1]           # identical rows: K_yy singular, K_yy + 0.1 I as ill-conditioned as it gets
    return y / y.norm(dim=-1, keepdim=True), x / x.norm(dim=-1, keepdim=True)


def cos_kernel(a, b):
    return ((a @ b.transpose(1, 2) - 1) / 0.2).exp()            # CosKernel, T = 0.2 (matcher.py:191-200)


def rel(x, ref):
    """normwise relative error per problem"""
    return ((x - ref).flatten(1).norm(dim=1) / ref.flatten(1).norm(dim=1)).tolist()


_REF = {}


def reference(kind, n, nrhs, batch):
    key = (kind, n, nrhs, batch)
    if key not in _REF:
        y, x = features(kind, n, batch, seed=n * 7 + batch)
        K64 = cos_kernel(y, y) + SIGMA * torch.eye(n, dtype=torch.float64)
        K = K64.float()                                       # what the solve gets; the fp64 reference solves the same fp32 matrix
        F = torch.cos(torch.randn(n, nrhs, generator=torch.Generator().manual_seed(n), dtype=torch.float64) * 3)[None].expand(batch, n, nrhs)
        a64 = torch.cholesky_solve(F, torch.linalg.cholesky(K.double()))
        L32 = torch.linalg.cholesky(K)
        a32 = torch.cholesky_solve(F.float(), L32)
        Kxy = cos_kernel(x, y)
        ev = torch.linalg.eigvalsh(K.double())
        _REF[key] = dict(K=K, F=F.float(), a64=a64, Kxy=Kxy, mu64=Kxy @ a64, cond=(ev[:, -1] / ev[:, 0]).tolist(),
                         err_a32=rel(a32.double(), a64), err_mu32=rel(Kxy @ a32.double(), Kxy @ a64),
                         err_llt32=rel((L32 @ L32.transpose(1, 2)).double(), K.double()))
    return _REF[key]


def workspace_floats(algo, n, nrhs, batch, ldw):
    """the workspace size the header (include/romab200.h, rb_gp_solve_args) asks for, in floats"""
    nb32, nb128 = (n + 31) // 32, (n + 127) // 128
    if algo == 1:
        return batch * nb32 * 1024 + 1
    if algo == 2:
        return batch * nb128 * 16384
    return batch * (nb128 * 16384 + max((n + nrhs) * 128 + 16384, nrhs * 128 + 16384 + 128 * ldw))


@pytest.mark.parametrize("algo", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["random", "smooth"])
@pytest.mark.parametrize("nrhs,batch", [(512, 1), (77, 3)])
@pytest.mark.parametrize("n", SIZES)
def test_gp_solve_vs_fp64(n, nrhs, batch, kind, algo):
    r = reference(kind, n, nrhs, batch)
    ldw = (n + 7) // 8 * 8
    nan = torch.tensor([NAN_WORD], dtype=torch.int32).view(torch.float32).item()
    # the pad columns [n, ldw) and the strict upper triangle of K (which the solve must not read) hold NaN
    Wk = torch.full((batch, n + nrhs, ldw), nan)
    Wk[:, :n, :n] = torch.where(torch.ones(n, n, dtype=torch.bool).tril(), r["K"], torch.full_like(r["K"], nan))
    Wk[:, n:, :n] = r["F"].transpose(1, 2)
    Wk = Wk.to(DEV)
    ws = None
    nws = 0
    if algo:
        nws = workspace_floats(algo, n, nrhs, batch, ldw)
        ws = torch.full((nws,), NAN_WORD, dtype=torch.int32, device=DEV).view(torch.float32)   # every entry that is read must have been written
    call("romab200_gp_solve", "rb_gp_solve_args", W=Wk, n=n, nrhs=nrhs, batch=batch, ldw=ldw, stride=(n + nrhs) * ldw,
         workspace=ws, workspace_bytes=nws * 4, algo=algo)
    W = Wk.cpu()
    alpha = W[:, n:, :n].transpose(1, 2).double()
    assert torch.isfinite(alpha).all(), f"non-finite alpha: {(~torch.isfinite(alpha)).sum().item()} entries"
    err_a, err_mu = rel(alpha, r["a64"]), rel(r["Kxy"] @ alpha, r["mu64"])
    bar_a = [ERR_FACTOR * max(e, ERR_FLOOR) for e in r["err_a32"]]
    bar_mu = [ERR_FACTOR * max(e, ERR_FLOOR) for e in r["err_mu32"]]
    print(f"n={n} nrhs={nrhs} {kind} algo {algo}: cond {['%.3g' % c for c in r['cond']]} alpha err {['%.2e' % e for e in err_a]} "
          f"(fp32 reference {['%.2e' % e for e in r['err_a32']]}), mu err {['%.2e' % e for e in err_mu]} (fp32 reference {['%.2e' % e for e in r['err_mu32']]})")
    assert all(e <= b for e, b in zip(err_a, bar_a)), (err_a, bar_a)
    assert all(e <= b for e, b in zip(err_mu, bar_mu)), (err_mu, bar_mu)
    if algo != 1:            # in-place schedules (0, 2, 3): the lower triangle now holds the Cholesky factor
        L = torch.tril(W[:, :n, :n].double())
        err_l = rel(L @ L.transpose(1, 2), r["K"].double())
        bar_l = [ERR_FACTOR * max(e, ERR_FLOOR) for e in r["err_llt32"]]
        assert all(e <= b for e, b in zip(err_l, bar_l)), (err_l, bar_l)
    if ldw > n:              # pad columns: untouched beyond the 16-byte granule of the row tail, zeros or untouched inside it
        gran = (n + 3) // 4 * 4
        assert W[:, :, gran:].isnan().all() and (W[:, :, n:gran].isnan() | (W[:, :, n:gran] == 0)).all()
