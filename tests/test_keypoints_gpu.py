"""`match_keypoints` on the device (csrc/keypoints.cu): the keypoint sampler against F.grid_sample, the mutual nearest neighbours
bit for bit against the exact-difference statement evaluated with float32 numpy ops, the reference's golden vectors, today's torch
statement on well-separated data, and a 100 000 x 100 000 problem in O(N) memory."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from roma_b200 import cabi
from roma_b200.matcher import RegressionMatcher, _keypoints_sample_device, _mutual_nn_device

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "helpers.npz"))
DEV = "cuda:0"


def _model():
    return RegressionMatcher.__new__(RegressionMatcher)


def exact_mnn(x_A_to_B, cert_A, x_B, max_dist, cert_th):
    """The device path's statement with explicit float32 numpy ops: D = sqrt(dx*dx + dy*dy), each operation rounded to fp32."""
    a, c, b = (np.asarray(t.cpu(), dtype=np.float32) for t in (x_A_to_B, cert_A, x_B))
    dx = a[:, None, 0] - b[None, :, 0]
    dy = a[:, None, 1] - b[None, :, 1]
    D = np.sqrt(dx * dx + dy * dy)
    with np.errstate(invalid="ignore"):
        mask = ((D == D.min(axis=1, keepdims=True)) & (D == D.min(axis=0, keepdims=True)) & (c[:, None] > np.float32(cert_th))
                & (D < np.float32(max_dist)))
    ia, ib = np.nonzero(mask)
    return torch.from_numpy(ia.astype(np.int64)), torch.from_numpy(ib.astype(np.int64))


def torch_statement(x_A, x_B, warp, certainty, max_dist, cert_th):
    x_A_to_B = F.grid_sample(warp[..., -2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False, mode="bilinear")[0, :, 0].mT
    cert = F.grid_sample(certainty[None, None], x_A[None, None], align_corners=False, mode="bilinear")[0, 0, 0]
    D = torch.cdist(x_A_to_B, x_B)
    mutual = (D == D.min(dim=-1, keepdim=True).values) * (D == D.min(dim=-2, keepdim=True).values)
    return torch.nonzero(mutual * (cert[:, None] > cert_th) * (D < max_dist), as_tuple=True)


def _check_mnn(x_A_to_B, cert_A, x_B, max_dist=0.005, cert_th=0.0):
    ia, ib = _mutual_nn_device(x_A_to_B.to(DEV), cert_A.to(DEV), x_B.to(DEV), max_dist, cert_th)
    ra, rb = exact_mnn(x_A_to_B, cert_A, x_B, max_dist, cert_th)
    assert ia.dtype == torch.int64 and ib.dtype == torch.int64
    assert torch.equal(ia.cpu(), ra) and torch.equal(ib.cpu(), rb)
    return ia.cpu(), ib.cpu()


def _identity_warp(h, w, g, disp=1e-3):
    """[h, w, 4] warp whose B half is the pixel-centre grid plus a small smooth displacement, so x_A_to_B ~ x_A."""
    xs = torch.linspace(-1 + 1 / w, 1 - 1 / w, w)
    ys = torch.linspace(-1 + 1 / h, 1 - 1 / h, h)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    grid = torch.stack((gx, gy), dim=-1)
    return torch.cat((grid, grid + disp * torch.sin(3 * grid + torch.rand(2, generator=g))), dim=-1)


def test_sampler_matches_grid_sample():
    g = torch.Generator().manual_seed(0)
    H, W = 23, 37
    warp_sym = (torch.rand(H, 2 * W, 4, generator=g) * 2 - 1).to(DEV)
    warp = warp_sym[:, :W]                                   # the A half of a symmetric warp: a non-contiguous view
    assert not warp.is_contiguous()
    cert = torch.rand(17, 29, generator=g).to(DEV)           # another size than the warp
    pts = torch.rand(3000, 2, generator=g) * 2.6 - 1.3      # inside and outside [-1, 1]
    border = torch.tensor([[-1, -1], [1, 1], [-1, 1], [1, -1], [-1, 0.3], [1, -0.2], [0.4, -1], [-0.7, 1],
                           [1 - 1 / W, 1 - 1 / H], [-1 + 1 / W, -1 + 1 / H], [1.0001, 0.0], [-1.0001, 0.0]], dtype=torch.float32)
    x = torch.cat((pts, border)).to(DEV)
    for wp, c in ((warp, cert), (warp_sym[:, :, 1:], cert.t()), (warp_sym.contiguous(), cert.contiguous())):
        xab, ca = _keypoints_sample_device(x, wp, c)
        ref_x = F.grid_sample(wp[..., -2:].permute(2, 0, 1)[None], x[None, None], align_corners=False, mode="bilinear")[0, :, 0].mT
        ref_c = F.grid_sample(c[None, None], x[None, None], align_corners=False, mode="bilinear")[0, 0, 0]
        assert (xab - ref_x).abs().max().item() <= 1e-6
        assert (ca - ref_c).abs().max().item() <= 1e-6
    far = torch.tensor([[1e30, 0.0], [0.0, -1e30]], device=DEV)
    xab, ca = _keypoints_sample_device(far, warp, cert)
    assert torch.equal(xab, torch.zeros_like(xab)) and torch.equal(ca, torch.zeros_like(ca))


def test_mnn_uniform_random():
    g = torch.Generator().manual_seed(1)
    a = torch.rand(1500, 2, generator=g) * 2 - 1
    b = torch.cat((a[:900] + 0.002 * torch.randn(900, 2, generator=g), torch.rand(800, 2, generator=g) * 2 - 1))
    c = torch.rand(1500, generator=g)
    ia, _ = _check_mnn(a, c, b, 0.005, 0.2)
    assert len(ia) > 100
    _check_mnn(a, c, b, 0.05, 0.0)
    _check_mnn(b[:1111], torch.rand(1111, generator=g), a, 0.01, 0.5)      # n_a < n_b and odd sizes


def test_mnn_clustered_near_ties():
    g = torch.Generator().manual_seed(2)
    centres = torch.rand(40, 2, generator=g) * 2 - 1
    a = centres[torch.randint(0, 40, (2000,), generator=g)] + 1e-6 * torch.randn(2000, 2, generator=g)
    b = centres[torch.randint(0, 40, (2500,), generator=g)] + 1e-6 * torch.randn(2500, 2, generator=g)
    b[::7] = torch.round(b[::7] * 1024) / 1024              # and some exactly representable coordinates
    a[::5] = torch.round(a[::5] * 1024) / 1024
    ia, _ = _check_mnn(a, torch.ones(2000), b)
    assert len(ia) > 10


def test_mnn_duplicates_give_every_tied_pair():
    g = torch.Generator().manual_seed(3)
    b = torch.rand(300, 2, generator=g) * 2 - 1
    b[10] = b[250] = b[40]                               # three identical x_B points
    a = b[:200].clone()
    a[120] = a[40]                                       # two identical x_A_to_B points, both at b[40]
    ia, ib = _check_mnn(a, torch.ones(200), b)
    both = [(i, j) for i, j in zip(ia.tolist(), ib.tolist()) if i in (10, 40, 120)]
    assert both == [(10, 10), (10, 40), (10, 250), (40, 10), (40, 40), (40, 250), (120, 10), (120, 40), (120, 250)]


def test_mnn_nan_propagates():
    g = torch.Generator().manual_seed(4)
    b = torch.rand(500, 2, generator=g) * 2 - 1
    a = b[:400] + 1e-4
    c = torch.ones(400)
    assert len(_check_mnn(a, c, b)[0]) > 300
    a_nan = a.clone()
    a_nan[3, 0] = float("nan")
    assert len(_check_mnn(a_nan, c, b)[0]) == 0
    b_nan = b.clone()
    b_nan[17, 1] = float("nan")
    assert len(_check_mnn(a, c, b_nan)[0]) == 0
    # grid samples at a NaN keypoint are NaN, so the whole call returns nothing, as the torch statement does
    x_A = torch.tensor([[0.1, 0.2], [float("nan"), 0.0], [-0.3, 0.5]], device=DEV)
    warp = _identity_warp(20, 30, g).to(DEV)
    cert = torch.ones(20, 30, device=DEV)
    ia, _ = _model().match_keypoints(x_A, x_A.clone(), warp, cert, return_inds=True)
    assert len(ia) == 0


def test_mnn_thresholds_are_strict():
    a = torch.tensor([[0.25, 0.5], [-0.5, -0.5], [0.75, -0.25]])
    b = torch.tensor([[0.25 + 3 / 1024, 0.5 - 1 / 256], [-0.5 + 1 / 512, -0.5], [0.75, -0.25 + 1 / 1024]])
    c = torch.tensor([0.5, 0.75, 0.625])
    d = np.sqrt(np.float32(3 / 1024) ** 2 + np.float32(1 / 256) ** 2, dtype=np.float32)
    above = float(np.nextafter(d, np.float32(1)))
    ia, ib = _check_mnn(a, c, b, max_dist=float(d), cert_th=0.4)          # row 0: D == max_dist
    assert ia.tolist() == [1, 2] and ib.tolist() == [1, 2]
    ia, _ = _check_mnn(a, c, b, max_dist=above, cert_th=0.5)              # row 0: cert == cert_th
    assert ia.tolist() == [1, 2]
    ia, _ = _check_mnn(a, c, b, max_dist=above, cert_th=0.4)
    assert ia.tolist() == [0, 1, 2]
    ia, _ = _check_mnn(a, c, b, max_dist=float(1 / 1024), cert_th=0.0)     # D == 1/1024 exactly for row 2
    assert ia.tolist() == []


def test_zero_matches_have_the_torch_shapes():
    m = _model()
    g = torch.Generator().manual_seed(5)
    warp = _identity_warp(16, 24, g)
    cert = torch.rand(16, 24, generator=g)
    x_A, x_B = torch.rand(50, 2, generator=g) * 2 - 1, torch.rand(60, 2, generator=g) * 2 - 1
    for kw in (dict(return_tuple=True, return_inds=True), dict(return_tuple=True, return_inds=False),
               dict(return_tuple=False, return_inds=True), dict(return_tuple=False, return_inds=False)):
        ref = m.match_keypoints(x_A, x_B, warp, cert, cert_th=2.0, **kw)
        out = m.match_keypoints(x_A.to(DEV), x_B.to(DEV), warp.to(DEV), cert.to(DEV), cert_th=2.0, **kw)
        ref, out = (ref, out) if isinstance(ref, tuple) else ((ref,), (out,))
        for r, o in zip(ref, out):
            assert o.is_cuda and o.shape == r.shape and o.dtype == r.dtype and o.numel() == 0


def test_golden_end_to_end():
    m = _model()
    W = G["warp"].shape[1] // 2
    warp = torch.from_numpy(G["warp"]).to(DEV)[:, :W]
    cert = torch.from_numpy(G["certainty"]).to(DEV)[:, :W]
    x_A, x_B = torch.from_numpy(G["x_A"]).to(DEV), torch.from_numpy(G["x_B"]).to(DEV)
    kw = dict(max_dist=0.005, cert_th=0.2)
    ia, ib = m.match_keypoints(x_A, x_B, warp, cert, return_tuple=True, return_inds=True, **kw)
    assert ia.is_cuda and torch.equal(ia.cpu(), torch.from_numpy(G["kp_inds_A"])) and torch.equal(ib.cpu(), torch.from_numpy(G["kp_inds_B"]))
    cat = m.match_keypoints(x_A, x_B, warp, cert, return_tuple=False, return_inds=False, **kw)
    assert torch.equal(cat.cpu(), torch.from_numpy(G["kp_cat"]))
    ka, kb = m.match_keypoints(x_A, x_B, warp, cert, **kw)
    assert torch.equal(torch.cat((ka, kb), dim=-1), cat)
    inds = m.match_keypoints(x_A, x_B, warp, cert, return_tuple=False, return_inds=True, **kw)
    assert torch.equal(inds, torch.cat((ia, ib), dim=-1))
    assert len(m.match_keypoints(x_A, x_B, warp, cert, return_inds=True, cert_th=2.0)[0]) == 0


def test_matches_torch_statement_on_separated_points():
    """Every row's and column's second-nearest neighbour is >= 2e-3 farther than its nearest and |D - max_dist| > 2e-3, far beyond
    the error of cdist's expansion, so today's statement and the device path must return the same pairs."""
    g = torch.Generator().manual_seed(6)
    k = torch.arange(40, dtype=torch.float32)
    gy, gx = torch.meshgrid(k, k, indexing="ij")
    x_B = torch.stack((gx, gy), dim=-1).reshape(-1, 2) * 0.048 - 0.94           # 1600 points, 0.048 apart
    ang = torch.rand(1600, generator=g) * 2 * np.pi
    near = torch.rand(1600, generator=g) < 0.7
    r = torch.where(near, 5e-4 + 2e-3 * torch.rand(1600, generator=g), torch.full((1600,), 0.016))
    x_A = x_B + r[:, None] * torch.stack((ang.cos(), ang.sin()), dim=-1)
    x_A = x_A[torch.randperm(1600, generator=g)]
    warp = _identity_warp(48, 64, g, disp=0.0)
    cert = torch.rand(48, 64, generator=g)
    ref_xab = F.grid_sample(warp[..., 2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False)[0, :, 0].mT.double()
    D = torch.cdist(ref_xab, x_B.double())
    for d in (D, D.t()):
        two = d.topk(2, dim=1, largest=False).values
        assert (two[:, 1] - two[:, 0]).min() > 2e-3
    assert (D - 0.005).abs().min() > 2e-3
    ref_c = F.grid_sample(cert[None, None], x_A[None, None], align_corners=False)[0, 0, 0].sort().values
    mid = ref_c[400:1200]
    gap = int((mid[1:] - mid[:-1]).argmax())
    cert_th = float((mid[gap] + mid[gap + 1]) / 2)                          # a threshold far from every sampled certainty
    args = [t.to(DEV) for t in (x_A, x_B, warp, cert)]
    for th in (0.0, cert_th):
        ia, ib = _model().match_keypoints(*args, return_inds=True, cert_th=th)
        ra, rb = torch_statement(*args, 0.005, th)
        assert len(ia) > 300 and torch.equal(ia, ra) and torch.equal(ib, rb)


def test_scale_100k_in_linear_memory():
    n = 100_000
    g = torch.Generator(device=DEV).manual_seed(7)
    x_A = torch.rand(n, 2, device=DEV, generator=g) * 2 - 1
    x_B = torch.cat((x_A[: n // 2] + 2e-3 * torch.randn(n // 2, 2, device=DEV, generator=g), torch.rand(n // 2, 2, device=DEV, generator=g) * 2 - 1))
    x_B = x_B[torch.randperm(n, device=DEV, generator=g)]
    warp = _identity_warp(512, 512, torch.Generator().manual_seed(7)).to(DEV)
    cert = torch.rand(512, 512, device=DEV, generator=g)
    m = _model()
    m.match_keypoints(x_A[:1000], x_B[:1000], warp, cert)               # warm-up: library load, first launches
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ia, ib = m.match_keypoints(x_A, x_B, warp, cert, return_inds=True, cert_th=0.1)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < 64 * 2 ** 20, growth
    ia2, ib2 = m.match_keypoints(x_A, x_B, warp, cert, return_inds=True, cert_th=0.1)
    assert torch.equal(ia, ia2) and torch.equal(ib, ib2)
    assert len(ia) > 10_000
    # the same statement in row chunks with torch's fp32 elementwise ops (separate kernels: no contraction), on the kernel's own samples
    xab, ca = _keypoints_sample_device(x_A, warp, cert)
    chunk = 2000
    rowmin = torch.empty(n, device=DEV)
    colmin = torch.full((n,), float("inf"), device=DEV)

    def dist(s):
        dx = xab[s:s + chunk, None, 0] - x_B[None, :, 0]
        dy = xab[s:s + chunk, None, 1] - x_B[None, :, 1]
        return torch.sqrt(dx * dx + dy * dy)
    for s in range(0, n, chunk):
        D = dist(s)
        rowmin[s:s + chunk] = D.min(dim=1).values
        colmin = torch.minimum(colmin, D.min(dim=0).values)
    ra, rb = [], []
    for s in range(0, n, chunk):
        D = dist(s)
        mask = (D == rowmin[s:s + chunk, None]) & (D == colmin[None]) & (ca[s:s + chunk, None] > 0.1) & (D < 0.005)
        a, b = torch.nonzero(mask, as_tuple=True)
        ra.append(a + s)
        rb.append(b)
    assert torch.equal(ia, torch.cat(ra)) and torch.equal(ib, torch.cat(rb))


def test_empty_inputs_raise_index_error():
    m = _model()
    warp = torch.zeros(8, 8, 4, device=DEV)
    cert = torch.ones(8, 8, device=DEV)
    pts = torch.zeros(5, 2, device=DEV)
    for a, b in ((pts[:0], pts), (pts, pts[:0])):
        with pytest.raises(IndexError):
            m.match_keypoints(a, b, warp, cert)


def test_float64_takes_the_torch_statement(monkeypatch):
    g = torch.Generator().manual_seed(8)
    warp = _identity_warp(16, 24, g).double().to(DEV)
    cert = torch.rand(16, 24, generator=g).double().to(DEV)
    x_A = (torch.rand(300, 2, generator=g) * 2 - 1).double().to(DEV)
    x_B = x_A + 1e-3
    ref = torch_statement(x_A, x_B, warp, cert, 0.005, 0.1)

    def refuse(*a, **k):
        raise AssertionError("float64 inputs must not reach the C ABI")
    monkeypatch.setattr(cabi, "call", refuse)
    ia, ib = _model().match_keypoints(x_A, x_B, warp, cert, return_inds=True, cert_th=0.1)
    assert len(ia) > 100 and torch.equal(ia, ref[0]) and torch.equal(ib, ref[1])
