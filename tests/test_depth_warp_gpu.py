"""The depth-based warps and the MegaDepth dense metric on the GPU (csrc/depth_warp.cu) against the torch oracle
(oracle/depth_warp.py) and the reference's goldens (tests/golden/make_golden_depth_warp.py)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from conftest import load_golden  # noqa: E402
from oracle import depth_warp as oracle  # noqa: E402
from roma_b200 import cabi, synthetic  # noqa: E402
from roma_b200.depth_warp import dense_geometric_dist, get_gt_warp, warp_kpts  # noqa: E402

DEV = "cuda:0"


def _close(ours, ref, rtol=1e-11):
    """Same NaN and inf positions, finite values within rtol * max(1, |ref|)."""
    ours, ref = ours.cpu(), ref.cpu()
    assert ours.shape == ref.shape and ours.dtype == ref.dtype
    assert torch.equal(torch.isnan(ours), torch.isnan(ref)) and torch.equal(torch.isinf(ours), torch.isinf(ref))
    fin = torch.isfinite(ref)
    err = ((ours[fin] - ref[fin]).abs() / ref[fin].abs().clamp(min=1)).max().item() if fin.any() else 0.0
    assert err <= rtol, err


def _bits(a, b):
    """Byte equality (NaN payloads included)."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))


def _boundary(details, h1, w1, thr=0.05):
    """Points whose decision sits within 1e-9 of a bound in the oracle: there the last bit of a sum may decide."""
    u, v, rel = (details[k].cpu() for k in ("u", "v", "rel"))
    near = (rel - thr).abs() <= 1e-9 * thr
    for x, hi in ((u, w1 - 1), (v, h1 - 1)):
        near |= (x.abs() <= 1e-9) | ((x - hi).abs() <= 1e-9)
    return near


def _check_valid(valid, ref_valid, details, h1, w1, thr=0.05):
    near = _boundary(details, h1, w1, thr).reshape(ref_valid.shape)
    assert near.sum().item() <= 8
    differ = valid.cpu().bool() != ref_valid.cpu().bool()
    assert not (differ & ~near).any(), int(differ.sum())


def _cuda(views):
    return [t.to(DEV) for t in views]


@pytest.fixture(scope="module")
def big():
    """The harness's shape: 8 pairs at 384 x 512, and 200 000 points per pair reaching past the image border."""
    views = synthetic.depth_scene(100, 8, 384, 512)
    g = torch.Generator().manual_seed(1)
    return views, torch.rand(8, 200_000, 2, generator=g, dtype=torch.float64) * 2.2 - 1.1


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_warp_kpts_on_the_reference_golden(mode):
    gd = load_golden("depth_warp")
    views = [torch.from_numpy(gd[k]).to(DEV) for k in ("depth0", "depth1", "T", "K0", "K1")]
    kpts = torch.from_numpy(gd["kpts"]).to(DEV)
    with torch.cuda.device(0):
        torch.cuda.set_sync_debug_mode("error")
        try:
            valid, warped = warp_kpts(kpts, *views, depth_interpolation_mode=mode)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert valid.dtype == torch.bool and valid.shape == (2, 3000) and warped.dtype == torch.float64 and warped.shape == (2, 3000, 2)
    _close(warped, torch.from_numpy(gd[f"warped_{mode}"]))
    d = {}
    oracle.warp_kpts(torch.from_numpy(gd["kpts"]), *[v.cpu() for v in views], depth_interpolation_mode=mode, details=d)
    _check_valid(valid, torch.from_numpy(gd[f"valid_{mode}"]), d, 60, 80)
    # get_gt_warp against the reference's: its pixel centres are float32 linspaces built by torch on the device in use
    same_grid = all(torch.equal(torch.linspace(-1 + 1 / n, 1 - 1 / n, n, device=DEV).cpu(), torch.linspace(-1 + 1 / n, 1 - 1 / n, n))
                    for n in (48, 64, 30, 44))
    for tag, hw in (("", {}), ("_hw", dict(H=30, W=44))):
        x2, prob = get_gt_warp(*views, depth_interpolation_mode=mode, **hw)
        _close(x2, torch.from_numpy(gd[f"x2{tag}_{mode}"]), 1e-11 if same_grid else 1e-6)
        assert (prob.cpu() != torch.from_numpy(gd[f"prob{tag}_{mode}"])).sum() <= (0 if same_grid else 8)


@pytest.mark.parametrize("kdtype, ddtype, mode", [(torch.float64, torch.float32, "bilinear"), (torch.float32, torch.float32, "bilinear"),
                                                  (torch.float32, torch.float64, "nearest"), (torch.float64, torch.float64, "bilinear")])
def test_warp_kpts_at_harness_size_vs_oracle(big, kdtype, ddtype, mode):
    views, kpts = big
    views = [views[0].to(ddtype), views[1].to(ddtype), *views[2:]]
    kpts = kpts.to(kdtype)
    valid, warped = warp_kpts(kpts.to(DEV), *_cuda(views), depth_interpolation_mode=mode)
    d = {}
    ref_valid, ref_warped = oracle.warp_kpts(kpts, *views, depth_interpolation_mode=mode, details=d)
    _close(warped, ref_warped)
    _check_valid(valid, ref_valid, d, 384, 512)
    fr = valid.double().mean().item()
    assert 0.15 < fr < 0.85, fr


def test_unequal_sizes_3x4_pose_threshold_and_strided_inputs():
    d0, d1, T, K0, K1 = synthetic.depth_scene(7, 3, 60, 80, 48, 64)
    g = torch.Generator().manual_seed(2)
    wide = torch.rand(3, 5000, 4, generator=g) * 2 - 1
    kpts = wide[..., 1:3]                                        # a non-contiguous view
    T34 = T[:, :3].float()                                       # [B, 3, 4], float32 like a data loader's
    padded = torch.zeros(3, 60, 100)
    padded[..., :80] = d0
    args = (kpts, padded[..., :80], d1, T34, K0.float(), K1)
    valid, warped = warp_kpts(*[a.to(DEV) for a in args], relative_depth_error_threshold=0.2)
    d = {}
    ref_valid, ref_warped = oracle.warp_kpts(*args, relative_depth_error_threshold=0.2, details=d)
    _close(warped, ref_warped)
    _check_valid(valid, ref_valid, d, 48, 64, 0.2)
    tight = warp_kpts(*[a.to(DEV) for a in args], relative_depth_error_threshold=0.01)[0]
    assert tight.sum() < valid.sum() and not (tight & ~valid).any()
    # the two maps in different dtypes
    v2, w2 = warp_kpts(kpts.to(DEV), d0.double().to(DEV), *[a.to(DEV) for a in args[2:]], relative_depth_error_threshold=0.2)
    assert _bits(w2, warped) and torch.equal(v2, valid)


def test_degenerate_points_and_empty_input():
    views = synthetic.depth_scene(9, 2, 40, 56)
    nan = float("nan")
    kpts = torch.tensor([[0.3, 0.2], [50.0, -80.0], [-1e30, 1e30], [nan, 0.0], [0.0, nan], [-1.0, -1.0], [1.0, 1.0]], dtype=torch.float64)
    kpts = kpts[None].expand(2, -1, -1).contiguous()
    views[0][1] = 0                                              # pair 1: zero depth everywhere in view 0
    views[1][0] = 0                                              # pair 0: zero depth under every warped point (0 / 0 in the consistency test)
    valid, warped = warp_kpts(kpts.to(DEV), *_cuda(views))
    ref_valid, ref_warped = oracle.warp_kpts(kpts, *views)
    assert not valid.any() and torch.equal(valid.cpu(), ref_valid)
    fin = torch.isfinite(ref_warped)
    assert torch.equal(torch.isfinite(warped.cpu()), fin)
    _close(torch.where(fin, warped.cpu(), torch.zeros(())), torch.where(fin, ref_warped, torch.zeros(())))
    valid, warped = warp_kpts(torch.zeros(2, 0, 2, device=DEV), *_cuda(views))
    assert valid.shape == (2, 0) and valid.dtype == torch.bool and warped.shape == (2, 0, 2) and warped.dtype == torch.float64
    with pytest.raises(RuntimeError, match=r"runs on the GPU only \(there is no CPU fallback\)"):
        warp_kpts(kpts, *_cuda(views))
    with pytest.raises(RuntimeError, match=r"runs on the GPU only \(there is no CPU fallback\)"):
        get_gt_warp(views[0], *_cuda(views)[1:])


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_gt_warp_is_warp_kpts_on_the_grid(big, mode):
    views = _cuda(big[0])
    for hw in ({}, dict(H=100, W=72)):
        H, W = hw.get("H", 384), hw.get("W", 512)
        x2, prob = get_gt_warp(*views, depth_interpolation_mode=mode, **hw)
        assert x2.shape == (8, H, W, 2) and x2.dtype == torch.float64 and prob.shape == (8, H, W) and prob.dtype == torch.float32
        xs, ys = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n, device=DEV) for n in (W, H))
        grid = torch.stack((xs[None].expand(H, W), ys[:, None].expand(H, W)), -1).reshape(1, H * W, 2).expand(8, -1, -1)
        for pts in (grid.contiguous(), grid.double()):           # float32 points widen exactly
            valid, warped = warp_kpts(pts, *views, depth_interpolation_mode=mode)
            assert _bits(warped.reshape(8, H, W, 2), x2) and torch.equal(valid.reshape(8, H, W).float(), prob)
        d = {}
        ref_x2, ref_prob = oracle.get_gt_warp(*views, depth_interpolation_mode=mode, details=d, **hw)      # the torch statement on the device
        _close(x2, ref_x2)
        _check_valid(prob, ref_prob, d, 384, 512)
        assert 0.2 < prob.mean().item() < 0.8


def _noisy_warp(views, seed, noise=2e-3):
    """A warp in the layout match() returns: (pixel centre, ground truth + noise), float32 [B, H, W, 4] on the CPU."""
    x2, _ = oracle.get_gt_warp(*views)
    B, H, W, _ = x2.shape
    g = torch.Generator().manual_seed(seed)
    xs, ys = torch.linspace(-1 + 1 / W, 1 - 1 / W, W), torch.linspace(-1 + 1 / H, 1 - 1 / H, H)
    grid = torch.stack((xs[None].expand(H, W), ys[:, None].expand(H, W)), -1)[None].expand(B, -1, -1, -1)
    x2 = torch.where(torch.isfinite(x2), x2, torch.zeros(())).float()
    return torch.cat((grid, x2 + noise * torch.randn(B, H, W, 2, generator=g) * torch.rand(B, 1, 1, 1, generator=g) * 4), dim=-1)


def _check_dense(res, ref, details, h1, w1):
    gd, pck_1, pck_3, pck_5, prob = res
    assert gd.dtype == torch.float64 and prob.dtype == torch.float32 and res.pair_count.dtype == torch.int64 and res.pair_sum.dtype == torch.float64
    for p in (pck_1, pck_3, pck_5):
        assert p.dim() == 0 and p.dtype == torch.float32 and p.is_cuda
    assert res.epe.dim() == 0 and res.epe.dtype == torch.float64
    assert torch.equal(torch.isnan(gd), prob != 1)
    near = _boundary(details, h1, w1).reshape(prob.shape)
    assert near.sum().item() == 0                                # so the counts below can be exact
    assert torch.equal(prob.cpu(), ref["prob"].cpu())
    _close(gd, ref["gd"])
    assert torch.equal(res.pair_count.cpu(), ref["pair_count"].cpu())
    _close(res.pair_sum, ref["pair_sum"], 1e-12)
    _close(res.epe, ref["epe"], 1e-12)
    # the scalars are what torch computes from the device outputs, bit for bit
    vec = gd[prob == 1]
    for p, t in zip((pck_1, pck_3, pck_5), (1.0, 3.0, 5.0)):
        assert _bits(p, (vec < t).float().mean())
    _close(res.epe, vec.mean(), 1e-13)
    assert torch.equal(res.pair_count[:, 0], (prob == 1).sum(dim=(1, 2)))


@pytest.mark.parametrize("ddtype", [torch.float32, torch.float64])
def test_dense_geometric_dist_at_harness_size(big, ddtype):
    views = [big[0][0].to(ddtype), big[0][1].to(ddtype), *big[0][2:]]
    dm = _noisy_warp(views, 3)
    with torch.cuda.device(0):
        cviews, cdm = _cuda(views), dm.to(DEV)
        torch.cuda.set_sync_debug_mode("error")
        try:
            res = dense_geometric_dist(*cviews, cdm)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    d = {}
    ref = oracle.dense_geometric_dist(*views, dm, details=d)
    _check_dense(res, ref, d, 384, 512)
    assert 0.2 < res.pck_1.item() < 0.99 and res.pck_1 <= res.pck_3 <= res.pck_5 and 0.05 < res.epe.item() < 5
    again = dense_geometric_dist(*cviews, cdm)
    for a, b in zip((*res, res.epe, res.pair_sum, res.pair_count), (*again, again.epe, again.pair_sum, again.pair_count)):
        assert _bits(a, b)
    # the left half of a symmetric warp, read in place
    sym = torch.cat((cdm, torch.rand_like(cdm)), dim=2)
    half = dense_geometric_dist(*cviews, sym[:, :, :512])
    for a, b in zip((*res, res.epe, res.pair_sum, res.pair_count), (*half, half.epe, half.pair_sum, half.pair_count)):
        assert _bits(a, b)


def test_dense_geometric_dist_unequal_sizes_and_pairs_without_valid_pixels():
    views = synthetic.depth_scene(12, 3, 60, 80, 48, 64)
    dm = _noisy_warp(views, 4)[:, 5:45, 8:72]                    # the warp's size differs from both depth maps; a strided view
    views[0][1] = 0
    d = {}
    res = dense_geometric_dist(*_cuda(views), dm.to(DEV))
    _check_dense(res, oracle.dense_geometric_dist(*views, dm, details=d), d, 48, 64)
    assert res.pair_count[1].tolist() == [0, 0, 0, 0] and res.pair_sum[1].item() == 0 and res.pair_count[0, 0].item() > 0
    views[0][:] = 0
    res = dense_geometric_dist(*_cuda(views), dm.to(DEV))
    ref = oracle.dense_geometric_dist(*views, dm)
    assert all(torch.isnan(x).all() for x in (res.gd, res.pck_1, res.pck_3, res.pck_5, res.epe))
    assert torch.isnan(ref["pck"]).all() and torch.isnan(ref["epe"]) and not res.prob.any() and not res.pair_count.any()


def test_dense_geometric_dist_after_tiny_match():
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    model = tiny_roma_v1_outdoor(DEV, weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    views = synthetic.depth_scene(31, 4, 96, 128)
    g = torch.Generator().manual_seed(5)
    a, b = torch.rand(4, 3, 96, 128, generator=g).to(DEV), torch.rand(4, 3, 96, 128, generator=g).to(DEV)
    cviews = _cuda(views)
    warp, _ = model.match(a, b)
    assert warp.shape == (4, 96, 128, 4)
    with torch.cuda.device(0):
        torch.cuda.set_sync_debug_mode("error")
        try:
            res = dense_geometric_dist(*cviews, warp)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    d = {}
    ref = oracle.dense_geometric_dist(*views, warp.cpu(), details=d)
    _check_dense(res, ref, d, 96, 128)
    assert all(torch.isfinite(x).all() for x in (res.pck_1, res.pck_3, res.pck_5, res.epe, res.pair_sum)) and res.pair_count[:, 0].min() > 0


def test_dense_geometric_dist_in_a_cuda_graph():
    views = _cuda(synthetic.depth_scene(40, 2, 96, 128))
    dm = _noisy_warp([v.cpu() for v in views], 6).to(DEV)
    keys = ("gd", "pck_1", "pck_3", "pck_5", "prob", "epe", "pair_sum", "pair_count")
    eager = dense_geometric_dist(*views, dm)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        dense_geometric_dist(*views, dm)
    torch.cuda.current_stream().wait_stream(side)
    launches = cabi.kernel_launches()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = dense_geometric_dist(*views, dm)
    assert cabi.kernel_launches() - launches == 2
    graph.replay()
    torch.cuda.synchronize()
    for k in keys:
        assert _bits(getattr(out, k), getattr(eager, k)), k
    dm.copy_(_noisy_warp([v.cpu() for v in views], 7))             # new input in the captured buffer
    graph.replay()
    fresh = dense_geometric_dist(*views, dm)
    torch.cuda.synchronize()
    for k in keys:
        assert _bits(getattr(out, k), getattr(fresh, k)), k
    assert not _bits(fresh.gd, eager.gd)


def test_smoke_entry_includes_the_metric():
    import __graft_entry__ as entry
    entry.smoke_depth_warp()
