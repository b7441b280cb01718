"""Dense reconstruction on the GPU: `triangulate_warps` inverts the depth-based ground-truth warp (`get_gt_warp`) on synthetic scenes,
agrees with the numpy oracle (oracle/dense.py) element by element wherever a decision is clear of its threshold, rejects each kind
of bad element with its reason, and gives byte-identical maps for any chunking and order of the pairs; `fuse_depth_maps` emits the
oracle's points, on the planted surfaces, with the colours of the nearest pixels; SIMPLE_RADIAL cameras; and `dense_cloud` equals
the hand-written match_pairs -> triangulate_warps -> fuse_depth_maps loop."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import dense as oracle  # noqa: E402
from roma_b200 import dense, roma_outdoor, synthetic  # noqa: E402
from roma_b200.dense import fuse_depth_maps, triangulate_warps  # noqa: E402

DEV = "cuda"


def _exhaustive(N):
    return [(i, j) for i in range(N) for j in range(i + 1, N)]


def _cams(v):
    return v["K"], v["R"], v["t"], v["image_sizes"]


def _bits(x):
    return x.contiguous().view(torch.uint8) if x.dtype.is_floating_point else x


def _equal(a, b):
    return all(torch.equal(_bits(getattr(a, k)), _bits(getattr(b, k))) for k in ("depth", "score", "source", "pair_counts"))


@pytest.fixture(scope="module")
def scene():
    views = synthetic.depth_views(1, 6, (96, 128))
    pairs = _exhaustive(6)
    warp, cert = synthetic.depth_view_warps(views, pairs, DEV)
    return views, pairs, warp, cert


def test_round_trip_recovers_the_planted_depth(scene):
    views, pairs, warp, cert = scene
    dm = triangulate_warps(pairs, warp, cert, *_cams(views))
    gt = views["depth"].to(DEV)
    got = dm.depth > 0
    assert got.float().mean() > 0.6 and (gt[got] > 0).all()
    rel = ((dm.depth[got].double() - gt[got].double()).abs() / gt[got].double())
    print(f"round trip: {int(got.sum())} pixels, relative depth error max {rel.max().item():.2e} median {rel.median().item():.2e}")
    assert rel.max().item() < 1e-4
    # the winners are certainty-1 elements, ties to the smallest 2 k + half
    assert (dm.score[got] == 1).all() and (dm.source[~got] == -1).all()
    assert int(dm.pair_counts.sum()) == cert.numel()


def _noisy(scene, seed):
    """The scene's warps with fp32 noise of a few px on a quarter of the elements, some certainties lowered and some matches pushed
    out of range, so that every reason but 3 and 4 occurs."""
    views, pairs, warp, cert = scene
    g = torch.Generator(device=DEV).manual_seed(seed)
    w, c = warp.clone(), cert.clone()
    pick = torch.rand(c.shape, generator=g, device=DEV) < 0.25
    half = w.shape[2] // 2
    side = torch.zeros_like(w[..., :1], dtype=torch.bool).expand_as(w).clone()
    side[:, :, :half, 2:4], side[:, :, half:, 0:2] = True, True
    noise = torch.randn(w.shape, generator=g, device=DEV) * (6.0 / 128)
    w = torch.where(pick[..., None] & side, w + noise, w)
    c = torch.where(torch.rand(c.shape, generator=g, device=DEV) < 0.1, c * 0.04, c)
    c = torch.where(c > 0, c * (0.5 + 0.5 * torch.rand(c.shape, generator=g, device=DEV)), c)
    return w, c


def test_against_the_oracle(scene):
    views, pairs, _, _ = scene
    warp, cert = _noisy(scene, 0)
    reg = np.ones(6, bool)
    reg[5] = False
    dm = triangulate_warps(pairs, warp, cert, *_cams(views), registered=torch.from_numpy(reg))
    K, R, t, sizes = (x.numpy() for x in _cams(views))
    table = dense.camera_table(K, R, t)
    maps, el = oracle.triangulate_warps(np.array(pairs), warp.cpu().numpy(), cert.cpu().numpy(), sizes, table, reg)
    # every decision of the oracle must be clear of its threshold by 1e-9 relative for the counts to be compared exactly
    unclear = 0
    for e in el.values():
        live = (e["reason"] == 0) | (e["reason"] >= oracle.REPROJ)
        err = np.maximum(e["eg"], e["em"])
        unclear += int((live & (np.abs(err - 16.0) <= 16.0 * 1e-9)).sum())
        live_a = e["reason"] == 0
        unclear += int((live_a & (np.abs(e["angle"] - math.radians(1.5)) <= math.radians(1.5) * 1e-9)).sum())
    assert unclear == 0
    counts = dm.pair_counts.cpu().numpy()
    np.testing.assert_array_equal(counts, maps["pair_counts"])
    assert (counts[:, [0, 1, 2, 3, 6]] > 0).any(0).all(), counts.sum(0)
    np.testing.assert_array_equal(dm.source.cpu().numpy(), maps["source"])
    np.testing.assert_array_equal(dm.score.cpu().numpy(), maps["score"])
    d, want = dm.depth.cpu().numpy(), maps["depth"]
    ulp = np.abs(d.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    print(f"oracle: worst depth difference {ulp.max()} float32 ulp over {(want > 0).sum()} pixels")
    assert ulp.max() <= 2


def _rig_warp(W, depths, dy_px=0.0):
    """The host test's rig (tests/test_dense_host.py): cameras f = 100 on 100 x 100 images, camera 1 one unit along +x."""
    warp = np.zeros((1, 1, 2 * W, 4), np.float32)
    for c in range(W):
        x, z = 100.0 * (c + 0.5) / W, depths[c]
        gx = 2 * x / 100 - 1
        warp[0, 0, c] = (gx, 0.0, 2 * (x - 100 / z) / 100 - 1, 2 * dy_px / 100)
        warp[0, 0, W + c] = (2 * (x + 100 / z) / 100 - 1, 2 * dy_px / 100, gx, 0.0)
    return torch.from_numpy(warp).to(DEV)


RIG = dict(K=torch.tensor([[[100.0, 0, 50], [0, 100.0, 50], [0, 0, 1]]] * 2, dtype=torch.float64),
           R=torch.eye(3, dtype=torch.float64).expand(2, 3, 3), t=torch.tensor([[0.0, 0, 0], [-1.0, 0, 0]], dtype=torch.float64),
           image_sizes=[(100, 100), (100, 100)])


@pytest.mark.parametrize("case", ["certainty", "range", "unregistered", "behind", "epipolar"])
def test_filters_reject_with_their_reason(case):
    W = 16
    depths = [-20.0] * W if case == "behind" else [20.0] * W      # 5 px of disparity: one edge element per half leaves the image
    warp = _rig_warp(W, depths, dy_px=0.0)
    cert = torch.full((1, 1, 2 * W), 0.9, device=DEV)
    kw = {}
    if case == "certainty":
        cert[:] = 0.05
    elif case == "range":
        warp[0, 0, :W, 2] = 1.0 + 2 ** -20
        warp[0, 0, W:, 0] = -1.0 - 2 ** -20
    elif case == "unregistered":
        kw["registered"] = torch.tensor([True, False])
    elif case == "epipolar":
        dy = torch.linspace(20, 50, W, device=DEV).repeat(2)       # 20-50 px across the (horizontal) epipolar lines
        warp[0, 0, :W, 3] = 2 * dy[:W] / 100
        warp[0, 0, W:, 1] = 2 * dy[W:] / 100
    reason = {"certainty": 1, "range": 2, "unregistered": 3, "behind": 5, "epipolar": 6}[case]
    dm = triangulate_warps([(0, 1)], warp, cert, RIG["K"], RIG["R"], RIG["t"], RIG["image_sizes"], **kw)
    want = [0] * 8
    want[reason] = 2 * W
    if reason > 2:
        want[reason], want[2] = 2 * W - 2, 2
    assert dm.pair_counts[0].tolist() == want
    assert (dm.depth == 0).all() and (dm.source == -1).all()
    ok = triangulate_warps([(0, 1)], _rig_warp(W, [20.0] * W), torch.full((1, 1, 2 * W), 0.9, device=DEV), RIG["K"], RIG["R"], RIG["t"],
                           RIG["image_sizes"])
    assert ok.pair_counts[0].tolist() == [2 * W - 2, 0, 2, 0, 0, 0, 0, 0]
    assert ((ok.depth[ok.depth > 0] - 20).abs() <= 2e-5).all()


def test_streaming_is_exact(scene):
    views, pairs, _, _ = scene
    warp, cert = _noisy(scene, 1)
    cams = _cams(views)
    whole = triangulate_warps(pairs, warp, cert, *cams)
    P = len(pairs)
    for chunk in (1, 3, P):
        dm = None
        for k0 in range(0, P, chunk):
            dm = triangulate_warps(pairs, warp[k0:k0 + chunk], cert[k0:k0 + chunk], *cams, first_pair=k0, depth_maps=dm)
        assert _equal(dm, whole), chunk
    order = torch.randperm(P, generator=torch.Generator().manual_seed(0)).tolist()
    dm = None
    for k in order:
        dm = triangulate_warps(pairs, warp[k:k + 1], cert[k:k + 1], *cams, first_pair=k, depth_maps=dm)
    assert _equal(dm, whole)
    assert _equal(triangulate_warps(pairs, warp, cert, *cams), whole)
    assert int((whole.source >= 0).sum()) > 0.5 * whole.source.numel()


def test_fusion_against_the_oracle_and_the_planted_surface(scene):
    views, pairs, warp, cert = scene
    cams = _cams(views)
    colors = [views["colors"][i].to(DEV) for i in range(6)]
    dm = triangulate_warps(pairs, warp, cert, *cams)
    cloud = fuse_depth_maps(dm, pairs, *cams, colors=colors)
    K, R, t, sizes = (x.numpy() for x in cams)
    table = dense.camera_table(K, R, t)
    margins = []
    ref = oracle.fuse_depth_maps(dm.depth.cpu().numpy(), dm.score.cpu().numpy(), np.array(pairs), sizes, table, np.ones(6, bool),
                                 colors=[c.numpy() for c in views["colors"]], margins=margins)
    M = cloud.points.shape[0]
    assert M > 1000
    key = lambda img, pix: set(zip(img.tolist(), pix.tolist()))     # noqa: E731
    got, want = key(cloud.image.cpu(), cloud.pixel.cpu()), key(ref["image"], ref["pixel"])
    unclear = {(i, p) for i, p in got ^ want if margins[i].reshape(-1)[p] <= 1e-9}
    assert got ^ want == unclear
    if not unclear:
        np.testing.assert_allclose(cloud.points.cpu().numpy(), ref["points"], rtol=0, atol=1e-9)
        np.testing.assert_array_equal(cloud.colors.cpu().numpy(), ref["colors"])
        np.testing.assert_array_equal(cloud.num_views.cpu().numpy(), ref["num_views"])
        np.testing.assert_array_equal(cloud.score.cpu().numpy(), ref["score"])
    # every point lies on the planted surface seen by its pixel: depth in its view within max_depth_error of the planted depth
    img, pix = cloud.image.long().cpu(), cloud.pixel.cpu()
    X = cloud.points.cpu()
    z = (torch.einsum("mij,mj->mi", views["R"][img], X) + views["t"][img])[:, 2]
    gt = views["depth"].reshape(6, -1)[img, pix].double()
    rel = (z - gt).abs() / gt
    zr = (np.einsum("mij,mj->mi", R[ref["image"]], ref["points"]) + t[ref["image"]])[:, 2]
    rel_ref = np.abs(zr - views["depth"].numpy().reshape(6, -1)[ref["image"], ref["pixel"]]) / zr
    print(f"fusion: {M} points, relative depth error max {rel.max().item():.2e} median {rel.median().item():.2e} "
          f"(oracle median {np.median(rel_ref):.2e})")
    assert rel.max().item() <= 0.01 and rel.median().item() <= 1.01 * np.median(rel_ref) + 1e-12
    assert (cloud.num_views >= 3).all()
    # colours: the nearest pixel of the view's colour image
    H, W = 96, 128
    r, c = pix // W, pix % W
    np.testing.assert_array_equal(cloud.colors.cpu().numpy(), views["colors"][img, r, c].numpy())
    # reruns are byte-identical
    again = fuse_depth_maps(dm, pairs, *cams, colors=colors)
    for name in ("points", "colors", "image", "pixel", "num_views", "score"):
        assert torch.equal(_bits(getattr(again, name)), _bits(getattr(cloud, name))), name


def test_matches_along_the_epipolar_line_are_triangulated_but_not_fused(scene):
    views, pairs, warp, cert = scene
    cams = _cams(views)
    # pair (0, 1)'s left half from view 0's depth scaled by 1.03: every match moves along its epipolar line
    moved = dict(views, depth=views["depth"].clone())
    moved["depth"][0] *= 1.03
    w01, c01 = synthetic.depth_view_warps(moved, [(0, 1)], DEV)
    W = warp.shape[2] // 2
    warp, cert = warp.clone(), cert.clone() * 0.9
    warp[0, :, :W], cert[0, :, :W] = w01[0, :, :W], c01[0, :, :W]          # the moved half wins view 0 by certainty
    dm = triangulate_warps(pairs, warp, cert, *cams)
    won = dm.source[0] == 0
    gt = views["depth"][0].to(DEV)
    assert won.sum() > 1000
    np.testing.assert_allclose((dm.depth[0][won] / gt[won]).cpu().numpy(), 1.03, rtol=1e-4)
    cloud = fuse_depth_maps(dm, pairs, *cams)
    bad = won.reshape(-1)[cloud.pixel[cloud.image == 0]]
    # a moved point can still land, in two neighbours, on a surface 3 % away (at an occluding edge): 8 of the 8121 moved pixels
    # on an H100; the bar leaves room for a few more
    print(f"moved pixels {int(won.sum())}, emitted {int(bad.sum())}")
    assert int(bad.sum()) <= 0.01 * int(won.sum()) and int((cloud.image == 0).sum()) > 0


def test_simple_radial_scene():
    views = synthetic.depth_views(2, 4, (96, 128), radial=(-0.08, 0.06))
    pairs = _exhaustive(4)
    warp, cert = synthetic.depth_view_warps(views, pairs, DEV)
    dm = triangulate_warps(pairs, warp, cert, None, views["R"], views["t"], views["image_sizes"], intrinsics=views["intrinsics"])
    gt = views["depth"].to(DEV)
    got = dm.depth > 0
    rel = (dm.depth[got].double() - gt[got].double()).abs() / gt[got].double()
    print(f"SIMPLE_RADIAL: {int(got.sum())} pixels, relative depth error max {rel.max().item():.2e} median {rel.median().item():.2e}")
    assert got.float().mean() > 0.5 and rel.max().item() < 1e-4 and rel.median().item() < 1e-6
    # the oracle's radial rule on the same warps
    table = dense.camera_table(None, views["R"].numpy(), views["t"].numpy(), views["intrinsics"].numpy())
    maps, _ = oracle.triangulate_warps(np.array(pairs), warp.cpu().numpy(), cert.cpu().numpy(), views["image_sizes"].numpy(), table,
                                       np.ones(4, bool), radial=1)
    np.testing.assert_array_equal(dm.source.cpu().numpy(), maps["source"])
    cloud = fuse_depth_maps(dm, pairs, None, views["R"], views["t"], views["image_sizes"], intrinsics=views["intrinsics"],
                            min_num_views=2)
    assert cloud.points.shape[0] > 1000


def test_dense_cloud_equals_the_hand_loop(weights):
    model = roma_outdoor(DEV, weights=weights[0], dinov2_weights=weights[1], coarse_res=112, upsample_res=168, amp_dtype=torch.float16)
    ims = [im for s in (3, 4) for im in synthetic.make_pil_pair(s)]
    sizes = [im.size[::-1] for im in ims]
    views = synthetic.depth_views(4, 4, (96, 128))
    K, R, t = views["K"], views["R"], views["t"]
    pairs = _exhaustive(4)
    opts = dict(min_certainty=0.0, max_error=1e3, min_angle=0.0, max_reproj_error=1e3, max_depth_error=10.0, min_num_views=2)
    torch.cuda.synchronize()
    model.match_pairs(ims, pairs, max_batch=2)           # encodes the bank, so the peaks below compare the pair stage only
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    warp, cert = model.match_pairs(ims, pairs, max_batch=2)
    dense_peak = torch.cuda.max_memory_allocated() - base
    del warp, cert
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    got = model.dense_cloud(ims, pairs, K, R, t, max_batch=2, **opts)
    cloud_peak = torch.cuda.max_memory_allocated() - base
    print(f"dense_cloud peak {cloud_peak / 2**20:.1f} MiB, match_pairs without on_batch {dense_peak / 2**20:.1f} MiB")
    assert cloud_peak < dense_peak
    state = {}

    def on_batch(k0, w, c):
        state["dm"] = triangulate_warps(pairs, w, c, K, R, t, sizes, first_pair=k0, depth_maps=state.get("dm"), min_certainty=0.0,
                                        max_error=1e3, min_angle=0.0)

    model.match_pairs(ims, pairs, max_batch=2, on_batch=on_batch)
    want = fuse_depth_maps(state["dm"], pairs, K, R, t, sizes, max_reproj_error=1e3, max_depth_error=10.0, min_num_views=2)
    assert got.points.shape[0] > 0
    for name in ("points", "colors", "image", "pixel", "num_views", "score"):
        assert torch.equal(_bits(getattr(got, name)), _bits(getattr(want, name))), name
