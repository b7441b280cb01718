"""Dense reconstruction on the host: the numpy oracle on hand-built cases and on synthetic scenes, the argument rules of the public
functions (checked before any device work), the PLY writer, and the scene generator."""
import math

import numpy as np
import pytest
import torch

from oracle import dense as oracle
from roma_b200 import camera, dense, synthetic
from roma_b200.dense import DenseCloud, fuse_depth_maps, triangulate_warps, write_ply

SIZE = 100.0


def _rig(z_pairs=None):
    """Two cameras f = 100 on a 100 x 100 image, R = I, camera 1 one unit along +x: the camera table, image sizes, and the pinhole
    parts."""
    K = np.array([[[100.0, 0, 50], [0, 100.0, 50], [0, 0, 1]]] * 2)
    R = np.stack([np.eye(3)] * 2)
    t = np.array([[0.0, 0, 0], [-1.0, 0, 0]])
    return dense.camera_table(K, R, t), np.array([[100, 100], [100, 100]]), K, R, t


def _warp_row(W, depths, dy_px=0.0):
    """A [1, 1, 2W, 4] symmetric warp on a 1 x W grid of the rig: grid pixel c of image 0 (centre x = 100 (c + 0.5) / W) seen at
    depth depths[c] (its match in image 1 shifted by 100 / z px, and by dy_px vertically), and the same in the right half from
    image 1 (match shifted by +100 / z)."""
    warp = np.zeros((1, 1, 2 * W, 4), np.float32)
    for c in range(W):
        x, z = SIZE * (c + 0.5) / W, depths[c]
        gx = 2 * x / SIZE - 1
        warp[0, 0, c] = (gx, 0.0, 2 * (x - 100 / z) / SIZE - 1, 2 * dy_px / SIZE)
        warp[0, 0, W + c] = (2 * (x + 100 / z) / SIZE - 1, 2 * dy_px / SIZE, gx, 0.0)
    return warp


def _run(warp, cert, registered=(True, True), pairs=((0, 1),), **kw):
    table, sizes, *_ = _rig()
    return oracle.triangulate_warps(np.array(pairs), warp, cert, sizes, table, np.array(registered), **kw)


def test_reasons_in_order_and_at_thresholds():
    W = 8
    # grid x = 6.25 + 12.5 c; z = 10 everywhere except a far point (angle) and a point behind the cameras
    depths = [10.0] * W
    depths[5] = 1000.0          # 0.057 degrees: rule 7
    depths[6] = -10.0           # behind both cameras: rule 5
    warp = _warp_row(W, depths)
    cert = np.full((1, 1, 2 * W), 0.9, np.float32)
    cert[0, 0, 0] = np.float32(0.05)                           # exactly min_certainty: rejected (<=)
    cert[0, 0, 1] = np.nextafter(np.float32(0.05), np.float32(1))
    cert[0, 0, 2] = np.nan
    warp[0, 0, 3, 2] = np.nextafter(np.float32(1), np.float32(2))    # just outside [-1, 1]
    warp[0, 0, 4, 3] = np.float32(0.4)                         # 20 px off the epipolar line: rule 6
    maps, el = _run(warp, cert)
    r = el[(0, 0)]["reason"][0]
    assert r.tolist() == [1, 0, 1, 2, 6, 7, 5, 0]
    np.testing.assert_allclose(el[(0, 0)]["depth"][0, [1, 7]], 10.0, rtol=1e-6)     # the warp is fp32
    assert maps["pair_counts"][0].tolist() == np.bincount(np.r_[r, el[(0, 1)]["reason"][0]], minlength=8).tolist()
    # u exactly 1 is inside the range
    warp[0, 0, 3, 2] = np.float32(1)
    assert _run(warp, cert)[1][(0, 0)]["reason"][0, 3] != oracle.RANGE
    # max_error exactly at the reprojection error of element 4 keeps it (the test is error^2 <= max_error^2)
    e = math.sqrt(max(el[(0, 0)]["eg"][0, 4], el[(0, 0)]["em"][0, 4]))
    assert _run(warp, cert, max_error=e * (1 + 1e-12))[1][(0, 0)]["reason"][0, 4] != oracle.REPROJ
    assert _run(warp, cert, max_error=e * (1 - 1e-12))[1][(0, 0)]["reason"][0, 4] == oracle.REPROJ


def test_unregistered_image_rejects_every_later_reason():
    W = 4
    warp = _warp_row(W, [10.0] * W)
    cert = np.full((1, 1, 2 * W), 0.9, np.float32)
    cert[0, 0, 0] = 0.01
    maps, el = _run(warp, cert, registered=(True, False))
    assert el[(0, 0)]["reason"][0].tolist() == [1, 3, 3, 3] and (el[(0, 1)]["reason"] == 3).all()
    assert (maps["depth"] == 0).all() and (maps["source"] == -1).all()


def test_certainty_ties_go_to_the_smallest_pair_half():
    W = 4
    warp = np.concatenate([_warp_row(W, [10.0] * W), _warp_row(W, [10.0 + 1e-3] * W)])
    cert = np.full((2, 1, 2 * W), 0.5, np.float32)
    cert[1, 0, 0] = 0.6                     # pair 1 wins pixel 0 of image 0 by certainty
    maps, _ = _run(warp, cert, pairs=((0, 1), (0, 1)))
    assert maps["source"][0, 0].tolist() == [2, 0, 0, 0] and maps["source"][1, 0].tolist() == [1, 1, 1, 1]
    assert maps["score"][0, 0, 0] == np.float32(0.6)
    np.testing.assert_allclose(maps["depth"][0, 0, 1:], 10.0, rtol=1e-6)
    # the same pairs streamed one at a time and in the other order give the same maps
    part, _ = _run(warp[1:], cert[1:], pairs=((0, 1), (0, 1)), first_pair=1)
    both, _ = _run(warp[:1], cert[:1], pairs=((0, 1), (0, 1)), maps=part)
    for k in ("depth", "score", "source", "pair_counts"):
        np.testing.assert_array_equal(both[k], maps[k])


def _fronto(d0, d1, max_depth_error, min_num_views=2):
    """An 8 x 8 grid of the rig on the plane z = 8, where one grid pixel of disparity (12.5 px) maps pixel c of image 0 onto pixel
    c - 1 of image 1 exactly; depth maps d0, d1 as given."""
    table, sizes, *_ = _rig()
    depth = np.stack([np.full((8, 8), d0, np.float32), np.full((8, 8), d1, np.float32)])
    return oracle.fuse_depth_maps(depth, np.ones_like(depth), np.array([[0, 1]]), sizes, table, np.array([True, True]),
                                  max_depth_error=max_depth_error, min_num_views=min_num_views)


def test_emission_when_agreement_is_one_sided():
    # depths 8 and 8.04: the relative depth test is 0.04 / 8 = 0.005 from the view at 8, 0.04 / 8.04 from the view at 8.04
    bar = 0.00499
    both = _fronto(8.0, 8.04, 0.0051)
    assert set(both["image"].tolist()) == {0} and (both["num_views"] == 2).all()      # symmetric: emitted from image 0 only
    low_agrees = _fronto(8.04, 8.0, bar)        # image 0 (8.04) agrees with image 1, image 1 not with image 0
    assert set(low_agrees["image"].tolist()) == {0} and len(low_agrees["image"]) == len(both["image"])
    high_agrees = _fronto(8.0, 8.04, bar)       # only image 1 agrees, and its agreeing neighbour 0 has the smaller index
    assert len(high_agrees["image"]) == 0
    assert len(_fronto(8.0, 8.04, 0.0051, min_num_views=3)["image"]) == 0


def test_fusion_points_and_colours():
    table, sizes, *_ = _rig()
    depth = np.stack([np.full((8, 8), 8.0, np.float32)] * 2)
    colors = [np.arange(16 * 24 * 3, dtype=np.uint8).reshape(16, 24, 3), np.zeros((5, 5, 3), np.uint8)]
    out = oracle.fuse_depth_maps(depth, np.ones_like(depth), np.array([[0, 1]]), sizes, table, np.array([True, True]), colors=colors,
                                 min_num_views=2)
    r, c = np.divmod(out["pixel"], 8)
    assert (c >= 1).all() and len(out["pixel"]) == 8 * 7
    np.testing.assert_allclose(out["points"][:, 2], 8.0, rtol=1e-12)
    np.testing.assert_array_equal(out["colors"], colors[0][(2 * r + 1) * 16 // 16, (2 * c + 1) * 24 // 16])


def _scene_warps(views, pairs):
    """Ground-truth warps of pinhole depth_views in numpy (the radial rule with k = 0 is the pinhole one)."""
    N, H, W = views["depth"].shape
    v = dict(views, intrinsics=torch.cat((views["K"][:, 0, 0:1], views["K"][:, 0, 2:3], views["K"][:, 1, 2:3], torch.zeros(N, 1)), 1))
    warps, certs = [], []
    for i, j in pairs:
        halves = []
        for a, b in ((i, j), (j, i)):
            R, t = views["R"], views["t"]
            Rr = R[b] @ R[a].T
            T = torch.eye(4, dtype=torch.float64)[None].clone()
            T[0, :3, :3], T[0, :3, 3] = Rr, t[b] - Rr @ t[a]
            x2, prob = synthetic._radial_gt_warp(v, torch.tensor([a]), torch.tensor([b]), T, H, W)
            gy, gx = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n) for n in (H, W))
            grid = torch.stack(torch.meshgrid(gy, gx, indexing="ij")[::-1], -1)
            halves.append((grid, x2[0], prob[0]))
        (g0, m0, p0), (g1, m1, p1) = halves
        warps.append(torch.cat((torch.cat((g0, m0), -1), torch.cat((m1, g1), -1)), 1))
        certs.append(torch.cat((p0, p1), 1))
    return torch.stack(warps).numpy(), torch.stack(certs).numpy()


def test_oracle_recovers_depth_views_depth():
    views = synthetic.depth_views(3, 3, (48, 64))
    views["K"][:, 1, 1] = views["K"][:, 0, 0]          # square pixels, the pinhole K of (f, cx, cy, 0)
    pairs = [(0, 1), (1, 2), (0, 2)]
    warp, cert = _scene_warps(views, pairs)
    table = dense.camera_table(views["K"].numpy(), views["R"].numpy(), views["t"].numpy())
    maps, el = oracle.triangulate_warps(np.array(pairs), warp, cert, views["image_sizes"].numpy(), table, np.ones(3, bool))
    ok = maps["depth"] > 0
    assert ok.mean() > 0.5
    gt = views["depth"].numpy()
    rel = np.abs(maps["depth"][ok] - gt[ok]) / gt[ok]
    assert rel.max() < 1e-4, rel.max()


def test_generator_views_agree():
    views = synthetic.depth_views(0, 4, (48, 64))
    d, K, R, t = (views[k].numpy() for k in ("depth", "K", "R", "t"))
    H, W = d.shape[1:]
    ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    rays = np.stack((xs, ys, np.ones_like(xs)), -1) @ np.linalg.inv(K[0]).T
    X = ((rays * d[0][..., None]) - t[0]) @ R[0]                    # world points of view 0
    p = (X @ R[1].T + t[1]) @ K[1].T
    u, v = p[..., 0] / p[..., 2], p[..., 1] / p[..., 2]
    inside = (d[0] > 0) & (u >= 0.5) & (u < W - 1.5) & (v >= 0.5) & (v < H - 1.5)
    # bilinear depth of view 1 at (u, v) against the point's depth there, where the four taps are valid and on one surface
    x0, y0 = np.floor(u - 0.5).astype(int), np.floor(v - 0.5).astype(int)
    x0, y0 = np.clip(x0, 0, W - 2), np.clip(y0, 0, H - 2)
    taps = np.stack([d[1][y0 + a, x0 + b] for a in (0, 1) for b in (0, 1)])
    flat = (taps > 0).all(0) & (taps.max(0) - taps.min(0) < 0.05 * taps.max(0))
    fx, fy = u - 0.5 - x0, v - 0.5 - y0
    bil = taps[0] * (1 - fx) * (1 - fy) + taps[1] * fx * (1 - fy) + taps[2] * (1 - fx) * fy + taps[3] * fx * fy
    close = inside & flat & (np.abs(bil - p[..., 2]) < 1e-3 * p[..., 2])
    assert close.sum() > 0.3 * inside.sum()           # the rest is occluded in view 1, lands on a hole or straddles an edge


def test_argument_rules_before_device_work():
    views = synthetic.depth_views(0, 2, (8, 12))
    K, R, t, sizes = views["K"], views["R"], views["t"], views["image_sizes"]
    warp, cert = torch.zeros(1, 8, 24, 4), torch.zeros(1, 8, 24)
    ok = dict(pairs=[(0, 1)], warp=warp, certainty=cert, K=K, R=R, t=t, image_sizes=sizes)

    def bad(match, **change):
        a = dict(ok, **change)
        kw = {k: a.pop(k) for k in ("first_pair", "registered", "intrinsics", "min_certainty", "max_error", "min_angle") if k in a}
        with pytest.raises(ValueError, match=match):
            triangulate_warps(a["pairs"], a["warp"], a["certainty"], a["K"], a["R"], a["t"], a["image_sizes"], **kw)

    bad("image index", pairs=[(0, 2)])
    bad("pairs must be", pairs=[(0, 1, 2)])
    bad("fp32", warp=warp.double())
    bad("symmetric", warp=torch.zeros(1, 8, 23, 4), certainty=torch.zeros(1, 8, 23))
    bad("certainty", certainty=torch.zeros(1, 8, 22))
    bad("do not fit", first_pair=1)
    bad("first_pair", first_pair=-1)
    bad("K must have shape", K=K[:1])
    bad("not finite", R=R * float("nan"))
    bad("K or intrinsics", intrinsics=camera.default_intrinsics(sizes))
    bad("K is required", K=None)
    bad("invertible", K=torch.zeros(2, 3, 3, dtype=torch.float64))
    bad("focal length", K=None, intrinsics=torch.zeros(2, 4, dtype=torch.float64))
    bad("registered", registered=[1, 1])
    bad("min_certainty", min_certainty=-0.1)
    bad("max_error", max_error=0.0)
    bad("min_angle", min_angle=180.0)
    bad("image sizes", image_sizes=torch.zeros(2, 2, dtype=torch.int64))
    bad("image_sizes must hold integers", image_sizes=sizes.double())
    bad("CUDA device")                                 # every argument is valid: the CPU tensors are refused last

    dm = dense.DepthMaps(torch.zeros(2, 8, 12), torch.zeros(2, 8, 12), torch.zeros(2, 8, 12, dtype=torch.int64), torch.zeros(1, 8))
    for match, kw in (("min_num_views", dict(min_num_views=0)), ("max_reproj_error", dict(max_reproj_error=-1.0)),
                      ("max_depth_error", dict(max_depth_error=float("inf"))), ("colors must hold", dict(colors=[])),
                      ("CUDA device", {})):
        with pytest.raises(ValueError, match=match):
            fuse_depth_maps(dm, [(0, 1)], K, R, t, sizes, **kw)
    with pytest.raises(ValueError, match="DepthMaps"):
        fuse_depth_maps(dm.depth, [(0, 1)], K, R, t, sizes)
    with pytest.raises(ValueError, match="unknown options"):
        dense.check_cameras("dense_cloud", [(0, 1)], K, R, t, sizes, min_views=2)


def test_ply_round_trip(tmp_path):
    g = torch.Generator().manual_seed(0)
    cloud = DenseCloud(torch.randn(5, 3, generator=g, dtype=torch.float64), torch.randint(0, 256, (5, 3), generator=g, dtype=torch.uint8),
                       torch.zeros(5, dtype=torch.int32), torch.arange(5), torch.full((5,), 3, dtype=torch.int32), torch.ones(5))
    path = tmp_path / "cloud.ply"
    write_ply(path, cloud)
    data = path.read_bytes()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    header = data[:end].decode("ascii").splitlines()
    assert header[:3] == ["ply", "format binary_little_endian 1.0", "element vertex 5"]
    assert header[3:9] == [f"property {t} {n}" for t, n in (("float", "x"), ("float", "y"), ("float", "z"), ("uchar", "red"),
                                                            ("uchar", "green"), ("uchar", "blue"))]
    v = np.frombuffer(data[end:], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("r", "u1"), ("g", "u1"), ("b", "u1")])
    assert len(v) == 5
    np.testing.assert_array_equal(np.stack((v["x"], v["y"], v["z"]), 1), cloud.points.numpy().astype(np.float32))
    np.testing.assert_array_equal(np.stack((v["r"], v["g"], v["b"]), 1), cloud.colors.numpy())
