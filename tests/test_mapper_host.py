"""CPU tests of the reconstruction driver (`roma_b200.mapper`): the library's new export and struct field, the ranking of the candidate
pairs and the argument checks (each ValueError before any device work), the numpy statement of the two-view statistics
(oracle/mapper.py) against cv2 and numpy, and the COLMAP text writer on a hand-built reconstruction, parsed back."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import mapper as om
from roma_b200 import MatchGraph, Points3D, Tracks, cabi, mapper, synthetic


def test_library_exports_the_two_view_score_and_the_pair_list():
    lib = cabi.load_library()
    assert "romab200_twoview_score" in cabi.FUNCTIONS and hasattr(lib, "romab200_twoview_score")
    fields = cabi.STRUCT_FIELDS["rb_verify_args"]
    assert fields[-1] == ("pair_list", ctypes.c_void_p)          # appended: every earlier field keeps its offset
    assert ctypes.sizeof(cabi.STRUCTS["rb_verify_args"]) == cabi.STRUCTS["rb_verify_args"].pair_list.offset + 8


def test_ranking_ties_and_bounds():
    off = np.concatenate([[0], np.cumsum([5, 120, 100, 120, 99, 300, 100])])
    assert mapper.rank_candidates(off, 100, 256) == [5, 1, 3, 2, 6]           # count descending, then pair index ascending
    assert mapper.rank_candidates(off, 100, 2) == [5, 1]
    assert mapper.rank_candidates(off, 301, 256) == []
    assert mapper.rank_candidates(off, 0, 256) == [5, 1, 3, 2, 6, 4, 0]
    for n in (1, 3, 7):
        assert om.rank(off, 100, n) == mapper.rank_candidates(off, 100, n)


def _cpu_graph():
    kp = torch.zeros(6, 2)
    return MatchGraph(torch.tensor([0, 3, 6]), kp, torch.ones(6), torch.tensor([0, 3]), torch.tensor([[0, 0], [1, 1], [2, 2]], dtype=torch.int32),
                      torch.ones(3))


@pytest.mark.parametrize("kw, msg", [(dict(num_candidates=0), "num_candidates"), (dict(num_candidates=4097), "num_candidates"),
                                     (dict(num_candidates=True), "num_candidates"), (dict(min_num_inliers=-1), "min_num_inliers"),
                                     (dict(max_error=0.0), "max_error"), (dict(max_error=float("nan")), "max_error"),
                                     (dict(min_tri_angle=180.0), "min_tri_angle"), (dict(max_forward_motion=-0.1), "max_forward_motion"),
                                     (dict(confidence=1.0), "confidence"), (dict(max_iters=0), "max_iters"), (dict(seed=-1), "seed"),
                                     (dict(), "CUDA device")])
def test_arguments_are_checked_before_device_work(monkeypatch, kw, msg):
    def no_device(*a, **k):
        raise AssertionError("device work before the argument checks")

    monkeypatch.setattr(cabi, "call", no_device)
    g = _cpu_graph()
    K = np.tile(np.eye(3), (2, 1, 1))
    with pytest.raises(ValueError, match=msg):
        mapper.initialize_reconstruction([(0, 1)], g, K, **kw)
    tr = Tracks(torch.tensor([0]), torch.zeros(0, 2, dtype=torch.int32), torch.full((6,), -1, dtype=torch.int32), 0)
    rkw = {("init_" + k if k in ("num_candidates", "min_num_inliers", "max_error", "min_tri_angle", "max_forward_motion") else k): v
           for k, v in kw.items() if k not in ("confidence", "max_iters")}
    if rkw or not kw:
        with pytest.raises(ValueError):
            mapper.reconstruct([(0, 1)], g, tr, K, **rkw)
    for bad in (dict(abs_max_error=0.0), dict(abs_min_inliers=-1), dict(ba_loss_scale=0.0), dict(ba_max_iterations=-1),
                dict(workspace_bytes=0)):
        with pytest.raises(ValueError, match=next(iter(bad))):
            mapper.reconstruct([(0, 1)], g, tr, K, **bad)


def test_oracle_score_against_cv2_and_numpy():
    cv2 = pytest.importorskip("cv2")
    s = synthetic.two_view_scene(3, 400, 0.0)
    R, t = s["R"], s["t"]
    x0, x1 = s["kpts0"], s["kpts1"]
    mask = np.ones(len(x0), bool)
    mask[::7] = False
    res = om.score(x0, x1, s["K0"], s["K1"], R, t, mask, 4.0)
    # rule 1 against cv2.triangulatePoints on the normalised points
    xn0 = cv2.undistortPoints(x0.reshape(-1, 1, 2), s["K0"], None).reshape(-1, 2)
    xn1 = cv2.undistortPoints(x1.reshape(-1, 1, 2), s["K1"], None).reshape(-1, 2)
    Q = cv2.triangulatePoints(np.eye(3, 4), np.c_[R, t], xn0.T, xn1.T)
    Xcv = (Q[:3] / Q[3]).T
    m = np.flatnonzero(mask)
    assert np.abs(res["X"][m] - Xcv[m]).max() <= 1e-9 * max(1.0, np.abs(Xcv[m]).max())
    assert np.isnan(res["X"][~mask]).all() and not res["good"][~mask].any()
    # rule 3 against a direct arccos where the angle is above 1 degree
    C1 = -R.T @ t
    a, b = res["X"][m], res["X"][m] - C1
    direct = np.degrees(np.arccos(np.clip((a * b).sum(1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1), -1, 1)))
    g = res["good"][m]
    big = g & (direct > 1.0)
    assert big.sum() > 100 and np.abs(res["angle"][m][big] - direct[big]).max() <= 1e-9
    # rule 4: the median of the good angles, the mean of the middle two for an even count
    ang = np.sort(res["angle"][res["good"]])
    n = ang.size
    assert res["num_good"] == n and n > 300
    assert res["median_angle"] == np.median(ang) == ((ang[n // 2 - 1] + ang[n // 2]) / 2 if n % 2 == 0 else ang[n // 2])
    assert res["forward"] == abs(t[2])
    even = om.score(x0[:4], x1[:4], s["K0"], s["K1"], R, t, np.ones(4, bool), 4.0)
    assert even["num_good"] == 4 and even["median_angle"] == np.median(np.sort(even["angle"])[1:3])
    assert om.score(x0, x1, s["K0"], s["K1"], R, t, np.zeros(len(x0), bool), 4.0)["median_angle"] == 0.0


def _quat_to_R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_shepperd_quaternions():
    rng = np.random.default_rng(0)
    Rs = [synthetic._scene_rotation(rng, 0.0, 179.9) for _ in range(200)]
    Rs += [np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])]     # each branch of the method
    q = mapper.rotation_to_quaternion(np.stack(Rs))
    assert (q[:, 0] >= 0).all() and np.abs(np.linalg.norm(q, axis=1) - 1).max() < 1e-15
    for R, qq in zip(Rs, q):
        assert np.abs(_quat_to_R(qq) - R).max() <= 1e-12


def _parse(path):
    def rows(name):
        return [ln.split() for ln in open(path / name).read().splitlines() if not ln.startswith("#")]
    cams = {int(r[0]): r for r in rows("cameras.txt")}
    im = rows("images.txt")
    images = {int(h[0]): (h, p) for h, p in zip(im[0::2], im[1::2])}
    pts = {int(r[0]): r for r in rows("points3D.txt")}
    return cams, images, pts


def _hand_built(seed=0):
    """A CPU reconstruction of planted_cameras' geometry with hand-made tracks: 4 images, 3 registered, 60 tracks of which some
    are not ok and some elements not inliers; points.error is the mean reprojection error of each ok track's inliers."""
    rng = np.random.default_rng(seed)
    N, T = 4, 60
    K = np.stack([synthetic._scene_intrinsics(rng, 512, 384) for _ in range(N)])
    R = np.stack([synthetic._scene_rotation(rng, 1, 30) for _ in range(N)])
    t = rng.normal(size=(N, 3)) + [0, 0, 10]
    X = rng.uniform(-2, 2, (T, 3))
    reg = np.array([True, True, False, True])
    R[~reg], t[~reg] = 0, 0
    kp_counts = rng.integers(T + 5, T + 20, N)
    kp_off = np.concatenate([[0], np.cumsum(kp_counts)])
    kps = rng.uniform(0, 500, (kp_off[-1], 2)).astype(np.float32)
    elements, tr_off, inlier = [], [0], []
    ids = [rng.permutation(kp_counts[i])[:T] for i in range(N)]
    for k in range(T):
        imgs = np.sort(rng.choice(N, rng.integers(2, N + 1), replace=False))
        for i in imgs:
            elements.append((i, ids[i][k]))
            inlier.append(bool(reg[i]) and rng.random() < 0.9)
            if reg[i]:
                p = K[i] @ (R[i] @ X[k] + t[i])
                kps[kp_off[i] + ids[i][k]] = (p[:2] / p[2] + rng.normal(scale=0.5, size=2)).astype(np.float32)
        tr_off.append(len(elements))
    el = np.array(elements, np.int32)
    inlier = np.array(inlier)
    tr_off = np.array(tr_off)
    track = np.repeat(np.arange(T), np.diff(tr_off))
    ok = np.array([inlier[tr_off[k]:tr_off[k + 1]].sum() >= 2 for k in range(T)]) & (rng.random(T) < 0.9)
    inlier &= ok[track]
    err = np.zeros(T)
    for k in np.flatnonzero(ok):
        e = [np.linalg.norm((lambda p: p[:2] / p[2])(K[i] @ (R[i] @ X[k] + t[i])) - kps[kp_off[i] + a]) for (i, a), u in
             zip(el[tr_off[k]:tr_off[k + 1]], inlier[tr_off[k]:tr_off[k + 1]]) if u]
        err[k] = np.mean(e)
    X[~ok] = 0
    graph = MatchGraph(torch.from_numpy(kp_off), torch.from_numpy(kps), torch.ones(len(kps)), torch.zeros(1, dtype=torch.int64),
                       torch.zeros(0, 2, dtype=torch.int32), torch.zeros(0))
    tracks = Tracks(torch.from_numpy(tr_off), torch.from_numpy(el), torch.full((len(kps),), -1, dtype=torch.int32), 0)
    pts = Points3D(torch.from_numpy(X), torch.from_numpy(ok), torch.zeros(T, dtype=torch.int32), torch.from_numpy(err),
                   torch.from_numpy(inlier))
    recon = mapper.Reconstruction(torch.from_numpy(reg), torch.from_numpy(R), torch.from_numpy(t), pts, None, [], "all_registered")
    return recon, graph, tracks, K, np.tile([384, 512], (N, 1))


def check_colmap_model(path, recon, graph, tracks, K, sizes):
    """Parses the model back: ids and counts, every POINT3D_ID <-> TRACK entry both ways, the cameras, and each point reprojected
    with the written cameras gives its written ERROR (points.error) to 1e-9."""
    cams, images, pts = _parse(path)
    N = K.shape[0]
    reg = recon.registered.cpu().numpy()
    ok = recon.points.ok.cpu().numpy()
    kp_off = graph.kp_offsets.cpu().numpy()
    kps = graph.keypoints.cpu().numpy().astype(np.float64)
    assert sorted(cams) == list(range(1, N + 1))
    for i in range(N):
        c = cams[i + 1]
        assert c[1] == "PINHOLE" and (int(c[2]), int(c[3])) == (sizes[i][1], sizes[i][0])
        assert [float(v) for v in c[4:]] == [K[i, 0, 0], K[i, 1, 1], K[i, 0, 2], K[i, 1, 2]]
    assert sorted(images) == [i + 1 for i in np.flatnonzero(reg)]
    assert sorted(pts) == [k + 1 for k in np.flatnonzero(ok)]
    Rw, tw = recon.R.cpu().numpy(), recon.t.cpu().numpy()
    cam_of, refs = {}, set()
    for iid, (h, p2d) in images.items():
        i = iid - 1
        q, tv = np.array(h[1:5], float), np.array(h[5:8], float)
        assert q[0] >= 0 and int(h[8]) == iid
        Rq = _quat_to_R(q)
        assert np.abs(Rq - Rw[i]).max() <= 1e-12 and np.array_equal(tv, tw[i])
        cam_of[iid] = (Rq, tv)
        trip = np.array(p2d, dtype=object).reshape(-1, 3)
        assert len(trip) == kp_off[i + 1] - kp_off[i]                          # every keypoint, POINT2D_IDX = keypoint id
        assert np.array_equal(trip[:, :2].astype(float), kps[kp_off[i]:kp_off[i + 1]])
        for a, pid in enumerate(trip[:, 2].astype(int)):
            if pid != -1:
                refs.add((pid, iid, a))
    back = set()
    for pid, r in pts.items():
        Xp = np.array(r[1:4], float)
        assert r[4:7] == ["128", "128", "128"]
        assert np.array_equal(Xp, recon.points.X[pid - 1].cpu().numpy())
        track = np.array(r[8:], int).reshape(-1, 2)
        errs = []
        for iid, a in track:
            back.add((pid, iid, a))
            Rq, tv = cam_of[iid]
            p = K[iid - 1] @ (Rq @ Xp + tv)
            errs.append(np.linalg.norm(p[:2] / p[2] - kps[kp_off[iid - 1] + a]))
        assert abs(np.mean(errs) - float(r[7])) <= 1e-9 and float(r[7]) == float(recon.points.error[pid - 1])
    assert refs == back and len(back) == int((recon.points.inlier.cpu().numpy()).sum())


def test_colmap_writer_round_trip(tmp_path):
    recon, graph, tracks, K, sizes = _hand_built()
    mapper.write_colmap_text(tmp_path, recon, graph, tracks, K, sizes)
    check_colmap_model(tmp_path, recon, graph, tracks, K, sizes)
    Ks = K.copy()
    Ks[1, 0, 1] = 0.5
    with pytest.raises(ValueError, match="skew"):
        mapper.write_colmap_text(tmp_path / "b", recon, graph, tracks, Ks, sizes)
    Kr = K.copy()
    Kr[2, 2, 2] = 2.0
    with pytest.raises(ValueError, match="pinhole"):
        mapper.write_colmap_text(tmp_path / "c", recon, graph, tracks, Kr, sizes)
    assert math.isfinite(float(recon.points.error.max()))
