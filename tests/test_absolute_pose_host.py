"""The absolute-pose oracle (`oracle/absolute_pose.py`) on the CPU: its Lambda Twist P3P gives cv2.solveP3P's solution set, its RANSAC
recovers planted poses at least as accurately as cv2.solvePnPRansac with the P3P solver, and the argument rules, the registration
oracles and the workspace formula of `register_images` hold.  None of this needs a GPU."""
import math

import cv2
import numpy as np
import pytest
import torch

from oracle import absolute_pose as ap
from oracle import register as oreg
from oracle.triangulate import triangulate as tri_oracle
from roma_b200 import cabi, geometry, register
from roma_b200.tracks import Tracks
from roma_b200.triangulate import Points3D


def _camera(rng):
    K = np.array([[rng.uniform(700, 900), 0, rng.uniform(300, 340)], [0, rng.uniform(700, 900), rng.uniform(220, 260)], [0, 0, 1.0]])
    R, _ = cv2.Rodrigues(rng.normal(size=3) * 0.5)
    return K, R, rng.uniform(-1, 1, 3) + [0, 0, 8]


def _project(K, R, t, X):
    p = (X @ R.T + t) @ K.T
    return p[:, :2] / p[:, 2:]


def _rot_deg(Ra, Rb):
    return math.degrees(math.acos(min(1.0, max(-1.0, (np.trace(Ra.T @ Rb) - 1) / 2))))


def test_p3p_matches_cv2_solve_p3p():
    rng = np.random.default_rng(0)
    n_sols = 0
    for _ in range(300):
        K, R, t = _camera(rng)
        X = rng.uniform(-2, 2, (3, 3))
        x = _project(K, R, t, X)
        ours = ap.p3p(ap.bearings(x, K), X)
        _, rv, tv = cv2.solveP3P(X, x, K, None, cv2.SOLVEPNP_P3P)
        theirs = [(cv2.Rodrigues(r)[0], tt.ravel()) for r, tt in zip(rv, tv)]
        assert len(ours) == len(theirs)
        for Rc, tc in theirs:        # the same set: every cv2 solution has a match within 1e-8, and the planted pose is among them
            assert min(max(np.abs(Rc - Ro).max(), np.abs(tc - to).max() / np.linalg.norm(tc)) for Ro, to in ours) <= 1e-8
        assert min(np.abs(Ro - R).max() for Ro, _ in ours) <= 1e-8
        n_sols += len(ours)
    assert n_sols >= 300


def _scene(seed, n, outlier_frac, noise=0.5):
    rng = np.random.default_rng(seed)
    K, R, t = _camera(rng)
    X = rng.uniform(-3, 3, (n, 3))
    x = _project(K, R, t, X) + rng.normal(scale=noise, size=(n, 2))
    out = rng.random(n) < outlier_frac
    x[out] = rng.uniform([0, 0], [640, 480], (int(out.sum()), 2))
    return K, R, t, X, x, out


@pytest.mark.parametrize("outlier_frac", [0.0, 0.2, 0.5])
def test_oracle_recovers_planted_poses_as_well_as_cv2(outlier_frac):
    errs, cv_errs = [], []
    for seed in range(8):
        K, R, t, X, x, out = _scene(seed, 400, outlier_frac)
        res = ap.estimate(x, X, K, max_error=4.0, confidence=0.9999, max_iters=10000, seed=seed)
        assert res["ok"]
        assert (res["mask"][~out].mean() > 0.97) and (not outlier_frac or res["mask"][out].mean() < 0.05)
        cv2.setRNGSeed(seed)
        okc, rv, tv, _ = cv2.solvePnPRansac(X, x, K, None, iterationsCount=10000, reprojectionError=4.0, confidence=0.9999,
                                           flags=cv2.SOLVEPNP_P3P)
        assert okc
        errs.append(_rot_deg(res["R"], R) + np.linalg.norm(res["t"] - t))
        cv_errs.append(_rot_deg(cv2.Rodrigues(rv)[0], R) + np.linalg.norm(tv.ravel() - t))
    print(f"outliers {outlier_frac}: oracle median {np.median(errs):.2e}, cv2 median {np.median(cv_errs):.2e}")
    assert np.median(errs) <= np.median(cv_errs) * 1.05 + 1e-9
    assert max(errs) < 0.05


def test_oracle_edge_cases():
    K, R, t, X, x, _ = _scene(0, 50, 0.0)
    assert not ap.estimate(x[:2], X[:2], K)["ok"]
    three = ap.estimate(x[:3], X[:3], K, max_error=4.0)
    assert three["ok"] and three["iters"] == 1 and three["num_inliers"] == 3
    coincident = ap.estimate(np.repeat(x[:1], 10, 0), np.repeat(X[:1], 10, 0), K)
    assert not coincident["ok"] and not coincident["mask"].any() and (coincident["R"] == 0).all()
    rng = np.random.default_rng(1)
    junk = ap.estimate(rng.uniform(0, 640, (40, 2)), rng.uniform(-3, 3, (40, 3)), K, max_error=0.01, max_iters=200)
    assert junk["num_inliers"] <= 3


def test_refine_lowers_the_cost_and_keeps_depths():
    K, R, t, X, x, _ = _scene(3, 300, 0.0, noise=1.0)
    R0 = ap.exp_so3(np.array([0.01, -0.02, 0.005])) @ R
    R1, t1, changes, _ = ap.refine(R0, t + 0.05, K, x, X)
    assert changes[0] > 0 and _rot_deg(R1, R) < 0.05
    e0, _ = ap.reprojection(R0, t + 0.05, K, x, X)
    e1, d1 = ap.reprojection(R1, t1, K, x, X)
    assert e1.sum() < e0.sum() and (d1 > 0).all()


def _graph_tracks(N=4, per=30, seed=0):
    """A small graph of N images with `per` keypoints each and tracks of every keypoint index across the images."""
    from roma_b200.match_graph import MatchGraph
    rng = np.random.default_rng(seed)
    kp_off = torch.arange(N + 1, dtype=torch.int64) * per
    kps = torch.from_numpy(rng.uniform(0, 500, (N * per, 2)).astype(np.float32))
    g = MatchGraph(kp_off, kps, torch.ones(N * per), torch.zeros(1, dtype=torch.int64), torch.zeros(0, 2, dtype=torch.int32), torch.zeros(0))
    el = torch.tensor([[i, a] for a in range(per) for i in range(N)], dtype=torch.int32)
    tr = Tracks(torch.arange(per + 1, dtype=torch.int64) * N, el, torch.zeros(N * per, dtype=torch.int32), 0)
    return g, tr


def test_gather_oracle_orders_by_element_and_skips_tracks_that_are_not_ok():
    g, tr = _graph_tracks()
    ok = np.arange(30) % 3 != 0
    P = np.arange(90, dtype=np.float64).reshape(30, 3)
    out = ap.gather(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, ok, P, [2, 0])
    x2, X2 = out[0]
    assert len(x2) == ok.sum() and np.array_equal(X2, P[ok])
    assert np.array_equal(x2, g.keypoints.numpy().astype(np.float64)[60:90][ok])
    with pytest.raises(ValueError, match="outside"):
        ap.gather(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements.clone().fill_(99), ok, P, [0])


def test_registered_triangulation_oracle_matches_the_plain_oracle_with_every_image():
    from roma_b200 import synthetic
    rng = np.random.default_rng(4)
    N, n = 4, 60
    K = np.stack([synthetic._scene_intrinsics(rng, 512, 384) for _ in range(N)])
    R = np.stack([cv2.Rodrigues(rng.normal(size=3) * 0.05)[0] for _ in range(N)])
    t = np.stack([[-1.0 + 0.7 * i, 0.0, 8.0] for i in range(N)])
    X = rng.uniform(-2, 2, (n, 3))
    kps = np.concatenate([_project(K[i], R[i], t[i], X) for i in range(N)]).astype(np.float32)
    kp_off = np.arange(N + 1) * n
    el = np.array([[i, a] for a in range(n) for i in range(N)], np.int32)
    off = np.arange(n + 1) * N
    ref = tri_oracle(kp_off, kps, off, el, K, R, t)
    same = oreg.triangulate(kp_off, kps, off, el, K, R, t, range(N))
    for k in ("X", "ok", "num_inliers", "inlier"):
        assert np.array_equal(ref[k], same[k])
    sub = oreg.triangulate(kp_off, kps, off, el, K, R, t, [1, 3])
    assert sub["ok"].all() and (sub["num_inliers"] == 2).all()
    assert not sub["inlier"][np.isin(el[:, 0], [0, 2])].any()
    # a camera that is not registered is not read: any finite values give the same result
    R2, t2 = R.copy(), t.copy()
    R2[0], t2[0] = np.eye(3) * 3, [5.0, 5.0, -5.0]
    sub2 = oreg.triangulate(kp_off, kps, off, el, K, R2, t2, [1, 3])
    assert np.array_equal(sub["X"], sub2["X"]) and np.array_equal(sub["inlier"], sub2["inlier"])


def test_estimator_argument_rules():
    x, X = np.zeros((5, 2)), np.zeros((5, 3))
    for kw in (dict(max_error=0), dict(max_error=float("nan")), dict(confidence=1.0), dict(confidence=0), dict(max_iters=0),
               dict(max_iters=True), dict(max_iters=1.5), dict(seed=-1), dict(seed=1 << 64)):
        with pytest.raises(ValueError):
            geometry.estimate_absolute_pose_batched([x], [X], np.eye(3), **kw)
    with pytest.raises(ValueError):
        geometry.estimate_absolute_pose_batched([], [], np.eye(3))
    with pytest.raises(ValueError):
        geometry.estimate_absolute_pose_batched([x], [X, X], np.eye(3))


def test_register_argument_rules():
    g, tr = _graph_tracks()
    T, E = 30, 120
    pts = Points3D(torch.zeros(T, 3, dtype=torch.float64), torch.ones(T, dtype=torch.bool), torch.zeros(T, dtype=torch.int32),
                   torch.zeros(T, dtype=torch.float64), torch.zeros(E, dtype=torch.bool))
    K = np.tile(np.eye(3), (4, 1, 1))
    bad = [dict(images=[0, 0]), dict(images=[4]), dict(images=[-1]), dict(images=[True]), dict(images=[0.5]), dict(min_inliers=-1),
           dict(max_error=0), dict(confidence=2), dict(max_iters=0), dict(workspace_bytes=0)]
    for kw in bad:
        args = dict(images=[1, 2])
        args.update(kw)
        with pytest.raises(ValueError):
            register.register_images(g, tr, pts, K, **args)
    with pytest.raises(ValueError, match="K"):
        register.register_images(g, tr, pts, np.eye(3), [1])
    with pytest.raises(ValueError, match="points"):
        register.register_images(g, tr, "points", K, [1])
    short = Points3D(pts.X[:5], pts.ok[:5], pts.num_inliers, pts.error, pts.inlier)
    with pytest.raises(ValueError, match="aligned"):
        register.register_images(g, tr, short, K, [1])
    with pytest.raises(ValueError, match="graph"):
        register.register_images("graph", tr, pts, K, [1])


def test_workspace_formula_matches_the_buffers(monkeypatch):
    """include/romab200.h's per-chunk bytes against what `geometry._abs_launch` and `register_images` allocate for a chunk, on the
    meta device (no kernel runs)."""
    allocated = {}
    monkeypatch.setattr(geometry, "_ransac_rounds", lambda *a, **k: None)
    monkeypatch.setattr(cabi, "call", lambda *a, **k: None)
    for ns in ([5], [3000, 10, 0], [20000] * 7, [1, 2, 3, 70000]):
        total = sum(ns)
        meta = dict(device="meta")
        x = torch.empty(max(total, 1), 2, dtype=torch.float64, **meta)
        X = torch.empty(max(total, 1), 3, dtype=torch.float64, **meta)
        off = torch.empty(len(ns) + 1, dtype=torch.int64, **meta)
        K = torch.empty(len(ns), 3, 3, dtype=torch.float64, **meta)
        images = torch.empty(len(ns), dtype=torch.int32, **meta)
        buf = geometry._abs_launch(x, X, off, K, max(ns), 1.0, 0.99, 100, 0)
        allocated = sum(v.numel() * v.element_size() for v in buf.values()) + sum(v.numel() * v.element_size() for v in (x, X, off, K, images))
        assert allocated == register.chunk_bytes(ns), (ns, allocated, register.chunk_bytes(ns))


def test_chunk_plan_covers_every_image_within_the_budget():
    ns = [20000, 5, 0, 70000, 3000, 12, 20000]
    for budget in (1, 1 << 20, 5 << 20, 1 << 30):
        plan = register.plan_chunks(ns, budget)
        assert [b for b, _ in plan] == [0] + [e for _, e in plan[:-1]] and plan[-1][1] == len(ns)
        for b, e in plan:
            assert e - b == 1 or register.chunk_bytes(ns[b:e]) <= budget
    assert register.plan_chunks(ns, 1 << 30) == [(0, len(ns))]
    assert register.plan_chunks([1] * (cabi.RB_ABS_MAX_BATCH + 5), 1 << 40) == [(0, cabi.RB_ABS_MAX_BATCH),
                                                                                (cabi.RB_ABS_MAX_BATCH, cabi.RB_ABS_MAX_BATCH + 5)]
