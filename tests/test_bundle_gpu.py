"""`bundle_adjust` on the GPU: on `planted_cameras` scenes with perturbed cameras, triangulated by `triangulate_tracks`, the device
agrees with `oracle/bundle.py` (the first trial's F and pred to 1e-10, the kept/rejected sequence wherever rho is clear of 1e-3,
the final cost to 1e-8 and the parameters to the flatness of the minimum); it reaches the points-only cost at the true cameras and
removes most of the camera error; the Cauchy loss resists moved observations; fixed poses come back bit-identical; edge cases and
byte-identical reruns."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.bundle import bundle_adjust as oracle_ba, track_costs  # noqa: E402
from roma_b200 import MatchGraph, Points3D, Tracks, build_tracks, bundle_adjust, consolidate_matches, synthetic, triangulate_tracks  # noqa: E402
from roma_b200 import verify_matches  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}


def _scene(seed, N, points, cs=1, outlier_frac=0.0, size=(384, 512), rot_deg=0.3, centre=0.05, drop_conflicts=True):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cs, outlier_frac=outlier_frac,
                                                                      device=DEV)
    g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    if outlier_frac > 0:
        g = verify_matches(pairs, g, threshold=THR[cs])[0]
    tr = build_tracks(pairs, g, drop_conflicts=drop_conflicts)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, rot_deg, centre)
    pts = triangulate_tracks(g, tr, K, R1, t1, max_error=20.0)
    return g, tr, pts, K, R1, t1, R, t, X


def _oracle(g, tr, pts, K, R, t, **kw):
    return oracle_ba(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.X, pts.ok, pts.inlier, K, R, t, **kw)


@pytest.mark.parametrize("seed, N, cs, outlier_frac, loss_scale, points", [
    (0, 3, 1, 0.0, None, 500), (1, 3, 4, 0.2, 1.0, 500), (2, 8, 1, 0.2, None, 400), (3, 8, 4, 0.0, 2.0, 400),
    (4, 16, 1, 0.0, 1.0, 300), (5, 16, 4, 0.2, None, 300)])
def test_device_matches_the_oracle(seed, N, cs, outlier_frac, loss_scale, points):
    g, tr, pts, K, R, t, *_ = _scene(seed, N, points, cs, outlier_frac)
    kw = dict(loss_scale=loss_scale, max_iterations=100, function_tolerance=1e-12)
    res = bundle_adjust(g, tr, pts, K, R, t, **kw)
    ref = _oracle(g, tr, pts, K, R, t, **kw)
    tri = ref["trials"]
    print(f"N={N} cs={cs} outliers={outlier_frac} loss={loss_scale}: F {res.cost[0]:.6g} -> {res.cost[-1]:.10g} in {res.accepted.size} "
          f"trials ({res.termination}); oracle {ref['cost'][-1]:.10g} in {ref['accepted'].size} ({ref['termination']})")
    assert abs(res.cost[0] - ref["cost"][0]) <= 1e-10 * ref["cost"][0]
    assert abs(res.pred[0] - tri[0]["pred"]) <= 1e-10 * abs(tri[0]["pred"])
    assert abs(res.cost[1] - ref["cost"][1]) <= 1e-10 * ref["cost"][1]
    # The kept/rejected sequence up to the first trial whose rho lies within rounding of 1e-3.  A cost is a sum of squared
    # differences of pixel coordinates, known to about 1e-12 F, so rho = (F - F_new) / pred is known to about 1e-12 F / |pred|.
    n = min(res.accepted.size, ref["accepted"].size)
    for k in range(n):
        if abs(tri[k]["margin"]) <= 1e-6 + 1e-10 * tri[k]["F"] / abs(tri[k]["pred"]):
            break
        assert res.accepted[k] == ref["accepted"][k], k
    assert abs(res.cost[-1] - ref["cost"][-1]) <= 1e-8 * ref["cost"][-1]
    # both stop where the cost is flat to rounding: the cameras agree to 1e-5 and the points to 2e-4 (as the oracle and scipy do)
    ok = pts.ok.cpu().numpy()
    assert np.abs(res.R.cpu().numpy() - ref["R"]).max() < 1e-5 and np.abs(res.t.cpu().numpy() - ref["t"]).max() < 1e-5
    assert np.abs(res.points.X.cpu().numpy()[ok] - ref["X"][ok]).max() < 2e-4
    assert torch.equal(res.R[0], R[0].double()) and torch.equal(res.t[0], t[0].double()) and res.t[1, 0] == t[1, 0]


def _align(C, Ct):
    """7-DoF (Umeyama) alignment of centres C onto Ct: (s, Q, T) with Ct ~ s Q C + T."""
    mc, mt = C.mean(0), Ct.mean(0)
    A, B = C - mc, Ct - mt
    U, S, Vt = np.linalg.svd(B.T @ A / len(C))
    D = np.eye(3)
    D[2, 2] = np.sign(np.linalg.det(U @ Vt))
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / (A * A).sum(1).mean()
    return s, Q, mt - s * Q @ mc


def _camera_errors(R, t, Rt, tt):
    """Median rotation error (degrees) and centre error after aligning the centres to the truth."""
    R, t, Rt, tt = (v.cpu().numpy() for v in (R, t, Rt, tt))
    C, Ct = -np.einsum("nji,nj->ni", R, t), -np.einsum("nji,nj->ni", Rt, tt)
    s, Q, T = _align(C, Ct)
    dR = np.einsum("nij,kj,nlk->nil", R, Q, Rt)                    # R Q^T Rt^T
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    return np.median(ang), np.median(np.linalg.norm(s * C @ Q.T + T - Ct, axis=1))


def test_quality_on_a_clean_scene():
    g, tr, pts, K, R, t, Rt, tt, X = _scene(6, 16, 2000, size=(768, 1024))
    res = bundle_adjust(g, tr, pts, K, R, t, function_tolerance=1e-12, max_iterations=100)
    N = K.shape[0]
    ref = bundle_adjust(g, tr, pts, K, Rt, tt, fixed_poses=range(N), function_tolerance=1e-12, max_iterations=100)
    r0, c0 = _camera_errors(R, t, Rt, tt)
    r1, c1 = _camera_errors(res.R, res.t, Rt, tt)
    print(f"F {res.cost[0]:.6g} -> {res.cost[-1]:.8g} ({res.termination}, {res.accepted.size} trials), points only at the true cameras "
          f"{ref.cost[-1]:.8g}; rotation error {r0:.4f} -> {r1:.5f} deg, centre error {c0:.4f} -> {c1:.5f}")
    assert res.cost[-1] <= (1 + 1e-6) * ref.cost[-1]
    assert r1 < 0.03 and c1 < 0.005


def _move(g, tr, pts, frac, seed):
    """Moves `frac` of the inlier observations of tracks of 3 elements or more by 20-50 px."""
    rng = np.random.default_rng(seed)
    off, el = tr.track_offsets.cpu().numpy(), tr.elements.cpu().numpy().astype(np.int64)
    L = np.diff(off)
    moved = np.repeat(L >= 3, L) & pts.inlier.cpu().numpy() & (rng.random(el.shape[0]) < frac)
    ang, r = rng.uniform(0, 2 * np.pi, moved.sum()), rng.uniform(20, 50, moved.sum())
    xy = g.keypoints.cpu().numpy().copy()
    xy[g.kp_offsets.cpu().numpy()[el[moved, 0]] + el[moved, 1]] += np.stack((r * np.cos(ang), r * np.sin(ang)), 1).astype(np.float32)
    return MatchGraph(g.kp_offsets, torch.from_numpy(xy).to(DEV), g.kp_scores, g.match_offsets, g.matches, g.match_scores), moved


def test_cauchy_loss_resists_moved_observations():
    g, tr, pts, K, R, t, Rt, tt, X = _scene(7, 16, 2000, size=(768, 1024))
    h, moved = _move(g, tr, pts, 0.1, 0)
    plain = bundle_adjust(h, tr, pts, K, R, t)
    robust = bundle_adjust(h, tr, pts, K, R, t, loss_scale=1.0)
    rp, rr = _camera_errors(plain.R, plain.t, Rt, tt)[0], _camera_errors(robust.R, robust.t, Rt, tt)[0]
    print(f"moved {moved.sum()} observations: rotation error {rp:.4f} deg without a loss, {rr:.4f} with loss_scale=1")
    assert moved.sum() > 1000 and rr < rp


def test_points_only():
    g, tr, pts, K, R, t, *_ = _scene(8, 8, 800)
    N = K.shape[0]
    # triangulate_tracks leaves each point at its own minimum, so start from points moved by up to 0.02 units
    gen = torch.Generator(device=DEV).manual_seed(0)
    moved = pts.X + torch.where(pts.ok[:, None], 0.02 * (2 * torch.rand(pts.X.shape, generator=gen, device=DEV, dtype=torch.float64) - 1), 0.0)
    start = Points3D(moved, pts.ok, pts.num_inliers, pts.error, pts.inlier)
    res = bundle_adjust(g, tr, start, K, R, t, fixed_poses=range(N), function_tolerance=1e-14, max_iterations=100)
    assert torch.equal(res.R, R.double()) and torch.equal(res.t, t.double()) and res.accepted.any()
    args = (g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements)
    before = track_costs(*args, pts.X, pts.ok, pts.inlier, K, R, t)
    after = track_costs(*args, res.points.X, pts.ok, pts.inlier, K, R, t)
    ok = pts.ok.cpu().numpy()
    # the tracks are independent with every pose fixed, and each one ends at its own minimum: at most its starting cost, to
    # the rounding of a cost
    worse = after[ok] > before[ok] * (1 + 1e-9) + 1e-9
    print(f"{ok.sum()} ok tracks, {int(worse.sum())} above their starting cost; total {before[ok].sum():.6g} -> {after[ok].sum():.6g}")
    assert not worse.any()


def test_edge_cases():
    g, tr, pts, K, R, t, *_ = _scene(9, 4, 400)
    N = K.shape[0]
    # a free camera with no observations keeps its pose
    el = tr.elements
    inl = pts.inlier & (el[:, 0] != N - 1)
    p2 = Points3D(pts.X, pts.ok, pts.num_inliers, pts.error, inl)
    res = bundle_adjust(g, tr, p2, K, R, t)
    assert res.accepted.any() and torch.equal(res.R[N - 1], R[N - 1].double()) and torch.equal(res.t[N - 1], t[N - 1].double())
    # tracks that are not ok keep X = 0, and ok, num_inliers and inlier come back as given
    ok = pts.ok.clone()
    ok[::3] = False
    p3 = Points3D(torch.where(ok[:, None], pts.X, 0.0), ok, pts.num_inliers, pts.error, pts.inlier)
    res = bundle_adjust(g, tr, p3, K, R, t)
    assert (res.points.X[~ok] == 0).all() and torch.equal(res.points.inlier, pts.inlier) and torch.equal(res.points.ok, ok)
    # max_iterations=0 and no tracks return the inputs
    res = bundle_adjust(g, tr, pts, K, R, t, max_iterations=0)
    assert res.termination == "max_iterations" and res.cost.size == 1 and res.accepted.size == 0
    assert torch.equal(res.points.X, pts.X) and torch.equal(res.R, R.double()) and torch.equal(res.t, t.double())
    empty = Tracks(torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(0, 2, dtype=torch.int32, device=DEV), tr.kp_track, 0)
    pe = Points3D(torch.zeros(0, 3, dtype=torch.float64, device=DEV), torch.zeros(0, dtype=torch.bool, device=DEV),
                  torch.zeros(0, dtype=torch.int32, device=DEV), torch.zeros(0, dtype=torch.float64, device=DEV),
                  torch.zeros(0, dtype=torch.bool, device=DEV))
    res = bundle_adjust(g, empty, pe, K, R, t)
    assert res.termination == "nothing_to_adjust" and res.points.X.shape == (0, 3) and torch.equal(res.R, R.double())
    # no used observations
    p4 = Points3D(pts.X, torch.zeros_like(pts.ok), pts.num_inliers, pts.error, pts.inlier)
    assert bundle_adjust(g, tr, p4, K, R, t).termination == "nothing_to_adjust"


@pytest.mark.parametrize("col, value", [(0, -1), (0, 5), (1, -1), (1, 1 << 20)])
def test_out_of_range_element_raises(col, value):
    g, tr, pts, K, R, t, *_ = _scene(10, 4, 400)
    k = int(torch.nonzero(pts.inlier)[0])
    el = tr.elements.clone()
    el[k, col] = value
    bad = Tracks(tr.track_offsets, el, tr.kp_track, tr.num_conflicting)
    with pytest.raises(ValueError, match="outside"):
        bundle_adjust(g, bad, pts, K, R, t)
    assert bundle_adjust(g, tr, pts, K, R, t).accepted.any()                  # the device is fine afterwards


def test_repeated_images_are_refused():
    g, tr, pts, K, R, t, *_ = _scene(11, 4, 400)
    off = tr.track_offsets.cpu()
    k = int(torch.nonzero((off[1:] - off[:-1]) >= 2)[0])
    el = tr.elements.clone()
    a = int(off[k])
    el[a + 1] = el[a]
    p = Points3D(pts.X, pts.ok.clone(), pts.num_inliers, pts.error, pts.inlier.clone())
    p.ok[k] = True
    p.inlier[a:a + 2] = True
    with pytest.raises(ValueError, match="repeat an image"):
        bundle_adjust(g, Tracks(tr.track_offsets, el, tr.kp_track, tr.num_conflicting), p, K, R, t)


def test_byte_identical_reruns():
    g, tr, pts, K, R, t, *_ = _scene(12, 8, 600, outlier_frac=0.2)
    a = bundle_adjust(g, tr, pts, K, R, t, loss_scale=1.0)
    b = bundle_adjust(g, tr, pts, K.cpu().numpy(), R.cpu(), t, loss_scale=1.0)
    for x, y in ((a.R, b.R), (a.t, b.t), (a.points.X, b.points.X), (a.points.error, b.points.error)):
        assert x.dtype == y.dtype and x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
    assert np.array_equal(a.cost, b.cost) and np.array_equal(a.accepted, b.accepted) and a.termination == b.termination
