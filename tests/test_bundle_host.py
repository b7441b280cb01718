"""CPU tests of bundle adjustment (`bundle_adjust`): the numpy oracle against `scipy.optimize.least_squares` on perturbed
`planted_cameras` scenes with both losses, Rodrigues and its small-angle branch, the camera-major list, `perturb_cameras`, every
argument rule (raised before any device work), the gauge defaults and the workspace formula."""
import math

import numpy as np
import pytest
import torch
from scipy.optimize import least_squares
from scipy.sparse import lil_matrix
from scipy.spatial.transform import Rotation

from oracle.bundle import bundle_adjust as oracle_ba, camera_major, rodrigues
from oracle.match_graph import consolidate
from oracle.tracks import tracks as oracle_tracks
from oracle.triangulate import triangulate
from roma_b200 import bundle as rb_ba, cabi, synthetic
from roma_b200.match_graph import MatchGraph
from roma_b200.tracks import Tracks
from roma_b200.triangulate import Points3D


def oracle_scene(seed, N, points, rot_deg=0.3, centre=0.05, size=(384, 512)):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size)
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy())
    tr = oracle_tracks(pairs.numpy(), g)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, rot_deg, centre)
    tri = triangulate(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], K, R1, t1, max_error=20.0)
    return g, tr, tri, K.numpy(), R1.numpy(), t1.numpy(), R.numpy(), t.numpy()


def scipy_ba(g, tr, tri, K, R, t, fixed_poses, fixed_tx, loss_scale):
    """The same problem through scipy: rotations as R = Rotation(v) R_0, translations without the held t_x, points of ok tracks."""
    off, el = tr["track_offsets"], tr["elements"].astype(np.int64)
    T, N = off.size - 1, K.shape[0]
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(tri["ok"], np.diff(off)) & tri["inlier"])
    img, trk = el[e, 0], track[e]
    obs = g["keypoints"].astype(np.float64)[g["kp_offsets"][img] + el[e, 1]]
    free = [i for i in range(N) if i not in fixed_poses]
    pts = np.unique(trk)
    cam_cols = {}
    col = 0
    for i in free:
        idx = []
        for j in range(6):
            if j == 3 and i in fixed_tx:
                idx.append(-1)
            else:
                idx.append(col)
                col += 1
        cam_cols[i] = idx
    pt_col = {k: col + 3 * n for n, k in enumerate(pts)}
    n_par = col + 3 * pts.size

    def unpack(p):
        Rs, ts, X = R.copy(), t.copy(), tri["X"].copy()
        for i in free:
            v = [p[c] if c >= 0 else 0.0 for c in cam_cols[i]]
            Rs[i] = Rotation.from_rotvec(v[:3]).as_matrix() @ R[i]
            ts[i] = t[i] + np.array(v[3:])
        for k in pts:
            X[k] = tri["X"][k] + p[pt_col[k]:pt_col[k] + 3]
        return Rs, ts, X

    def fun(p):
        Rs, ts, X = unpack(p)
        q = np.einsum("mij,mj->mi", K[img], np.einsum("mij,mj->mi", Rs[img], X[trk]) + ts[img])
        r = q[:, :2] / q[:, 2:3] - obs
        if loss_scale is None:
            return r.reshape(-1)
        # scipy's loss acts on each residual and rule 2's on each observation's s = |r|^2, so the loss goes into the residuals:
        # r sqrt(rho(s) / s) has the squared norm rho(s), scipy's loss="cauchy", f_scale=c of the observation
        s = (r * r).sum(1)
        c2 = loss_scale * loss_scale
        return (r * np.sqrt(c2 * np.log1p(s / c2) / s)[:, None]).reshape(-1)

    rows = 2
    sp = lil_matrix((rows * e.size, n_par), dtype=int)
    for m, (i, k) in enumerate(zip(img, trk)):
        for c in cam_cols.get(i, []):
            if c >= 0:
                sp[rows * m:rows * m + rows, c] = 1
        sp[rows * m:rows * m + rows, pt_col[k]:pt_col[k] + 3] = 1
    res = least_squares(fun, np.zeros(n_par), jac="3-point", jac_sparsity=sp, method="trf", x_scale="jac", ftol=1e-15, xtol=1e-15,
                        gtol=1e-15, max_nfev=500)
    Rs, ts, X = unpack(res.x)
    return res.cost, Rs, ts, X


@pytest.mark.parametrize("seed, N, points, loss_scale", [(0, 3, 300, None), (1, 4, 300, 1.0), (2, 5, 200, None), (3, 5, 200, 2.0)])
def test_oracle_reaches_the_scipy_minimum(seed, N, points, loss_scale):
    g, tr, tri, K, R, t, Rt, tt = oracle_scene(seed, N, points)
    kw = dict(fixed_poses=(0,), fixed_tx=(1,), loss_scale=loss_scale)
    ref = oracle_ba(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"], K, R, t,
                    max_iterations=200, function_tolerance=1e-15, **kw)
    cost, Rs, ts, X = scipy_ba(g, tr, tri, K, R, t, [0], [1], loss_scale)
    ok = tri["ok"]
    print(f"N={N}: F {ref['cost'][0]:.6g} -> {ref['cost'][-1]:.10g} in {ref['accepted'].size} trials ({ref['termination']}), scipy {cost:.10g}")
    assert ref["cost"][-1] <= ref["cost"][0] and abs(ref["cost"][-1] - cost) <= 1e-8 * cost
    dR, dt, dX = np.abs(ref["R"] - Rs).max(), np.abs(ref["t"] - ts).max(), np.abs(ref["X"][ok] - X[ok]).max()
    print(f"largest differences: R {dR:.1e}, t {dt:.1e}, X {dX:.1e}")
    # both stop where the cost is flat to about 1e-10 relative, which fixes the cameras to about 1e-5 and the points to 2e-4
    assert dR < 1e-5 and dt < 1e-5 and dX < 2e-4
    assert np.array_equal(ref["R"][0], R[0]) and np.array_equal(ref["t"][0], t[0]) and ref["t"][1, 0] == t[1, 0]


def test_oracle_lowers_the_camera_error():
    g, tr, tri, K, R, t, Rt, tt = oracle_scene(4, 5, 400)
    ref = oracle_ba(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"], K, R, t)
    assert ref["termination"] == "function_tolerance" and ref["cost"][-1] < 0.2 * ref["cost"][0]
    assert all(np.isfinite([tr_["margin"] for tr_ in ref["trials"]]))


def test_rodrigues_and_its_small_angle_branch():
    rng = np.random.default_rng(0)
    w = rng.normal(size=(50, 3)) * rng.uniform(1e-3, 3.0, (50, 1))
    assert np.allclose(rodrigues(w), Rotation.from_rotvec(w).as_matrix(), atol=1e-14)
    tiny = np.array([[1e-9, -2e-9, 3e-9], [0.0, 0.0, 0.0]])
    E = rodrigues(tiny)
    assert np.array_equal(E[1], np.eye(3))
    assert E[0, 0, 1] == -tiny[0, 2] and E[0, 2, 1] == tiny[0, 0] and E[0, 0, 0] == 1.0     # I + [w]x exactly
    assert np.allclose(E[0], Rotation.from_rotvec(tiny[0]).as_matrix(), atol=1e-17)
    edge = np.array([[2.0 ** -26 * 1.0001, 0, 0]])                                          # just above the branch point
    assert np.allclose(rodrigues(edge), Rotation.from_rotvec(edge).as_matrix(), atol=1e-16)


def test_camera_major_list():
    off = np.array([0, 3, 5, 8])
    el = np.array([[2, 0], [0, 1], [1, 0], [0, 0], [2, 1], [1, 1], [0, 2], [2, 2]])
    ok = np.array([True, False, True])
    inl = np.array([1, 1, 0, 1, 1, 1, 1, 1], bool)
    oo, obs = camera_major(off, el, ok, inl, 4)
    assert obs.tolist() == [1, 6, 5, 0, 7] and oo.tolist() == [0, 2, 3, 5, 5]


def test_perturb_cameras():
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(0, 6, 10)
    R1, t1 = synthetic.perturb_cameras(3, R, t, 0.3, 0.05)
    R2, t2 = synthetic.perturb_cameras(3, R.numpy(), t.numpy(), 0.3, 0.05)
    assert isinstance(R1, torch.Tensor) and np.array_equal(R1.numpy(), R2) and np.array_equal(t1.numpy(), t2)
    ang = np.degrees(np.arccos(np.clip((np.einsum("nij,nij->n", R1.numpy(), R.numpy()) - 1) / 2, -1, 1)))
    C0, C1 = (-np.einsum("nji,nj->ni", a, b) for a, b in ((R.numpy(), t.numpy()), (R2, t2)))
    assert np.allclose(ang, 0.3, atol=1e-6) and np.allclose(np.linalg.norm(C1 - C0, axis=1), 0.05)
    assert np.allclose(np.einsum("nij,nkj->nik", R2, R2), np.eye(3), atol=1e-14)


def test_workspace_formula_equals_the_buffers():
    for N, F, T, E in ((1, 0, 1, 1), (3, 2, 10, 25), (16, 15, 1000, 4097), (50, 49, 40000, 1 << 20)):
        b = rb_ba._buffers("meta", N, F, T, E)
        assert sum(v.numel() * v.element_size() for v in b.values()) == rb_ba.workspace_bytes(N, F, T, E), (N, F, T, E)
    assert rb_ba.workspace_bytes(200, 199, 40000, 4_000_000) < rb_ba.WORKSPACE_BYTES


# ---- argument rules -------------------------------------------------------------------------------------------------------
KF = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])


def mg(N=2):
    kp = torch.arange(0, 2 * N + 1, 2, dtype=torch.int64)
    return MatchGraph(kp, torch.zeros(2 * N, 2), torch.zeros(2 * N), torch.zeros(2, dtype=torch.int64), torch.zeros(0, 2, dtype=torch.int32),
                      torch.zeros(0))


def tk(N=2):
    el = torch.tensor([(i, 0) for i in range(N)], dtype=torch.int32).reshape(-1, 2)
    return Tracks(torch.tensor([0, N], dtype=torch.int64), el, torch.zeros(2 * N, dtype=torch.int32), 0)


def pts(T=1, E=2):
    return Points3D(torch.zeros(T, 3, dtype=torch.float64), torch.ones(T, dtype=torch.bool), torch.zeros(T, dtype=torch.int32),
                    torch.zeros(T, dtype=torch.float64), torch.ones(E, dtype=torch.bool))


def cams(N=2):
    return dict(K=np.repeat(KF[None], N, 0), R=np.repeat(np.eye(3)[None], N, 0), t=np.zeros((N, 3)))


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case", [
    dict(graph={"kp_offsets": torch.zeros(1, dtype=torch.int64)}),
    dict(tracks=(torch.zeros(1, dtype=torch.int64), torch.zeros(0, 2))),
    dict(R=np.eye(3)), dict(t=np.array([[0.0, 0, 0], [np.nan, 0, 0]])), dict(K=np.repeat(np.eye(3, dtype=np.int64)[None], 2, 0)),
    dict(points=(torch.zeros(1, 3),)),
    dict(points=Points3D(torch.zeros(1, 3), torch.ones(1, dtype=torch.bool), torch.zeros(1, dtype=torch.int32), torch.zeros(1),
                         torch.ones(2, dtype=torch.bool))),                          # X not float64
    dict(points=pts(T=2)), dict(points=pts(E=3)),
    dict(points=Points3D(torch.zeros(1, 3, dtype=torch.float64), torch.ones(1, dtype=torch.uint8), torch.zeros(1, dtype=torch.int32),
                         torch.zeros(1), torch.ones(2, dtype=torch.bool))),          # ok not bool
    dict(fixed_poses=(2,)), dict(fixed_poses=(-1,)), dict(fixed_poses=(0.5,)), dict(fixed_poses=5), dict(fixed_tx=(3,)),
    dict(fixed_tx=(True,)),
    dict(loss_scale=0.0), dict(loss_scale=-1.0), dict(loss_scale=math.inf), dict(loss_scale=math.nan), dict(loss_scale="one"),
    dict(max_iterations=-1), dict(max_iterations=2.0), dict(max_iterations=True),
    dict(function_tolerance=-1e-9), dict(function_tolerance=math.nan), dict(function_tolerance=None),
    dict(workspace_bytes=100), dict(workspace_bytes=1.5),
    {},                                                                               # CPU tensors: the call runs on a CUDA device only
])
def test_argument_errors_before_device_work(no_device, case):
    kw = dict(graph=mg(), tracks=tk(), points=pts(), **cams())
    kw.update(case)
    with pytest.raises(ValueError) as e:
        rb_ba.bundle_adjust(kw.pop("graph"), kw.pop("tracks"), kw.pop("points"), kw.pop("K"), kw.pop("R"), kw.pop("t"), **kw)
    assert ("CUDA device" in str(e.value)) == (not case), str(e.value)
    assert str(e.value).startswith("bundle_adjust: ")


@pytest.mark.parametrize("N", [1, 2])
def test_gauge_defaults_hold_for_one_and_two_cameras(no_device, N):
    with pytest.raises(ValueError, match="CUDA device"):               # the defaults pass every rule; only the device rule fails
        rb_ba.bundle_adjust(mg(N), tk(N), pts(E=N), **cams(N))
    with pytest.raises(ValueError, match="fixed_tx"):
        rb_ba.bundle_adjust(mg(N), tk(N), pts(E=N), **cams(N), fixed_tx=(5,))


def test_entry_points_and_exports():
    import roma_b200
    assert {f"romab200_ba_{n}" for n in ("setup", "linearize", "cameras", "cholesky", "step", "cost", "error")} <= set(cabi.FUNCTIONS)
    assert roma_b200.bundle_adjust is rb_ba.bundle_adjust and roma_b200.BundleResult is rb_ba.BundleResult
    assert cabi.RB_BA_CAM == 21 and cabi.RB_BA_TRACK == 13 and cabi.RB_BA_NB == 32
    assert not any(f.startswith("dtype") for f, _ in cabi.STRUCT_FIELDS["rb_ba_args"])
