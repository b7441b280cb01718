"""CPU tests of self-calibration: the SIMPLE_RADIAL bundle-adjustment oracle (`oracle/bundle_radial.py`) against central differences,
a dense damped Hessian with pinned rows and the pinhole oracle; the undistortion oracle (`oracle/camera.py`); the camera helpers
and every new argument rule of `bundle_adjust` and `undistort_graph` (raised before any device work); `planted_cameras` with
SIMPLE_RADIAL truth and the spread geometry."""
import numpy as np
import pytest
import torch

from oracle import bundle_radial as orad
from oracle.bundle import bundle_adjust as oracle_ba
from oracle.camera import distort, undistort, undistort_graph_keypoints
from oracle.match_graph import consolidate
from oracle.tracks import tracks as oracle_tracks
from oracle.triangulate import triangulate
from roma_b200 import bundle as rb_ba, cabi, camera, synthetic
from roma_b200.match_graph import MatchGraph
from roma_b200.tracks import Tracks
from roma_b200.triangulate import Points3D


def radial_scene(seed, N, points, size=(384, 512), k=(-0.05, 0.05), spread=True, ferr=0.03):
    """A SIMPLE_RADIAL scene in numpy: the graph, tracks and a triangulation with the perturbed cameras and a prior whose f is off by
    up to `ferr` (k = 0), on undistorted keypoints; the keypoints of the graph stay raw."""
    pairs, m, c, sizes, views, intr, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, radial=k, spread=spread)
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy())
    tr = oracle_tracks(pairs.numpy(), g)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
    rng = np.random.default_rng(seed)
    prior = intr.numpy().copy()
    prior[:, 0] *= 1 + rng.uniform(-ferr, ferr, N)
    prior[:, 3] = 0.0
    tri = triangulate(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], camera.pinhole_K(prior), R1.numpy(),
                      t1.numpy(), max_error=20.0)
    return g, tr, tri, prior, R1.numpy(), t1.numpy(), intr.numpy()


# ---- the model and its Jacobian -------------------------------------------------------------------------------------------
def test_jacobian_matches_central_differences():
    rng = np.random.default_rng(0)
    M = 40
    intr = np.c_[rng.uniform(400, 700, M), rng.uniform(200, 300, M), rng.uniform(150, 250, M), rng.uniform(-0.2, 0.2, M)]
    R = orad.rodrigues(rng.normal(scale=0.3, size=(M, 3)))
    t = rng.normal(size=(M, 3)) + np.array([0, 0, 6.0])
    X = rng.normal(size=(M, 3))
    u, _, Jc, JX = orad.project(intr, R, t, X, True)
    h = 1e-6
    for j in range(8):
        dp, dm = [np.zeros((M, 8)) for _ in range(2)]
        dp[:, j], dm[:, j] = h, -h

        def at(d):
            i2 = intr.copy()
            i2[:, 0] += d[:, 6]
            i2[:, 3] += d[:, 7]
            return orad.project(i2, orad.rodrigues(d[:, :3]) @ R, t + d[:, 3:6], X, False)[0]
        num = (at(dp) - at(dm)) / (2 * h)
        assert np.abs(num - Jc[:, :, j]).max() <= 1e-6 * (1 + np.abs(Jc[:, :, j]).max()), j
    for j in range(3):
        d = np.zeros(3)
        d[j] = h
        num = (orad.project(intr, R, t, X + d, False)[0] - orad.project(intr, R, t, X - d, False)[0]) / (2 * h)
        assert np.abs(num - JX[:, :, j]).max() <= 1e-6 * (1 + np.abs(JX).max()), j


def test_system_equals_the_dense_schur_complement_with_pinned_rows():
    g, tr, tri, prior, R, t, _ = radial_scene(1, 4, 120)
    # camera 0: fixed pose with free intrinsics; camera 2: fixed intrinsics; camera 1: fixed t_x; camera 3: fully free
    kw = dict(fixed_poses=(0,), fixed_tx=(1,), fixed_intrinsics=(2,))
    systems = ["dense"]
    orad.bundle_adjust(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"], prior, R, t,
                       max_iterations=1, systems=systems, **kw)
    s = systems[0]
    N, T = 4, tri["ok"].size
    pin = orad.pins(N, **kw)
    H, gr = s["H"], s["g"]
    ok = np.flatnonzero(tri["ok"])
    pts_idx = np.concatenate([8 * N + 3 * k + np.arange(3) for k in ok])
    cam_idx = np.arange(8 * N)
    Hcc, Hcp, Hpp = H[np.ix_(cam_idx, cam_idx)], H[np.ix_(cam_idx, pts_idx)], H[np.ix_(pts_idx, pts_idx)]
    Sd = Hcc - Hcp @ np.linalg.solve(Hpp, Hcp.T)
    bd = -gr[cam_idx] + Hcp @ np.linalg.solve(Hpp, gr[pts_idx])
    for j in np.flatnonzero(pin.reshape(-1)):
        Sd[j, :] = Sd[:, j] = 0.0
        Sd[j, j] = 1.0
        bd[j] = 0.0
    assert s["free"] == [0, 1, 2, 3]
    scale = np.abs(s["S"]).max()
    assert np.abs(np.tril(s["S"]) - np.tril(Sd)).max() <= 1e-12 * scale
    assert np.abs(s["b"] - bd).max() <= 1e-12 * np.abs(bd).max()
    assert (s["dc"].reshape(N, 8)[pin] == 0).all()


def test_pinned_intrinsics_with_k_zero_equal_the_pinhole_oracle():
    g, tr, tri, prior, R, t, _ = radial_scene(2, 4, 150)
    args = (g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"])
    a = orad.bundle_adjust(*args, prior, R, t, refine_focal_length=False, refine_extra_params=False, max_iterations=20)
    b = oracle_ba(*args, camera.pinhole_K(prior), R, t, max_iterations=20)
    assert (a["accepted"] == b["accepted"]).all()
    assert np.abs(a["cost"] - b["cost"]).max() <= 1e-9 * b["cost"][0]
    assert np.abs(a["R"] - b["R"]).max() < 1e-9 and np.abs(a["t"] - b["t"]).max() < 1e-9
    assert (a["intrinsics"] == prior).all()


def test_oracle_recovers_focal_length_and_distortion():
    g, tr, tri, prior, R, t, truth = radial_scene(3, 8, 400)
    res = orad.bundle_adjust(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"], prior,
                             R, t, max_iterations=100, function_tolerance=1e-12)
    ferr = np.abs(res["intrinsics"][:, 0] / truth[:, 0] - 1)
    kerr = np.abs(res["intrinsics"][:, 3] - truth[:, 3])
    print(f"prior f error {np.abs(prior[:, 0] / truth[:, 0] - 1).max():.4f} -> {ferr.max():.5f}, k error -> {kerr.max():.5f}")
    assert np.median(ferr) < 0.5 * np.median(np.abs(prior[:, 0] / truth[:, 0] - 1))
    assert ferr.max() < 0.02 and kerr.max() < 0.02


# ---- undistortion -----------------------------------------------------------------------------------------------------------
def _grid(f=500.0, cx=256.0, cy=192.0, n=41):
    x, y = np.meshgrid(np.linspace(-2 * cx, 4 * cx, n), np.linspace(-2 * cy, 4 * cy, n))
    return np.c_[x.ravel(), y.ravel()].astype(np.float32)


@pytest.mark.parametrize("k", [-0.3, -0.05, -0.01, 0.01, 0.05, 0.3])
def test_undistort_round_trip_and_monotone_newton(k):
    kp = _grid()
    c = np.tile([500.0, 256.0, 192.0, k], (kp.shape[0], 1))
    hist = []
    out, clamp = undistort(kp, c, hist)
    assert np.isfinite(out).all()
    # the round trip in float64 (before the fp32 store): distort(undistort(x)) = x to 1e-9 px
    h = hist[0]
    last = np.where(np.isnan(h), -np.inf, np.arange(h.shape[0])[:, None]).argmax(0)
    rho = h[last, np.arange(h.shape[1])]
    dx, dy = kp[:, 0].astype(np.float64) - 256.0, kp[:, 1].astype(np.float64) - 192.0
    rd = np.hypot(dx, dy) / 500.0
    live = ~clamp & (rd > 0)
    s = rho[live] / rd[live]
    und = np.c_[256.0 + dx[live] * s, 192.0 + dy[live] * s]
    back = distort(und, c[live])
    assert np.abs(back - kp[live].astype(np.float64)).max() <= 1e-9
    # monotone: every live keypoint's iterates move in one direction (down for k > 0, up for k < 0), up to the rounding of the
    # last iterates, which wander by a few ulp around the root
    steps = np.diff(h[:, live], axis=0)
    back_steps = np.where(np.isnan(steps), 0.0, steps if k > 0 else -steps)
    assert (back_steps <= 8 * np.finfo(np.float64).eps * np.nan_to_num(h[1:, live], nan=1.0)).all()
    assert (np.nan_to_num(h[1:, live] - h[:1, live]) * np.sign(k) <= 8 * np.finfo(np.float64).eps * h[:1, live]).all()
    if k < 0:
        turn = 2.0 / (3.0 * np.sqrt(-3.0 * k))
        assert (clamp == (rd >= turn)).all() and (clamp.any() or rd.max() < turn)
        r_out = np.hypot(out[clamp, 0] - 256.0, out[clamp, 1] - 192.0) / 500.0
        assert np.allclose(r_out, 1.0 / np.sqrt(-3.0 * k), rtol=1e-6)
    else:
        assert not clamp.any()


def test_undistort_clamps_at_and_beyond_the_turning_point():
    k = -0.1
    turn = 2.0 / (3.0 * np.sqrt(-3.0 * k))
    r = np.array([0.5 * turn, np.nextafter(turn, 0), turn, 1.5 * turn])
    kp = np.c_[100.0 + 400.0 * r, np.full(4, 50.0)].astype(np.float32)
    c = np.tile([400.0, 100.0, 50.0, k], (4, 1))
    rd = (kp[:, 0].astype(np.float64) - 100.0) / 400.0
    out, clamp = undistort(kp, c)
    assert (clamp == (rd >= turn)).all() and clamp[-1] and not clamp[0]
    assert undistort_graph_keypoints(np.asarray([0, 4]), kp, c[:1])[1] == int(clamp.sum())


def test_undistort_with_k_zero_is_the_identity():
    kp = _grid()
    out, clamp = undistort(kp, np.tile([500.0, 256.0, 192.0, 0.0], (kp.shape[0], 1)))
    assert out.tobytes() == kp.tobytes() and not clamp.any()


# ---- camera helpers and argument rules ----------------------------------------------------------------------------------
def test_default_intrinsics_and_pinhole_K():
    d = camera.default_intrinsics(torch.tensor([[768, 1024], [1200, 900]]))
    assert d.dtype == np.float64 and (d == np.array([[1228.8, 512.0, 384.0, 0.0], [1440.0, 450.0, 600.0, 0.0]])).all()
    K = camera.pinhole_K(d)
    assert (K[1] == np.array([[1440.0, 0, 450.0], [0, 1440.0, 600.0], [0, 0, 1]])).all()
    Kt = camera.pinhole_K(torch.from_numpy(d))
    assert isinstance(Kt, torch.Tensor) and (Kt.numpy() == K).all()
    for bad in ([[768]], [[0, 10]], np.zeros((0, 2))):
        with pytest.raises(ValueError, match="default_intrinsics"):
            camera.default_intrinsics(bad)


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


INTR = np.array([[500.0, 320.0, 240.0, 0.01], [510.0, 320.0, 240.0, -0.02]])


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case", [
    dict(camera_model="OPENCV"), dict(camera_model=1), dict(refine_focal_length=1), dict(refine_extra_params=None),
    dict(fixed_intrinsics=(2,)), dict(fixed_intrinsics=(True,)), dict(fixed_intrinsics=5),
    dict(K=INTR[:, :3]), dict(K=np.repeat(INTR[None], 2, 0)), dict(K=INTR.astype(np.int64)),
    dict(K=INTR * np.array([[-1.0, 1, 1, 1]])), dict(K=INTR * np.array([[0.0, 1, 1, 1]])), dict(K=INTR + np.array([[0, 0, np.nan, 0]])),
    dict(camera_model="PINHOLE", fixed_intrinsics=(0,)), dict(camera_model="PINHOLE"),    # PINHOLE takes K [N, 3, 3]
    dict(workspace_bytes=100),
    {},                                                                               # CPU tensors: the call runs on a CUDA device only
])
def test_bundle_argument_errors_before_device_work(no_device, case):
    kw = dict(graph=mg(), tracks=tk(), points=pts(), K=INTR, R=np.repeat(np.eye(3)[None], 2, 0), t=np.zeros((2, 3)),
              camera_model="SIMPLE_RADIAL")
    kw.update(case)
    with pytest.raises(ValueError) as e:
        rb_ba.bundle_adjust(kw.pop("graph"), kw.pop("tracks"), kw.pop("points"), kw.pop("K"), kw.pop("R"), kw.pop("t"), **kw)
    assert ("CUDA device" in str(e.value)) == (not case), str(e.value)
    assert str(e.value).startswith("bundle_adjust: ")


@pytest.mark.parametrize("case", [dict(graph=None), dict(intrinsics=INTR[:1]), dict(intrinsics=INTR[:, :3]),
                                  dict(intrinsics=INTR * np.array([[0.0, 1, 1, 1]])), dict(intrinsics=INTR.astype(np.int32)),
                                  dict(intrinsics=INTR + np.array([[np.inf, 0, 0, 0]])), {}])
def test_undistort_argument_errors_before_device_work(no_device, case):
    kw = dict(graph=mg(), intrinsics=INTR)
    kw.update(case)
    with pytest.raises(ValueError, match="undistort_keypoints: ") as e:
        camera.undistort_graph(kw["graph"], kw["intrinsics"])
    assert ("CUDA device" in str(e.value)) == (not case), str(e.value)


def test_workspace_formula_equals_the_buffers():
    for N, F, T, E in ((1, 1, 1, 1), (3, 3, 10, 25), (16, 15, 1000, 4097), (50, 50, 40000, 1 << 20)):
        b = rb_ba._buffers("meta", N, F, T, E, 1)
        assert sum(v.numel() * v.element_size() for v in b.values()) == rb_ba.workspace_bytes(N, F, T, E, "SIMPLE_RADIAL"), (N, F, T, E)
    assert rb_ba.workspace_bytes(200, 200, 40000, 4_000_000, "SIMPLE_RADIAL") < rb_ba.WORKSPACE_BYTES


def test_free_cameras_and_pins():
    free, pins = rb_ba._free_and_pins(4, [0], [1], True, True, True, [2])
    assert free == [0, 1, 2, 3]
    assert (pins == orad.pins(4, (0,), (1,), True, True, (2,))).all()
    free, pins = rb_ba._free_and_pins(3, [0, 1], [], True, False, True, [0])
    assert free == [1, 2] and pins[0].tolist() == [1] * 7 + [0]
    free, _ = rb_ba._free_and_pins(3, [0], [], False, True, True, [])
    assert free == [1, 2]


def test_entry_points_and_exports():
    import roma_b200
    assert {"romab200_undistort_keypoints"} <= set(cabi.FUNCTIONS)
    assert roma_b200.undistort_graph is camera.undistort_graph and roma_b200.default_intrinsics is camera.default_intrinsics
    assert roma_b200.pinhole_K is camera.pinhole_K
    assert [f for f, _ in cabi.STRUCT_FIELDS["rb_ba_args"][-2:]] == ["camera_model", "pin"]
    assert cabi.RB_BA_CAM1 == 16
    assert rb_ba.BundleResult.__dataclass_fields__["intrinsics"].default is None


# ---- synthetic scenes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spread", [False, True])
def test_radial_observations_reproject_within_the_noise(spread):
    H, W = 384, 512
    pairs, m, c, sizes, views, intr, R, t, X = synthetic.planted_cameras(4, 6, 400, size=(H, W), radial=(-0.05, 0.05), spread=spread,
                                                                         noise=0.5)
    intr, R, t, X, v = intr.numpy(), R.numpy(), t.numpy(), X.numpy(), views.numpy()
    assert intr.shape == (6, 4) and (intr[:, 1] == W / 2).all() and (intr[:, 2] == H / 2).all() and (np.abs(intr[:, 3]) <= 0.05).all()
    p, i = np.nonzero(v >= 0)
    u = orad.project(intr[i], R[i], t[i], X[p], False)[0]
    cell = np.c_[v[p, i] % W + 0.5, v[p, i] // W + 0.5]             # cell_size 1: the observation lies in this pixel
    err = np.abs(u - cell).max(1)
    assert np.quantile(err, 0.99) < 0.5 + 4 * 0.5 and np.median(err) < 1.0
    # the same seed without the options: the same points and visibility draws, other cameras only where spread moves them
    base = synthetic.planted_cameras(4, 6, 400, size=(H, W))
    assert torch.equal(base[8], torch.from_numpy(X))
    if not spread:
        assert torch.equal(base[6], torch.from_numpy(R))


# ---- reconstruct with intrinsics and the SIMPLE_RADIAL COLMAP model -------------------------------------------------------------
def test_colmap_writer_round_trip_with_simple_radial(tmp_path):
    from roma_b200 import mapper
    from test_mapper_host import _hand_built, _parse, _quat_to_R
    recon, graph, tracks, K, sizes = _hand_built(1)
    N = K.shape[0]
    intr = np.c_[K[:, 0, 0], K[:, 0, 2], K[:, 1, 2], np.linspace(-0.04, 0.05, N)]
    recon = mapper.Reconstruction(recon.registered, recon.R, recon.t, recon.points, None, [], "all_registered", torch.from_numpy(intr))
    mapper.write_colmap_text(tmp_path, recon, graph, tracks, None, sizes)
    cams, images, pts = _parse(tmp_path)
    for i in range(N):
        c = cams[i + 1]
        assert c[1] == "SIMPLE_RADIAL" and (int(c[2]), int(c[3])) == (sizes[i][1], sizes[i][0])
        assert [float(v) for v in c[4:]] == intr[i].tolist()                       # 17 digits: exact
    kp_off, kps = graph.kp_offsets.numpy(), graph.keypoints.numpy().astype(np.float64)
    for iid, (h, p2d) in images.items():
        trip = np.array(p2d, dtype=object).reshape(-1, 3)
        assert np.array_equal(trip[:, :2].astype(float), kps[kp_off[iid - 1]:kp_off[iid]])   # raw keypoints
        assert np.abs(_quat_to_R(np.array(h[1:5], float)) - recon.R[iid - 1].numpy()).max() <= 1e-12
    assert sorted(pts) == [k + 1 for k in np.flatnonzero(recon.points.ok.numpy())]
    for pid, r in pts.items():
        assert float(r[7]) == float(recon.points.error[pid - 1]) and np.array_equal(np.array(r[1:4], float), recon.points.X[pid - 1].numpy())
    bad = mapper.Reconstruction(recon.registered, recon.R, recon.t, recon.points, None, [], "all_registered",
                                torch.from_numpy(intr * np.array([0.0, 1, 1, 1])))
    with pytest.raises(ValueError, match="write_colmap_text"):
        mapper.write_colmap_text(tmp_path / "b", bad, graph, tracks, None, sizes)


@pytest.mark.parametrize("kw, msg", [
    (dict(intrinsics=INTR, K=np.tile(np.eye(3), (2, 1, 1))), "K=None"), (dict(intrinsics=INTR[:1]), "intrinsics"),
    (dict(intrinsics=INTR * np.array([[0.0, 1, 1, 1]])), "focal"), (dict(intrinsics=INTR.astype(np.int64)), "float"),
    (dict(intrinsics=INTR, refine_intrinsics=1), "refine_intrinsics"), (dict(refine_intrinsics=True), "needs intrinsics"),
    (dict(intrinsics=INTR, abs_max_error=0.0), "abs_max_error"), (dict(intrinsics=INTR, init_num_candidates=0), "reconstruct: "),
    (dict(intrinsics=INTR, refine_intrinsics=True), "CUDA device")])
def test_reconstruct_intrinsics_arguments_before_device_work(no_device, kw, msg):
    from roma_b200 import mapper
    kp = torch.zeros(6, 2)
    g = MatchGraph(torch.tensor([0, 3, 6]), kp, torch.ones(6), torch.tensor([0, 3]), torch.tensor([[0, 0], [1, 1], [2, 2]], dtype=torch.int32),
                   torch.ones(3))
    tr = Tracks(torch.tensor([0]), torch.zeros(0, 2, dtype=torch.int32), torch.full((6,), -1, dtype=torch.int32), 0)
    kw = dict(kw)
    K = kw.pop("K", np.tile(np.eye(3), (2, 1, 1)) if "intrinsics" not in kw else None)
    with pytest.raises(ValueError, match=msg):
        mapper.reconstruct([(0, 1)], g, tr, K, **kw)
