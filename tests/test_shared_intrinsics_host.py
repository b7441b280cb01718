"""Shared cameras (`camera_ids`) on the host: `oracle/bundle_shared.py` (its Jacobian in the shared parameters against central
differences, its reduced system against P^T (dense damped Hessian) P with pins, its summation scale S'_abs against P^T S_abs P from
a dense Jacobian written out over |term|, singleton groups against oracle/bundle_radial.py),
the argument rules of `bundle_adjust` and `reconstruct`, the group layout and workspace formula, `write_colmap_text` with one
camera per group, and `planted_cameras(camera_ids=...)` leaving existing calls unchanged."""
import numpy as np
import pytest
import torch

from oracle import bundle_radial as orad
from oracle import bundle_shared as osh
from oracle.match_graph import consolidate
from oracle.tracks import tracks as oracle_tracks
from oracle.triangulate import triangulate
from roma_b200 import bundle as rb_ba, cabi, camera, synthetic
from roma_b200.match_graph import MatchGraph
from roma_b200.tracks import Tracks
from roma_b200.triangulate import Points3D


def shared_scene(seed, ids, points, size=(384, 512), spread=True, ferr=0.03):
    """A planted SIMPLE_RADIAL scene with shared cameras `ids`, in numpy: graph, tracks, a triangulation with perturbed cameras,
    and a prior whose f is off by up to `ferr` per group (k = 0), equal within each group."""
    ids = np.asarray(ids)
    N = ids.size
    pairs, m, c, sizes, views, intr, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, radial=(-0.05, 0.05), spread=spread,
                                                                         camera_ids=ids)
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy())
    tr = oracle_tracks(pairs.numpy(), g)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
    rng = np.random.default_rng(seed)
    prior = intr.numpy().copy()
    prior[:, 0] *= 1 + rng.uniform(-ferr, ferr, ids.max() + 1)[ids]
    prior[:, 3] = 0.0
    tri = triangulate(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], camera.pinhole_K(prior), R1.numpy(),
                      t1.numpy(), max_error=20.0)
    return g, tr, tri, prior, R1.numpy(), t1.numpy(), intr.numpy()


def _args(g, tr, tri):
    return g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], tri["X"], tri["ok"], tri["inlier"]


# ---- the oracle ---------------------------------------------------------------------------------------------------------------
def test_shared_jacobian_matches_central_differences():
    """The oracle's gradient J'^T r in the shared parameters (the pose of each camera, (f, k) per group; squared loss, nothing
    pinned) against central differences of the cost: J' is built directly in those parameters."""
    ids = np.array([0, 0, 1, 1, 1])
    g, tr, tri, prior, R, t, _ = shared_scene(5, ids, 120)
    args = _args(g, tr, tri)
    kw = dict(fixed_poses=(), fixed_tx=())
    systems = []
    osh.bundle_adjust(*args, prior, R, t, ids, max_iterations=1, systems=systems, **kw)
    s = systems[0]
    assert s["free"] == list(range(5)) and s["groups"] == [0, 1]
    N = ids.size
    from oracle.bundle_radial import track_costs

    def cost(d):
        intr = prior.copy()
        intr[:, 0] += d[30 + 2 * ids]
        intr[:, 3] += d[31 + 2 * ids]
        R1 = orad.rodrigues(d[:30].reshape(N, 6)[:, :3]) @ R
        t1 = t + d[:30].reshape(N, 6)[:, 3:]
        return track_costs(*args, intr, R1, t1).sum()

    h = np.r_[np.full(30, 1e-7), np.tile([1e-4, 1e-7], 2)]
    num = np.zeros(34)
    for j in range(34):
        e = np.zeros(34)
        e[j] = h[j]
        num[j] = (cost(e) - cost(-e)) / (2 * h[j])
    # the oracle's plain gradient g = sum w J'^T r (J' built in the shared parameters)
    gc = s["gc"]
    assert np.abs(num - gc).max() <= 1e-5 * np.abs(gc).max(), np.abs(num - gc).max() / np.abs(gc).max()


def _P(ids, free, groups, N, T):
    """P [8N + 3T, n' + 3T]: camera i's pose rows to its free index's, its f, k to its group's; the points unchanged."""
    F, G = len(free), len(groups)
    n = 6 * F + 2 * G
    P = np.zeros((8 * N + 3 * T, n + 3 * T))
    for fi, i in enumerate(free):
        P[8 * i + np.arange(6), 6 * fi + np.arange(6)] = 1.0
        gl = groups.index(ids[i])
        P[8 * i + 6 + np.arange(2), 6 * F + 2 * gl + np.arange(2)] = 1.0
    P[8 * N + np.arange(3 * T), n + np.arange(3 * T)] = 1.0
    return P


@pytest.mark.parametrize("ids, gauge", [
    ([0, 0, 1, 1, 1, 2], dict(fixed_poses=(0,), fixed_tx=(1,))),
    ([0, 0, 1, 1, 1, 2], dict(fixed_poses=(0, 4), fixed_tx=(2,), fixed_intrinsics=(2,))),
    ([0, 1, 0, 1, 0, 1], dict(fixed_poses=(0, 1, 2), fixed_tx=(), refine_extra_params=False)),
])
def test_reduced_system_equals_the_folded_dense_hessian(ids, gauge):
    """The oracle's S', b' against the Schur complement of P^T (H + lambda D) P from oracle/bundle_radial.py's dense per-image
    Hessian, with the pinned rows set to the identity.  P^T D P sums the members' clamped diagonals, which is rule 5''."""
    ids = np.asarray(ids)
    g, tr, tri, prior, R, t, _ = shared_scene(6, ids, 150)
    args = _args(g, tr, tri)
    N, T = ids.size, tri["ok"].size
    systems = []
    osh.bundle_adjust(*args, prior, R, t, ids, max_iterations=1, systems=systems, **gauge)
    s = systems[0]
    dense = ["dense"]
    gk = {k: v for k, v in gauge.items() if k != "fixed_intrinsics"}
    fin_imgs = [i for i in range(N) if ids[i] in gauge.get("fixed_intrinsics", ())]
    orad.bundle_adjust(*args, prior, R, t, max_iterations=1, systems=dense, fixed_intrinsics=fin_imgs, **gk)
    H, gr = dense[0]["H"], dense[0]["g"]
    P = _P(ids, s["free"], s["groups"], N, T)
    Hs, gs = P.T @ H @ P, P.T @ gr
    n = 6 * len(s["free"]) + 2 * len(s["groups"])
    ok = np.flatnonzero(tri["ok"])
    pi = np.concatenate([n + 3 * k + np.arange(3) for k in ok])
    ci = np.arange(n)
    Hcc, Hcp, Hpp = Hs[np.ix_(ci, ci)], Hs[np.ix_(ci, pi)], Hs[np.ix_(pi, pi)]
    Sd = Hcc - Hcp @ np.linalg.solve(Hpp, Hcp.T)
    bd = -gs[ci] + Hcp @ np.linalg.solve(Hpp, gs[pi])
    pose_pin, group_pin, free, groups = osh.layout(ids, **gauge)
    pinned = np.r_[pose_pin[free].reshape(-1), group_pin[groups].reshape(-1)]
    for j in np.flatnonzero(pinned):
        Sd[j, :] = Sd[:, j] = 0.0
        Sd[j, j] = 1.0
        bd[j] = 0.0
    scale = np.abs(s["S"]).max()
    assert np.abs(s["S"] - Sd).max() <= 1e-10 * scale, np.abs(s["S"] - Sd).max() / scale
    assert np.abs(s["b"] - bd).max() <= 1e-10 * np.abs(bd).max()
    assert (s["d"][pinned] == 0).all()


def _close_scale(a, ref, rtol=1e-12):
    """Two sums of the same nonnegative terms in different orders: equal to rtol of each entry (0 where ref is 0)."""
    assert a.shape == ref.shape and (a >= 0).all() and (ref >= 0).all()
    assert (np.abs(a - ref) <= rtol * ref).all(), np.max(np.abs(a - ref) / np.where(ref > 0, ref, 1.0))


@pytest.mark.parametrize("ids, loss_scale, gauge", [
    ([0, 0, 1, 1, 1, 2], None, dict(fixed_poses=(0,), fixed_tx=(1,))),
    ([0, 0, 1, 1, 1, 2], 1.0, dict(fixed_poses=(0, 4), fixed_tx=(2,), fixed_intrinsics=(2,))),
    ([0, 1, 0, 1, 0, 1], None, dict(fixed_poses=(0, 1, 2), fixed_tx=(), refine_extra_params=False)),
])
def test_summation_scale_is_the_folded_per_image_scale(ids, loss_scale, gauge):
    """The oracle's S'_abs and b'_abs bound |S'| and |b'| entry by entry, and equal P^T S_abs P and P^T b_abs, where S_abs and b_abs
    are assembled here over |term| from an explicit dense Jacobian in the per-image parameters (8 per camera, then 3 per track)."""
    ids = np.asarray(ids)
    g, tr, tri, prior, R, t, _ = shared_scene(6, ids, 150)
    args = _args(g, tr, tri)
    N, T = ids.size, tri["ok"].size
    systems = []
    osh.bundle_adjust(*args, prior, R, t, ids, max_iterations=1, loss_scale=loss_scale, systems=systems, **gauge)
    s = systems[0]
    pose_pin, group_pin, free, groups = osh.layout(ids, **gauge)
    pinned = np.r_[pose_pin[free].reshape(-1), group_pin[groups].reshape(-1)]
    # a pinned row is e_r in S' and 0 in S'_abs: no rounding reaches it
    keep = ~pinned
    assert (np.abs(s["S"])[np.ix_(keep, keep)] <= s["S_abs"][np.ix_(keep, keep)]).all() and (np.abs(s["b"])[keep] <= s["b_abs"][keep]).all()
    # every used observation's Jacobian in the per-image parameters, written out densely
    kpo, xy = np.asarray(g["kp_offsets"], np.int64), np.asarray(g["keypoints"], np.float64)
    off, el = np.asarray(tr["track_offsets"], np.int64), np.asarray(tr["elements"], np.int64).reshape(-1, 2)
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(np.asarray(tri["ok"], bool), np.diff(off)) & np.asarray(tri["inlier"], bool))
    img, trk = el[e, 0], track[e]
    X = np.asarray(tri["X"], np.float64)
    u, _, Jc, JX = orad.project(prior[img], R[img], t[img], X[trk], True)
    r = u - xy[kpo[img] + el[e, 1]]
    c2 = 0.0 if loss_scale is None else loss_scale ** 2
    w = 1.0 / (1.0 + (r * r).sum(1) / c2) if c2 else np.ones(e.size)
    nc, lam = 8 * N, s["lam"]
    J = np.zeros((e.size, 2, nc + 3 * T))
    for q in range(e.size):
        J[q, :, 8 * img[q]:8 * img[q] + 8] = Jc[q]
        J[q, :, nc + 3 * trk[q]:nc + 3 * trk[q] + 3] = JX[q]
    H = np.einsum("m,mai,maj->ij", w, J, J)
    Habs = np.einsum("m,mai,maj->ij", w, np.abs(J), np.abs(J))
    gabs = np.einsum("m,mai,ma->i", w, np.abs(J), np.abs(r))
    Dc = np.clip(np.diag(H)[:nc], 1e-6, 1e32)
    S_abs, b_abs = Habs[:nc, :nc] + lam * np.diag(Dc), gabs[:nc].copy()
    for k in np.unique(trk):
        p = nc + 3 * k + np.arange(3)
        Vk = H[np.ix_(p, p)]
        Vinv = np.abs(np.linalg.inv(Vk + lam * np.diag(np.clip(np.diag(Vk), 1e-6, 1e32))))
        S_abs += Habs[:nc, p] @ Vinv @ Habs[p, :nc]
        b_abs += Habs[:nc, p] @ Vinv @ gabs[p]
    n = 6 * len(s["free"]) + 2 * len(s["groups"])
    P = _P(ids, s["free"], s["groups"], N, T)[:nc, :n]
    S_ref, b_ref = P.T @ S_abs @ P, P.T @ b_abs
    S_ref[pinned, :] = S_ref[:, pinned] = b_ref[pinned] = 0.0
    _close_scale(s["S_abs"], S_ref)
    _close_scale(s["b_abs"], b_ref)


@pytest.mark.parametrize("seed, N, loss_scale, gauge", [(7, 4, None, {}), (8, 6, 1.0, dict(fixed_poses=(0, 3), fixed_intrinsics=(2,)))])
def test_singleton_groups_equal_the_per_image_oracle(seed, N, loss_scale, gauge):
    g, tr, tri, prior, R, t, _ = shared_scene(seed, np.arange(N), 150)
    args = _args(g, tr, tri)
    kw = dict(loss_scale=loss_scale, max_iterations=8, **gauge)
    a = osh.bundle_adjust(*args, prior, R, t, np.arange(N), **kw)
    b = orad.bundle_adjust(*args, prior, R, t, **kw)
    assert (a["accepted"] == b["accepted"]).all() and a["termination"] == b["termination"]
    assert np.abs(a["cost"] - b["cost"]).max() <= 1e-10 * b["cost"][0]
    for name in ("R", "t", "intrinsics", "X"):
        assert np.abs(a[name] - b[name]).max() <= 1e-10 * max(1.0, np.abs(b[name]).max()), name


@pytest.mark.parametrize("seed, N, loss_scale, gauge", [(7, 4, None, {}), (8, 6, 1.0, dict(fixed_poses=(0, 3), fixed_intrinsics=(2,)))])
def test_singleton_groups_summation_scale_equals_the_per_image_one(seed, N, loss_scale, gauge):
    """With singleton groups, S'_abs and b'_abs are oracle/bundle_radial.py's S_abs and b_abs with the rows in the order (poses, then
    groups)."""
    g, tr, tri, prior, R, t, _ = shared_scene(seed, np.arange(N), 150)
    args = _args(g, tr, tri)
    sa, sb = [], []
    osh.bundle_adjust(*args, prior, R, t, np.arange(N), loss_scale=loss_scale, max_iterations=1, systems=sa, **gauge)
    orad.bundle_adjust(*args, prior, R, t, loss_scale=loss_scale, max_iterations=1, systems=sb, **gauge)
    F = len(sa[0]["free"])
    assert sa[0]["free"] == sb[0]["free"] and sa[0]["groups"] == sa[0]["free"]
    perm = np.r_[(8 * np.arange(F)[:, None] + np.arange(6)).reshape(-1), (8 * np.arange(F)[:, None] + np.arange(6, 8)).reshape(-1)]
    _close_scale(sa[0]["S_abs"], sb[0]["S_abs"][np.ix_(perm, perm)])
    _close_scale(sa[0]["b_abs"], sb[0]["b_abs"][perm])


def test_shared_groups_stay_equal_and_fit_a_single_camera_scene():
    ids = np.zeros(6, np.int64)
    g, tr, tri, prior, R, t, truth = shared_scene(9, ids, 300)
    res = osh.bundle_adjust(*_args(g, tr, tri), prior, R, t, ids, max_iterations=60, function_tolerance=1e-12)
    intr = res["intrinsics"]
    assert (intr == intr[0]).all()
    assert res["cost"][-1] < res["cost"][0]
    ferr = abs(intr[0, 0] / truth[0, 0] - 1)
    print(f"single camera: prior f error {abs(prior[0, 0] / truth[0, 0] - 1):.4f} -> {ferr:.2e}, k {intr[0, 3]:.5f} vs {truth[0, 3]:.5f}")
    assert ferr < 2e-3 and abs(intr[0, 3] - truth[0, 3]) < 5e-3


# ---- host rules of bundle_adjust ---------------------------------------------------------------------------------------------
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


INTR = np.array([[500.0, 320.0, 240.0, 0.01], [500.0, 320.0, 240.0, 0.01]])


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case, msg", [
    (dict(camera_ids=[0, 0], camera_model="PINHOLE", K=np.tile(np.eye(3), (2, 1, 1))), "needs camera_model"),
    (dict(camera_ids=[0, 0, 0]), "integer array"), (dict(camera_ids=[0.0, 0.0]), "integer array"),
    (dict(camera_ids=[True, False]), "integer array"), (dict(camera_ids=[-1, 0]), ">= 0"),
    (dict(camera_ids=[0, 0], K=INTR * np.array([[1.0, 1, 1, 1], [1 + 1e-16 * 4, 1, 1, 1]])), "intrinsics differ"),
    (dict(camera_ids=[0, 0], K=INTR + np.array([[0, 0, 0, 0], [0, 0, 0, 1e-3]])), "intrinsics differ"),
    (dict(camera_ids=[0, 0], fixed_intrinsics=(1,)), "fixed_intrinsics"),
    (dict(camera_ids=[0, 1], fixed_intrinsics=(2,)), "fixed_intrinsics"),
    (dict(camera_ids=[0, 0], workspace_bytes=1000), "workspace"),
    (dict(camera_ids=np.array([0, 0])), "CUDA device"), (dict(camera_ids=torch.tensor([1, 0]), K=INTR * [[1.0], [1.0]]), "CUDA device"),
])
def test_bundle_camera_ids_errors_before_device_work(no_device, case, msg):
    kw = dict(graph=mg(), tracks=tk(), points=pts(), K=INTR, R=np.repeat(np.eye(3)[None], 2, 0), t=np.zeros((2, 3)),
              camera_model="SIMPLE_RADIAL")
    kw.update(case)
    with pytest.raises(ValueError, match=msg) as e:
        rb_ba.bundle_adjust(kw.pop("graph"), kw.pop("tracks"), kw.pop("points"), kw.pop("K"), kw.pop("R"), kw.pop("t"), **kw)
    assert str(e.value).startswith("bundle_adjust: ")


def test_group_layout_and_pins():
    ids = np.array([2, 0, 2, 1, 0, 2])
    free, pins = rb_ba._free_and_pins(6, [0, 3], [1], True, True, True, [1], ids)
    # image 3 (camera 1, pinned intrinsics) has a fixed pose, so it is not free
    assert free == [0, 1, 2, 4, 5]
    assert [p[6:].tolist() for p in pins] == [[0, 0]] * 5
    groups, off, mem, gp = rb_ba._groups(ids, free, pins)
    assert groups == [0, 2] and off.tolist() == [0, 2, 5] and mem.tolist() == [1, 3, 0, 2, 4] and gp.tolist() == [[0, 0], [0, 0]]
    free, pins = rb_ba._free_and_pins(6, [0], [], True, True, False, [2], ids)
    groups, off, mem, gp = rb_ba._groups(ids, free, pins)
    assert groups == [0, 1, 2] and gp.tolist() == [[0, 1], [0, 1], [1, 1]]
    assert (pins[free.index(2), 6:] == [1, 1]).all()                    # members carry their group's pins
    pose_pin, group_pin, ofree, ogroups = osh.layout(ids, (0,), (), True, False, (2,))
    assert ofree == free and ogroups == groups and (group_pin[groups] == gp.astype(bool)).all()


def test_workspace_formula_equals_the_buffers():
    for N, F, T, E, G in ((1, 1, 1, 1, 1), (3, 3, 10, 25, 2), (16, 15, 1000, 4097, 1), (50, 50, 40000, 1 << 20, 50)):
        b = rb_ba._buffers("meta", N, F, T, E, 1, G)
        assert sum(v.numel() * v.element_size() for v in b.values()) == rb_ba.workspace_bytes(N, F, T, E, "SIMPLE_RADIAL", G), (N, F, T, E)
    assert rb_ba.workspace_bytes(3, 3, 10, 25, "SIMPLE_RADIAL", 0) == rb_ba.workspace_bytes(3, 3, 10, 25, "SIMPLE_RADIAL")
    assert rb_ba.workspace_bytes(200, 200, 40000, 4_000_000, "SIMPLE_RADIAL", 1) < rb_ba.WORKSPACE_BYTES


def test_entry_points_and_exports():
    """The C ABI of the groups path: its own struct, rb_ba_groups_args, and three entry points; rb_ba_args is unchanged."""
    import roma_b200
    assert {"romab200_ba_fold", "romab200_ba_groups_cholesky", "romab200_ba_unfold"} <= set(cabi.FUNCTIONS)
    assert roma_b200.undistort_graph is camera.undistort_graph and roma_b200.default_intrinsics is camera.default_intrinsics
    assert roma_b200.pinhole_K is camera.pinhole_K
    assert [f for f, _ in cabi.STRUCT_FIELDS["rb_ba_args"][-2:]] == ["camera_model", "pin"]
    assert [f for f, _ in cabi.STRUCT_FIELDS["rb_ba_groups_args"]] == ["num_free", "num_groups", "group_offsets", "group_members",
                                                                       "group_pin", "S", "rhs", "S_groups", "rhs_groups", "result"]
    assert cabi.RB_BA_CAM1 == 16
    assert rb_ba.BundleResult.__dataclass_fields__["intrinsics"].default is None
    assert roma_b200.Reconstruction.__dataclass_fields__["camera_ids"].default is None


# ---- reconstruct and the COLMAP model -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, msg", [
    (dict(camera_ids=[0, 0]), "needs intrinsics"),
    (dict(intrinsics=INTR, camera_ids=[0, 0, 0]), "integer array"),
    (dict(intrinsics=INTR * np.array([[1.0, 1, 1, 1], [1.01, 1, 1, 1]]), camera_ids=[0, 0]), "intrinsics differ"),
    (dict(intrinsics=INTR, camera_ids=[0, 0], refine_intrinsics=True), "CUDA device")])
def test_reconstruct_camera_ids_arguments_before_device_work(no_device, kw, msg):
    from roma_b200 import mapper
    kp = torch.zeros(6, 2)
    g = MatchGraph(torch.tensor([0, 3, 6]), kp, torch.ones(6), torch.tensor([0, 3]), torch.tensor([[0, 0], [1, 1], [2, 2]], dtype=torch.int32),
                   torch.ones(3))
    tr = Tracks(torch.tensor([0]), torch.zeros(0, 2, dtype=torch.int32), torch.full((6,), -1, dtype=torch.int32), 0)
    K = None if "intrinsics" in kw else np.tile(np.eye(3), (2, 1, 1))
    with pytest.raises(ValueError, match=msg) as e:
        mapper.reconstruct([(0, 1)], g, tr, K, **kw)
    assert str(e.value).startswith("reconstruct: ")


def test_colmap_writer_with_camera_groups(tmp_path):
    from roma_b200 import mapper
    from test_mapper_host import _hand_built, _parse
    recon, graph, tracks, K, sizes = _hand_built(1)
    N = K.shape[0]
    ids = np.arange(N) % 2
    intr = np.c_[K[:, 0, 0], K[:, 0, 2], K[:, 1, 2], np.linspace(-0.04, 0.05, N)]
    intr = intr[ids]                                      # group rows equal: those of images 0 and 1
    sizes = np.asarray(sizes)[ids]
    base = mapper.Reconstruction(recon.registered, recon.R, recon.t, recon.points, None, [], "all_registered", torch.from_numpy(intr))
    grouped = mapper.Reconstruction(recon.registered, recon.R, recon.t, recon.points, None, [], "all_registered", torch.from_numpy(intr),
                                    torch.from_numpy(ids))
    mapper.write_colmap_text(tmp_path / "a", base, graph, tracks, None, sizes)
    mapper.write_colmap_text(tmp_path / "b", grouped, graph, tracks, None, sizes)
    cams, images, pts = _parse(tmp_path / "b")
    assert sorted(cams) == [1, 2]
    for g in (0, 1):
        c = cams[g + 1]
        assert c[1] == "SIMPLE_RADIAL" and (int(c[2]), int(c[3])) == (sizes[g][1], sizes[g][0])
        assert [float(v) for v in c[4:]] == intr[g].tolist()
    for iid, (h, _) in images.items():
        assert int(h[8]) == ids[iid - 1] + 1
    # images.txt differs only in CAMERA_ID; points3D.txt is the same
    a_cams, a_images, _ = _parse(tmp_path / "a")
    assert sorted(a_cams) == list(range(1, N + 1)) and sorted(a_images) == sorted(images)
    for iid in images:
        ha, pa = a_images[iid]
        hb, pb = images[iid]
        assert ha[:8] + ha[9:] == hb[:8] + hb[9:] and pa == pb
    assert (tmp_path / "a" / "points3D.txt").read_bytes() == (tmp_path / "b" / "points3D.txt").read_bytes()
    bad = mapper.Reconstruction(recon.registered, recon.R, recon.t, recon.points, None, [], "all_registered",
                                torch.from_numpy(intr + np.arange(N)[:, None]), torch.from_numpy(ids))
    with pytest.raises(ValueError, match="write_colmap_text"):
        mapper.write_colmap_text(tmp_path / "c", bad, graph, tracks, None, sizes)


# ---- synthetic scenes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(), dict(radial=(-0.05, 0.05)), dict(radial=(-0.05, 0.05), spread=True), dict(outlier_frac=0.2)])
def test_planted_cameras_without_camera_ids_is_unchanged(kw):
    """Existing calls return the same arrays as the explicit camera_ids=None call; with camera_ids, the group rows are equal and the
    scene (points, poses and, without radial, nothing else) is the same draw."""
    a = synthetic.planted_cameras(3, 6, 300, size=(384, 512), **kw)
    b = synthetic.planted_cameras(3, 6, 300, size=(384, 512), camera_ids=None, **kw)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    ids = np.array([0, 0, 1, 1, 1, 2])
    c = synthetic.planted_cameras(3, 6, 300, size=(384, 512), camera_ids=ids, **kw)
    K = c[5].numpy()
    for g in range(3):
        assert (K[ids == g] == K[np.flatnonzero(ids == g)[0]]).all()
    assert (K[[0, 2, 5]] == a[5].numpy()[[0, 2, 5]])[..., 0].all()   # each group keeps its first image's f
    assert torch.equal(c[6], a[6]) and torch.equal(c[7], a[7]) and torch.equal(c[8], a[8])
