"""Shared cameras (`camera_ids`) on the GPU: `bundle_adjust` against `oracle/bundle_shared.py` (which builds the shared Jacobian
directly and never folds), the folded system entry by entry, singleton groups against the per-image problem, byte-identical reruns
and equal group rows; PINHOLE and per-image SIMPLE_RADIAL outputs byte-identical to the build before shared cameras
(tests/golden/ba_digests.json); `reconstruct(..., camera_ids=...)` against the loop written out with the device stages, and its
recovery of a single camera's f against per-image self-calibration."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import bundle_shared as osh  # noqa: E402
from roma_b200 import build_tracks, bundle_adjust, cabi, consolidate_matches, reconstruct, synthetic, triangulate_tracks  # noqa: E402
from roma_b200 import verify_matches  # noqa: E402
from roma_b200.camera import pinhole_K, undistort_graph  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}
HERE = os.path.dirname(os.path.abspath(__file__))


def _scene(seed, ids, points, cs=1, outlier_frac=0.0, spread=False, ferr=(0.02, 0.05)):
    """Raw graph and tracks of a planted scene with shared cameras `ids`, a prior with each group's f off by ferr (sign random) and
    k = 0, a triangulation under the prior on the undistorted graph, and perturbed poses."""
    ids = np.asarray(ids)
    N, C = ids.size, ids.max() + 1
    pairs, m, c, sizes, views, intr, R, t, X = synthetic.planted_cameras(seed, N, points, size=(384, 512), cell_size=cs,
                                                                         outlier_frac=outlier_frac, radial=(-0.05, 0.05), spread=spread,
                                                                         camera_ids=ids, device=DEV)
    g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    if outlier_frac > 0:
        g = verify_matches(pairs, g, threshold=THR[cs])[0]
    tr = build_tracks(pairs, g)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
    rng = np.random.default_rng(seed)
    prior = intr.cpu().numpy().copy()
    prior[:, 0] *= (1 + rng.choice([-1.0, 1.0], C) * rng.uniform(*ferr, C))[ids]
    prior[:, 3] = 0.0
    pts = triangulate_tracks(undistort_graph(g, prior), tr, pinhole_K(prior), R1, t1, max_error=20.0)
    return g, tr, pts, prior, R1, t1, intr


def _oracle(g, tr, pts, prior, R, t, ids, **kw):
    return osh.bundle_adjust(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.X, pts.ok, pts.inlier, prior, R, t, ids, **kw)


def _close(res, ref, tol):
    """Parameters within tol of the oracle's, relative to each quantity's largest magnitude (at least 1)."""
    for name, a in (("R", res.R), ("t", res.t), ("intrinsics", res.intrinsics), ("X", res.points.X)):
        b = ref[name]
        assert np.abs(a.cpu().numpy() - b).max() <= tol * max(1.0, np.abs(b).max()), (name, np.abs(a.cpu().numpy() - b).max())


CASES = [
    (0, [0, 0, 1, 1, 1, 2], 1, 0.0, None, {}),
    (1, [0, 0, 1, 1, 1, 2], 4, 0.2, 1.0, {}),                                          # the Cauchy loss
    (2, [0, 0, 1, 1, 1, 2], 1, 0.0, None, dict(fixed_intrinsics=(1,))),                # a fixed group
    (3, [0, 1, 0, 1, 0, 1, 0, 1], 1, 0.0, 2.0, dict(fixed_poses=(0, 2, 4, 6))),         # fixed poses with a free group
    (4, [1, 1, 1, 1, 0, 0, 0, 0, 0, 0], 1, 0.2, None, dict(fixed_poses=(0, 5), fixed_tx=(1,), refine_extra_params=False)),
]


@pytest.mark.parametrize("seed, ids, cs, outlier_frac, loss_scale, gauge", CASES)
def test_device_matches_the_oracle(seed, ids, cs, outlier_frac, loss_scale, gauge):
    g, tr, pts, prior, R, t, _ = _scene(seed, ids, 300, cs, outlier_frac)
    kw = dict(loss_scale=loss_scale, max_iterations=10, function_tolerance=0.0, **gauge)
    res = bundle_adjust(g, tr, pts, prior, R, t, camera_model="SIMPLE_RADIAL", camera_ids=ids, **kw)
    ref = _oracle(g, tr, pts, prior, R, t, ids, **kw)
    print(f"ids {ids} {gauge}: F {res.cost[0]:.6g} -> {res.cost[-1]:.10g} ({res.accepted.sum()} of {res.accepted.size} kept); oracle "
          f"{ref['cost'][-1]:.10g}; worst cost difference {np.abs(res.cost - ref['cost']).max() / ref['cost'].max():.1e}")
    # kept/rejected agree up to the first trial whose rho lies within rounding of 1e-3 (near the minimum F - F_new and pred are
    # both at the rounding floor of F); the costs agree at every trial
    tri = ref["trials"]
    for k in range(min(res.accepted.size, len(tri))):
        if abs(tri[k]["margin"]) <= 1e-6 + 1e-10 * tri[k]["F"] / abs(tri[k]["pred"]):
            break
        assert res.accepted[k] == ref["accepted"][k], k
        assert abs(res.pred[k] - tri[k]["pred"]) <= 1e-9 * abs(tri[k]["pred"]), k
    assert res.cost.size == ref["cost"].size and np.abs(res.cost - ref["cost"]).max() <= 1e-9 * ref["cost"].max()
    _close(res, ref, 1e-8)
    intr = res.intrinsics.cpu().numpy()
    ida = np.asarray(ids)
    for gid in range(ida.max() + 1):
        assert (intr[ida == gid] == intr[np.flatnonzero(ida == gid)[0]]).all()          # group rows equal bit for bit
    assert (intr[:, 1:3] == prior[:, 1:3]).all()
    for gid in gauge.get("fixed_intrinsics", ()):
        assert (intr[ida == gid] == prior[ida == gid]).all()
    for i in gauge.get("fixed_poses", (0,)):
        assert torch.equal(res.R[i], R[i].double()) and torch.equal(res.t[i], t[i].double())


U = np.finfo(np.float64).eps / 2


def test_folded_system_matches_the_oracle(monkeypatch):
    """S' and b' as romab200_ba_fold leaves them, against the oracle's system built in the shared parameters, at the first trial;
    fixed poses, a fixed t_x and a fixed group included."""
    ids = [0, 0, 1, 1, 1, 2, 2]
    gauge = dict(fixed_poses=(0, 3), fixed_tx=(1,), fixed_intrinsics=(2,))
    g, tr, pts, prior, R, t, _ = _scene(5, ids, 300)
    caps = []
    orig = cabi.call

    def spy(fn, struct, **a):
        orig(fn, struct, **a)
        if fn == "romab200_ba_fold":
            n = 6 * a["num_free"] + 2 * a["num_groups"]
            caps.append((a["S_groups"].view(n, n).cpu().numpy().copy(), a["rhs_groups"].cpu().numpy().copy()))

    monkeypatch.setattr(cabi, "call", spy)
    bundle_adjust(g, tr, pts, prior, R, t, camera_model="SIMPLE_RADIAL", camera_ids=ids, max_iterations=1, **gauge)
    monkeypatch.setattr(cabi, "call", orig)
    systems = []
    _oracle(g, tr, pts, prior, R, t, ids, max_iterations=1, systems=systems, **gauge)
    S, b = caps[0]
    sy = systems[0]
    lo = np.tril_indices(S.shape[0])
    rS = np.abs(S[lo] - sy["S"][lo]).max() / np.abs(sy["S"]).max()
    rB = np.abs(b - sy["b"]).max() / np.abs(sy["b"]).max()
    print(f"n' = {S.shape[0]}: |S' - S'_oracle| {rS / U:.1f} u max|S'|, |b' - b'_oracle| {rB / U:.1f} u max|b'|")
    assert S.shape[0] == 6 * len(sy["free"]) + 2 * len(sy["groups"])
    assert rS <= 1e-11 and rB <= 1e-11


@pytest.mark.parametrize("seed, N, loss_scale", [(6, 8, None), (7, 12, 1.0)])
def test_singleton_groups_equal_per_image_intrinsics(seed, N, loss_scale):
    g, tr, pts, prior, R, t, _ = _scene(seed, np.arange(N), 300)
    # function_tolerance stops both runs before trials at the rounding floor of F, where one may keep a step the other rejects
    kw = dict(camera_model="SIMPLE_RADIAL", loss_scale=loss_scale, max_iterations=30, function_tolerance=1e-9)
    a = bundle_adjust(g, tr, pts, prior, R, t, camera_ids=np.arange(N), **kw)
    b = bundle_adjust(g, tr, pts, prior, R, t, **kw)
    print(f"N={N}: {a.accepted.size} and {b.accepted.size} trials ({a.termination}, {b.termination}), F -> {a.cost[-1]:.10g}")
    assert (a.accepted == b.accepted).all() and a.termination == b.termination
    assert np.abs(a.cost - b.cost).max() <= 1e-9 * b.cost.max()
    _close(a, dict(R=b.R.cpu().numpy(), t=b.t.cpu().numpy(), intrinsics=b.intrinsics.cpu().numpy(), X=b.points.X.cpu().numpy()), 1e-8)


def test_reruns_are_byte_identical_and_unobserved_members_follow_their_group():
    ids = np.zeros(10, np.int64)
    g, tr, pts, prior, R, t, _ = _scene(8, ids, 400, cs=4, outlier_frac=0.2)
    # images 7-9 have fixed poses and no observations: they are free cameras only through their group's intrinsics
    from roma_b200.triangulate import Points3D
    el = tr.elements.long()
    inl = pts.inlier & (el[:, 0] < 7)
    p2 = Points3D(pts.X, pts.ok, pts.num_inliers, pts.error, inl)
    kw = dict(camera_model="SIMPLE_RADIAL", camera_ids=ids, loss_scale=1.0, fixed_poses=(0, 7, 8, 9))
    a = bundle_adjust(g, tr, p2, prior, R, t, **kw)
    b = bundle_adjust(g, tr, p2, prior, R, t, **kw)
    for x, y in ((a.R, b.R), (a.t, b.t), (a.intrinsics, b.intrinsics), (a.points.X, b.points.X), (a.points.error, b.points.error)):
        assert torch.equal(x, y)
    assert a.cost.tobytes() == b.cost.tobytes() and a.pred.tobytes() == b.pred.tobytes()
    assert a.accepted.any() and (a.intrinsics == a.intrinsics[0]).all() and a.intrinsics[0, 0] != prior[0, 0]


def test_pinhole_and_per_image_outputs_are_unchanged():
    """The digests of tests/golden/make_golden_ba_digests.py, written by the build before shared cameras."""
    spec = importlib.util.spec_from_file_location("make_golden_ba_digests", os.path.join(HERE, "golden", "make_golden_ba_digests.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    with open(os.path.join(HERE, "golden", "ba_digests.json")) as f:
        want = json.load(f)
    got = mod.digests()
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k] == want[k], k


# ---- reconstruct ----------------------------------------------------------------------------------------------------------------
def _mapper_scene(seed, ids, ferr, points=1500):
    """The spread geometry at 384 x 512 with truth k in +-0.05; the prior's f is off by `ferr` (sign random) for every image of a
    camera alike, and k = 0."""
    ids = np.asarray(ids)
    pairs, m, c, sizes, views, intr, R, t, X = synthetic.planted_cameras(seed, ids.size, points, size=(384, 512), radial=(-0.05, 0.05),
                                                                         spread=True, camera_ids=ids, device=DEV)
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    rng = np.random.default_rng(seed)
    prior = intr.cpu().numpy().copy()
    prior[:, 0] *= (1 + rng.choice([-1.0, 1.0], ids.max() + 1) * ferr)[ids]
    prior[:, 3] = 0.0
    return pairs, g, tr, prior, intr.cpu().numpy(), R.cpu().numpy(), t.cpu().numpy(), sizes


def _cam_errors(rec, Rg, tg):
    from test_mapper_gpu import _errors
    return _errors(rec.R.cpu().numpy(), rec.t.cpu().numpy(), Rg, tg, rec.registered.cpu().numpy())


# Bars from the first H100 run of these 8 cases, with a 2x margin: the shared run's f error was 1.5e-3 to 2.5e-3 at a 10 % prior
# and 5.6e-3 to 6.7e-3 at 20 % (per-image worst: 3.8e-3 to 5.5e-3 and 8.4e-3 to 1.4e-2); its worst centre error 0.0085 to 0.0356
# (per-image 0.019 to 0.048).
SHARED_FERR_MAX, SHARED_CENTRE_MAX = 1.4e-2, 0.075


@pytest.mark.parametrize("ferr", [0.10, 0.20])
@pytest.mark.parametrize("seed", [40, 41, 42, 43])
def test_shared_camera_recovers_f_better_than_per_image(seed, ferr):
    ids = np.zeros(30, np.int64)
    pairs, g, tr, prior, truth, Rg, tg, sizes = _mapper_scene(seed, ids, ferr)
    per = reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True)
    sh = reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True, camera_ids=ids)
    assert torch.equal(sh.camera_ids.cpu(), torch.from_numpy(ids)) and per.camera_ids is None
    out = {}
    for name, rec in (("per-image", per), ("shared", sh)):
        f = rec.intrinsics.cpu().numpy()
        fe = np.abs(f[:, 0] / truth[:, 0] - 1)[rec.registered.cpu().numpy()]
        ang, cen = _cam_errors(rec, Rg, tg)
        out[name] = (int(rec.registered.sum()), fe.max(), np.median(fe), cen.max(), np.median(cen))
        print(f"seed {seed} prior {ferr:.0%} {name}: {out[name][0]} registered, f error max {fe.max():.2e} median {np.median(fe):.2e}, "
              f"centre worst {cen.max():.4f} median {np.median(cen):.4f}, k {f[0, 3]:+.5f} (truth {truth[0, 3]:+.5f})")
    f = sh.intrinsics.cpu().numpy()
    assert (f == f[0]).all()
    assert out["shared"][0] >= out["per-image"][0]
    assert out["shared"][1] < out["per-image"][1] and out["shared"][3] < out["per-image"][3]
    assert out["shared"][1] <= SHARED_FERR_MAX and out["shared"][3] <= SHARED_CENTRE_MAX


def test_reconstruct_with_camera_ids_equals_the_hand_written_loop(tmp_path):
    """Two cameras (images alternate), one of them registered only from the second round on; the loop written out with the
    device stages gives byte-identical results; the COLMAP model has one camera per group."""
    from roma_b200 import bundle_adjust as ba, initialize_reconstruction, register_images, write_colmap_text
    from roma_b200.mapper import MIN_REGISTERED_TO_REFINE
    ids = np.array([0, 1] * 6)
    pairs, g, tr, prior, truth, Rg, tg, sizes = _mapper_scene(44, ids, 0.05, points=1200)
    rec = reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True, camera_ids=ids)
    N, cur = ids.size, prior.copy()
    ug, Kc = undistort_graph(g, cur), pinhole_K(cur)
    init = initialize_reconstruction(pairs, ug, Kc)
    a, b = init.images[init.chosen].tolist()
    R = torch.zeros(N, 3, 3, dtype=torch.float64, device=DEV)
    t = torch.zeros(N, 3, dtype=torch.float64, device=DEV)
    R[a] = torch.eye(3, dtype=torch.float64, device=DEV)
    R[b], t[b] = init.R[init.chosen], init.t[init.chosen]
    registered, rounds = sorted((a, b)), []
    while True:
        rest = [i for i in range(N) if i not in registered]
        pts = triangulate_tracks(ug, tr, Kc, R, t, images=registered)
        free = len(registered) >= MIN_REGISTERED_TO_REFINE
        fixed_groups = [c for c in range(2) if c not in set(ids[registered].tolist())]
        res = ba(g, tr, pts, cur, R, t, fixed_poses=[a] + rest, fixed_tx=[b], camera_model="SIMPLE_RADIAL", refine_focal_length=free,
                 refine_extra_params=free, camera_ids=ids, fixed_intrinsics=fixed_groups)
        R, t = res.R.clone(), res.t.clone()
        if free:
            cur = res.intrinsics.cpu().numpy()
            ug, Kc = undistort_graph(g, cur), pinhole_K(cur)
        pts = triangulate_tracks(ug, tr, Kc, R, t, images=registered)
        rounds.append((list(registered), fixed_groups))
        if not rest:
            break
        reg = register_images(ug, tr, pts, Kc, rest)
        acc = reg.accepted.tolist()
        added = [i for m, i in enumerate(rest) if acc[m]]
        if not added:
            break
        rows = torch.tensor([m for m in range(len(rest)) if acc[m]], device=DEV)
        R[torch.tensor(added, device=DEV)], t[torch.tensor(added, device=DEV)] = reg.R[rows], reg.t[rows]
        registered = sorted(registered + added)
    print(f"rounds (registered, fixed groups): {rounds}")
    assert [r["registered"] for r in rec.rounds] == [r[0] for r in rounds]
    assert rec.registered.nonzero().flatten().tolist() == registered
    assert torch.equal(rec.R, R) and torch.equal(rec.t, t) and torch.equal(rec.intrinsics.cpu(), torch.from_numpy(cur))
    for name in ("X", "ok", "error", "inlier"):
        assert torch.equal(getattr(rec.points, name), getattr(pts, name)), name
    write_colmap_text(tmp_path, rec, g, tr, None, sizes)
    from test_mapper_host import _parse
    cams, images, _ = _parse(tmp_path)
    assert sorted(cams) == [1, 2] and all(int(h[8]) == ids[iid - 1] + 1 for iid, (h, _) in images.items())
