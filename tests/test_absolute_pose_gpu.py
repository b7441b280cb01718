"""`estimate_absolute_pose_batched`, `register_images` and `triangulate_tracks(images=...)` on the GPU: on `planted_cameras` scenes the
device agrees with `oracle/absolute_pose.py` (ok exactly; num_inliers and mask wherever the oracle's decisions are clear of rounding;
R and t to 1e-9, or to a few Gauss-Newton steps where a keep-or-stop decision was within rounding); a batch item is byte-identical to
the item alone and reruns are byte-identical; edge cases; restricted triangulation against `oracle/register.py`, and images=None byte-identical to
the release before the argument; and the incremental loop the feature enables registers every offered image of a 10-image scene
within bars set from the same loop run with the oracles."""
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import absolute_pose as ap  # noqa: E402
from oracle import register as oreg  # noqa: E402
from roma_b200 import (build_tracks, bundle_adjust, consolidate_matches, estimate_absolute_pose, estimate_absolute_pose_batched,  # noqa: E402
                       register_images, synthetic, triangulate_tracks, verify_matches)
from roma_b200.tracks import Tracks  # noqa: E402
from test_triangulate_gpu import _compare as tri_compare  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}


def _scene(seed, N, points, cs=1, outlier_frac=0.0, size=(384, 512)):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cs, outlier_frac=outlier_frac,
                                                                      device=DEV)
    g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    if outlier_frac > 0:
        g = verify_matches(pairs, g, threshold=THR[cs])[0]
    return g, build_tracks(pairs, g), K, R, t


def _rot_deg(Ra, Rb):
    return math.degrees(math.acos(min(1.0, max(-1.0, (np.trace(Ra.T @ Rb) - 1) / 2))))


def _compare(R, t, ok, n, mask, ref):
    """Asserts one item's agreement with the oracle; returns whether its decisions were clear of rounding.  Clear means every
    squared error of every scored model and of the final pose lies more than 1e-6 px^2 from max_error^2 and every depth more than
    1e-9 from 0: then every count is the same integer on both sides, so the sequential loop takes the same (h, solution) at every
    change of the best, ties included, and stops at the same hypothesis."""
    assert bool(ok) == ref["ok"]
    if not ref["ok"]:
        assert not mask.any() and (R == 0).all() and (t == 0).all() and n == 0
        return True
    clear = (ref["hyp_margin"] > 1e-6 and np.nanmin(np.abs(ref["err2_margin"])) > 1e-6 and np.nanmin(np.abs(ref["depth"])) > 1e-9)
    if clear:
        assert n == ref["num_inliers"] and np.array_equal(mask, ref["mask"])
        tol = max(1e-9, 4 * ref["gn_step"])
        assert np.abs(R - ref["R"]).max() <= tol and np.abs(t - ref["t"]).max() <= tol * (1 + np.abs(ref["t"]).max()), \
            (np.abs(R - ref["R"]).max(), np.abs(t - ref["t"]).max(), ref["gn_step"])
    return clear


@pytest.mark.parametrize("seed, N, cs, outlier_frac, points", [(0, 3, 1, 0.0, 800), (1, 3, 4, 0.2, 800), (2, 8, 1, 0.2, 800),
                                                                (3, 8, 4, 0.0, 800), (4, 30, 1, 0.2, 300), (5, 30, 4, 0.0, 300)])
def test_registration_matches_the_oracle(seed, N, cs, outlier_frac, points):
    """Every listed image, accepted or not: R, t, ok, num_inliers and mask against the oracle.  register_images must equal the
    batched estimator on the gathered correspondences, which also gives the masks of the images that are not accepted."""
    g, tr, K, R, t = _scene(seed, N, points, cs, outlier_frac)
    pts = triangulate_tracks(g, tr, K, R, t, max_error=THR[cs] * 2, images=[0, 1])
    images = list(range(N))[::-1]
    reg = register_images(g, tr, pts, K, images, max_error=12.0, min_inliers=30, seed=seed)
    corr = ap.gather(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.ok, pts.X, images)
    Kn = K.cpu().numpy()[images]
    eR, et, eok, en, emask = estimate_absolute_pose_batched([c[0] for c in corr], [c[1] for c in corr], Kn, max_error=12.0, seed=seed)
    assert np.array_equal(reg.R.cpu().numpy(), eR) and np.array_equal(reg.t.cpu().numpy(), et)
    assert np.array_equal(reg.ok.cpu().numpy(), eok) and np.array_equal(reg.num_inliers.cpu().numpy(), en)
    el_img = tr.elements[:, 0].cpu().numpy()
    el_ok = np.repeat(pts.ok.cpu().numpy(), np.diff(tr.track_offsets.cpu().numpy()))
    inlier = reg.inlier.cpu().numpy()
    left_out = 0
    for m, i in enumerate(images):
        x, X = corr[m]
        assert int(reg.num_correspondences[m]) == len(x)
        acc = bool(reg.accepted[m])
        assert acc == (bool(eok[m]) and en[m] >= 30)
        elems = np.flatnonzero((el_img == i) & el_ok)
        assert np.array_equal(inlier[elems], emask[m] if acc else np.zeros(len(x), bool))
        assert not inlier[(el_img == i) & ~el_ok].any()
        ref = ap.estimate(x, X, Kn[m], max_error=12.0, seed=seed)
        clear = _compare(eR[m], et[m], eok[m], int(en[m]), emask[m], ref)
        left_out += not clear
        if acc:
            assert _rot_deg(eR[m], R[i].cpu().numpy()) < 2.0        # registered against two-view points: a loose sanity bar
    print(f"{int(reg.accepted.sum())} of {N} images accepted, {left_out} left out for a decision within rounding")
    assert left_out <= max(1, N // 10)
    # against the points of two cameras only, an image that sees fewer than min_inliers of them is rightly not accepted (at N = 30
    # with 300 points, 23 and 27 of 30 are)
    assert int(reg.accepted.sum()) >= N * 2 // 3


def test_batch_items_are_byte_identical_to_single_calls_and_reruns():
    g, tr, K, R, t = _scene(7, 8, 600, 1, 0.2)
    pts = triangulate_tracks(g, tr, K, R, t, images=[0, 1])
    corr = ap.gather(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.ok, pts.X, range(8))
    xs = [torch.from_numpy(c[0]).to(DEV) for c in corr]
    Xs = [torch.from_numpy(c[1]).float().to(DEV) for c in corr]          # any float dtype, widened to float64
    Kb = K.float()
    out = estimate_absolute_pose_batched(xs, Xs, Kb, seed=3)
    again = estimate_absolute_pose_batched(xs, Xs, Kb, seed=3)
    rev = estimate_absolute_pose_batched(xs[::-1], Xs[::-1], Kb.flip(0), seed=3)
    for a, b in zip(out[:4], again[:4]):
        assert torch.equal(a, b)
    for m in range(8):
        single = estimate_absolute_pose(xs[m], Xs[m], Kb[m], seed=3)
        assert single is not None and out[2][m]
        assert torch.equal(single[0], out[0][m]) and torch.equal(single[1], out[1][m]) and torch.equal(single[2], out[4][m])
        assert torch.equal(rev[0][7 - m], out[0][m]) and torch.equal(rev[4][7 - m], out[4][m])
    # register_images: byte-identical to the batched estimator on the same correspondences, for any workspace and order
    reg = register_images(g, tr, pts, K, range(8), seed=3)
    small = register_images(g, tr, pts, K, list(range(8))[::-1], seed=3, workspace_bytes=1)
    ref = estimate_absolute_pose_batched(xs, [torch.from_numpy(c[1]).to(DEV) for c in corr], K, seed=3)
    assert torch.equal(reg.R, ref[0]) and torch.equal(reg.t, ref[1]) and torch.equal(reg.num_inliers, ref[3])
    assert torch.equal(small.R.flip(0), reg.R) and torch.equal(small.inlier, reg.inlier)
    # numpy in, numpy out
    npo = estimate_absolute_pose_batched([c[0] for c in corr], [c[1] for c in corr], K.cpu().numpy(), seed=3)
    assert isinstance(npo[0], np.ndarray) and np.array_equal(npo[0], ref[0].cpu().numpy())


def test_edge_cases():
    rng = np.random.default_rng(0)
    K = np.array([[500.0, 0, 256], [0, 500.0, 192], [0, 0, 1]])
    X = rng.uniform(-2, 2, (60, 3))
    Y = X + [0, 0, 8]
    x = (Y @ K.T)[:, :2] / Y[:, 2:]
    items_x = [x[:2], x[:0], x[:3], np.repeat(x[:1], 20, 0), rng.uniform(0, 500, (60, 2)), x]
    items_X = [X[:2], X[:0], X[:3], np.repeat(X[:1], 20, 0), rng.uniform(-2, 2, (60, 3)), X]
    R, t, ok, n, masks = estimate_absolute_pose_batched(items_x, items_X, K, max_error=1.0)
    assert list(ok) == [False, False, True, False, bool(ok[4]), True]
    for b in (0, 1, 3):
        assert not masks[b].any() and (R[b] == 0).all() and (t[b] == 0).all() and n[b] == 0
    assert n[2] == 3 and n[4] <= 4 and n[5] == 60
    assert np.abs(R[5] - np.eye(3)).max() < 1e-9 and np.abs(t[5] - [0, 0, 8]).max() < 1e-8
    for b in range(6):
        ref = ap.estimate(items_x[b], items_X[b], K, max_error=1.0)
        assert bool(ok[b]) == ref["ok"]
    assert estimate_absolute_pose(x[:2], X[:2], K) is None
    # a bad element id raises before any kernel indexes with it
    g, tr, Kc, Rc, tc = _scene(9, 3, 300)
    pts = triangulate_tracks(g, tr, Kc, Rc, tc, images=[0, 1])
    el = tr.elements.clone()
    el[len(el) // 2, 1] = 10 ** 6
    with pytest.raises(ValueError, match="outside"):
        register_images(g, Tracks(tr.track_offsets, el, tr.kp_track, 0), pts, Kc, [2])
    empty = register_images(g, tr, pts, Kc, [])
    assert empty.R.shape == (0, 3, 3) and not empty.inlier.any()


@pytest.mark.parametrize("seed, N, cs, outlier_frac", [(0, 8, 1, 0.2), (1, 8, 4, 0.0)])
def test_restricted_triangulation(seed, N, cs, outlier_frac):
    g, tr, K, R, t = _scene(seed, N, 600, cs, outlier_frac)
    base = triangulate_tracks(g, tr, K, R, t)
    every = triangulate_tracks(g, tr, K, R, t, images=list(range(N)))
    for f in ("X", "ok", "num_inliers", "error", "inlier"):
        assert torch.equal(getattr(base, f), getattr(every, f))
    sub = [0, 2, 5]
    Rj, tj = R.clone(), t.clone()
    Rj[1], tj[1] = torch.eye(3, dtype=torch.float64) * 7, torch.tensor([1.0, 2.0, -30.0], dtype=torch.float64)   # not read
    res = triangulate_tracks(g, tr, K, Rj, tj, images=sub)
    ref = oreg.triangulate(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, K, R, t, sub)
    el_img = tr.elements[:, 0].cpu().numpy()
    assert not res.inlier.cpu().numpy()[~np.isin(el_img, sub)].any()
    left_out = tri_compare(res, ref, tr)          # ok, num_inliers and every inlier flag on clear tracks; X, error to tolerance
    print(f"{left_out} of {len(ref['ok'])} tracks left out for a decision within rounding")
    assert left_out <= max(2, len(ref["ok"]) // 100)


@pytest.mark.parametrize("tag, seed, N, points, cs, outlier_frac", [("a", 12, 6, 400, 1, 0.2), ("b", 13, 5, 400, 4, 0.0)])
def test_images_none_is_byte_identical_to_the_previous_release(tag, seed, N, points, cs, outlier_frac):
    """tests/golden/triangulate_before_images.npz holds what triangulate_tracks returned on these scenes before it had the images
    argument (tests/golden/make_golden_triangulate.py)."""
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "triangulate_before_images.npz"))
    g, tr, K, R, t = _scene(seed, N, points, cs, outlier_frac)
    for images in (None, list(range(N))):
        res = triangulate_tracks(g, tr, K, R, t, images=images)
        for f in ("X", "ok", "num_inliers", "error", "inlier"):
            v = getattr(res, f).cpu().numpy()
            assert v.dtype == gold[f"{tag}_{f}"].dtype and v.tobytes() == gold[f"{tag}_{f}"].tobytes(), f


@pytest.mark.parametrize("withheld", [None, 9])
def test_incremental_reconstruction(withheld):
    """Two known cameras, then triangulate -> register -> re-triangulate until no image is added, then bundle_adjust with the
    never-registered images held fixed (`withheld` is never offered for registration, so it stays at a zero camera in fixed_poses).
    Bars, set from oracle/register.py's `incremental` (the same loop on the CPU with the numpy oracles) on this scene: it registers
    every offered image, and its worst rotation and centre errors are 0.104 degrees and 0.0175 units with every image offered, 0.069
    degrees and 0.0102 units with image 9 withheld (medians about 0.04 degrees and 0.004 units).  The device must register the
    same images within 0.15 degrees and 0.025 units on every registered camera (the scene spans about 8 units at 8-10 units from the
    cameras) and leave the withheld camera untouched."""
    N = 10
    g, tr, K, R, t = _scene(11, N, 1500, 1, 0.2)
    offered = [i for i in range(N) if i != withheld]
    Rw, tw = torch.zeros_like(R), torch.zeros_like(t)
    Rw[:2], tw[:2] = R[:2], t[:2]
    registered = [0, 1]
    while True:
        pts = triangulate_tracks(g, tr, K, Rw, tw, images=registered)
        rest = [i for i in offered if i not in registered]
        if not rest:
            break
        reg = register_images(g, tr, pts, K, rest)
        new = [i for m, i in enumerate(rest) if bool(reg.accepted[m])]
        if not new:
            break
        for m, i in enumerate(rest):
            if bool(reg.accepted[m]):
                Rw[i], tw[i] = reg.R[m], reg.t[m]
        registered = sorted(registered + new)
    assert registered == offered
    fixed = [0] + [i for i in range(N) if i not in registered]
    assert fixed == ([0] if withheld is None else [0, withheld])
    if withheld is not None:
        assert not pts.inlier[tr.elements[:, 0] == withheld].any()
    ba = bundle_adjust(g, tr, pts, K, Rw, tw, fixed_poses=fixed)
    Rf, tf = ba.R.cpu().numpy(), ba.t.cpu().numpy()
    Rg, tg = R.cpu().numpy(), t.cpu().numpy()
    rot = [_rot_deg(Rf[i], Rg[i]) for i in registered]
    cen = [np.linalg.norm(-Rf[i].T @ tf[i] + Rg[i].T @ tg[i]) for i in registered]
    print(f"rotation error max {max(rot):.4f} deg, median {np.median(rot):.4f}; centre error max {max(cen):.5f}, median {np.median(cen):.5f}")
    assert max(rot) < 0.15 and max(cen) < 0.025
    if withheld is not None:
        assert (Rf[withheld] == 0).all() and (tf[withheld] == 0).all()
