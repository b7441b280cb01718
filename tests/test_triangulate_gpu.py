"""`triangulate_tracks` on the GPU: on `planted_cameras` scenes (clean, and with 20 % outlier samples through `verify_matches`, and a
graph whose tracks keep their conflicts) the device agrees with `oracle/triangulate.py` (X to 1e-9 (1 + |X|); ok, num_inliers and
inlier exactly wherever the oracle's decisions are clear of rounding); reruns are byte-identical; a long track takes the drawn-pair
path; the clean-scene accuracy and the robustness to moved observations meet their bars; a bad element id raises ValueError."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.triangulate import triangulate  # noqa: E402
from roma_b200 import MatchGraph, Tracks, build_tracks, consolidate_matches, synthetic, triangulate_tracks, verify_matches  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}


def _scene(seed, N, points, cs=1, outlier_frac=0.0, size=(384, 512), drop_conflicts=True, **kw):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cs, outlier_frac=outlier_frac,
                                                                      device=DEV, **kw)
    g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    if outlier_frac > 0 and drop_conflicts:
        g = verify_matches(pairs, g, threshold=THR[cs])[0]
    return g, build_tracks(pairs, g, drop_conflicts=drop_conflicts), views, K, R, t, X


def _oracle(g, tr, K, R, t, **kw):
    return triangulate(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, K, R, t, **kw)


def _compare(res, ref, tr):
    """Asserts the agreement of the device and the oracle; returns the number of tracks left out for a decision within rounding."""
    off = tr.track_offsets.cpu().numpy()
    T = off.size - 1
    seg = off[:-1]
    e2 = np.nan_to_num(np.abs(ref["err2_margin"]), nan=np.inf)
    dp = np.nan_to_num(np.abs(ref["depth"]), nan=np.inf)
    e2_t = np.minimum.reduceat(e2, seg) if T else e2
    dp_t = np.minimum.reduceat(dp, seg) if T else dp
    clear = (np.minimum(e2_t, ref["hyp_margin"]) > 1e-6) & (dp_t > 1e-9) & (ref["hyp_margin"] > 1e-9) & (np.abs(ref["angle_margin"]) > 1e-9)
    el_clear = np.repeat(clear, np.diff(off))
    ok, n, inl = res.ok.cpu().numpy(), res.num_inliers.cpu().numpy(), res.inlier.cpu().numpy()
    assert np.array_equal(ok[clear], ref["ok"][clear])
    assert np.array_equal(n[clear], ref["num_inliers"][clear])
    assert np.array_equal(inl[el_clear], ref["inlier"][el_clear])
    both = clear & ok
    X, Xr = res.X.cpu().numpy(), ref["X"]
    # X to 1e-9 (1 + |X|), or to a few times the Gauss-Newton step whose keep-or-stop decision the oracle found within rounding
    tol = np.maximum(1e-9 * (1 + np.linalg.norm(Xr[both], axis=1)), 4 * ref["gn_step"][both])
    assert (np.linalg.norm(X[both] - Xr[both], axis=1) <= tol).all(), np.abs(X[both] - Xr[both]).max()
    print(f"X within 1e-9 (1 + |X|) on {int((np.linalg.norm(X[both] - Xr[both], axis=1) <= 1e-9 * (1 + np.linalg.norm(Xr[both], axis=1))).sum())} "
          f"of {int(both.sum())} ok tracks, {int((ref['gn_step'][both] > 0).sum())} with a Gauss-Newton stop within rounding")
    assert np.allclose(res.error.cpu().numpy()[both], ref["error"][both], rtol=1e-6, atol=1e-9)
    assert (X[~ok] == 0).all() and (n[~ok] == 0).all() and not inl[np.repeat(~ok, np.diff(off))].any()
    return int((~clear).sum())


@pytest.mark.parametrize("seed, N, cs, outlier_frac, points", [(0, 3, 1, 0.0, 800), (1, 3, 4, 0.2, 800), (2, 8, 1, 0.2, 800),
                                                                (3, 8, 4, 0.0, 800), (4, 30, 1, 0.2, 300), (5, 30, 4, 0.0, 300)])
def test_device_matches_the_oracle(seed, N, cs, outlier_frac, points):
    g, tr, views, K, R, t, X = _scene(seed, N, points, cs, outlier_frac)
    res = triangulate_tracks(g, tr, K, R, t)
    ref = _oracle(g, tr, K, R, t)
    left_out = _compare(res, ref, tr)
    # Acceptance is measured on the tracks of planted points.  With outliers, matches that pass verification by lying near their
    # epipolar line also form tracks, mostly of two views; such a track has a consistent two-view point, so no triangulation rule
    # can tell it from a true one, and about half of them pass the angle test.
    planted = synthetic.track_points(tr.track_offsets, tr.elements, g.kp_offsets, g.keypoints, views, 512, cs) >= 0
    ok = res.ok.cpu().numpy()
    print(f"N={N} cs={cs} outliers={outlier_frac}: {len(tr)} tracks, {int(planted.sum())} of planted points, {ok[planted].mean():.4f} of "
          f"those ok, {ok[~planted].mean() if (~planted).any() else 0:.4f} of the others ok, {left_out} left out")
    assert planted.sum() > 100 and left_out <= max(2, len(tr) // 500) and ok[planted].mean() > 0.95


def test_conflicting_tracks_match_the_oracle():
    g, tr, views, K, R, t, X = _scene(6, 16, 20000, 1, 0.2, size=(768, 1024), drop_conflicts=False)
    assert tr.num_conflicting > 0
    res = triangulate_tracks(g, tr, K, R, t)
    ref = _oracle(g, tr, K, R, t)
    assert _compare(res, ref, tr) <= max(2, len(tr) // 500)


def test_options_and_byte_identical_reruns():
    g, tr, views, K, R, t, X = _scene(7, 8, 800, 1, 0.2)
    kw = dict(max_error=2.5, min_angle=3.0, max_hypotheses=6, seed=11)
    a = triangulate_tracks(g, tr, K, R, t, **kw)
    b = triangulate_tracks(g, tr, K.cpu().numpy(), R.cpu(), t, **kw)               # the same cameras as an array and a CPU tensor
    f = triangulate_tracks(g, tr, K.float(), R.float(), t.half())                 # any float dtype, widened on the host
    assert f.X.dtype == torch.float64 and f.ok.float().mean() > 0.9
    c = triangulate_tracks(g, tr, K, R, t, **kw)
    for other in (b, c):
        for name in ("X", "ok", "num_inliers", "error", "inlier"):
            x, y = getattr(a, name), getattr(other, name)
            assert x.dtype == y.dtype and x.shape == y.shape and x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes(), name
    assert a.X.dtype == torch.float64 and a.ok.dtype == torch.bool and a.num_inliers.dtype == torch.int32
    assert a.error.dtype == torch.float64 and a.inlier.dtype == torch.bool and a.inlier.shape == (tr.elements.shape[0],)
    assert _compare(a, _oracle(g, tr, K, R, t, **kw), tr) <= max(2, len(tr) // 500)


def test_a_long_track_takes_the_drawn_pairs():
    g, tr, views, K, R, t, X = _scene(8, 600, 1, 1, 0.0, size=(768, 1024), visibility=1.0)
    L = int(tr.elements.shape[0])
    assert len(tr) == 1 and L * (L - 1) // 2 > 256 and L >= 300
    res = triangulate_tracks(g, tr, K, R, t)
    ref = _oracle(g, tr, K, R, t)
    assert _compare(res, ref, tr) == 0 and bool(res.ok[0])
    assert np.linalg.norm(res.X[0].cpu().numpy() - X[0].cpu().numpy()) < 0.01


def test_accuracy_on_clean_scenes():
    g, tr, views, K, R, t, X = _scene(0, 8, 2000, 1, size=(768, 1024))
    res = triangulate_tracks(g, tr, K, R, t)
    pts = synthetic.track_points(tr.track_offsets, tr.elements, g.kp_offsets, g.keypoints, views, 1024)
    ok = res.ok.cpu().numpy() & (pts >= 0)
    err = np.linalg.norm(res.X.cpu().numpy()[ok] - X.cpu().numpy()[pts[ok]], axis=1)
    print(f"{ok.sum()} of {len(tr)} tracks: 3-D error median {np.median(err):.4f}, p95 {np.percentile(err, 95):.3f}")
    assert ok.mean() > 0.99 and np.median(err) < 0.015 and np.percentile(err, 95) < 0.1


def _move_observations(g, tr, frac, seed):
    """Moves `frac` of the observations of tracks of 3 elements or more by 20-50 px: (MatchGraph with the moved keypoints, moved [E])."""
    rng = np.random.default_rng(seed)
    off, el = tr.track_offsets.cpu().numpy(), tr.elements.cpu().numpy().astype(np.int64)
    L = np.diff(off)
    moved = np.repeat(L >= 3, L) & (rng.random(el.shape[0]) < frac)
    ang, r = rng.uniform(0, 2 * np.pi, moved.sum()), rng.uniform(20, 50, moved.sum())
    xy = g.keypoints.cpu().numpy().copy()
    rows = g.kp_offsets.cpu().numpy()[el[moved, 0]] + el[moved, 1]
    xy[rows] += np.stack((r * np.cos(ang), r * np.sin(ang)), 1).astype(np.float32)
    h = MatchGraph(g.kp_offsets, torch.from_numpy(xy).to(DEV), g.kp_scores, g.match_offsets, g.matches, g.match_scores)
    return h, moved


def test_robustness_to_moved_observations():
    g, tr, views, K, R, t, X = _scene(1, 16, 2000, 1, size=(768, 1024))
    h, moved = _move_observations(g, tr, 0.1, 0)
    res = triangulate_tracks(h, tr, K, R, t)
    inl = res.inlier.cpu().numpy()
    rejected, kept, accepted = (~inl[moved]).mean(), inl[~moved].mean(), res.ok.float().mean().item()
    print(f"moved {moved.sum()} of {moved.size}: rejected {rejected:.4f}, others kept {kept:.4f}, tracks accepted {accepted:.4f}")
    assert moved.sum() > 1000 and rejected >= 0.99 and kept >= 0.995 and accepted >= 0.99


@pytest.mark.parametrize("col, value", [(0, -1), (0, 3), (1, -1), (1, 1 << 20)])
def test_out_of_range_element_raises(col, value):
    g, tr, views, K, R, t, X = _scene(9, 3, 400)
    el = tr.elements.clone()
    el[5, col] = value
    bad = Tracks(tr.track_offsets, el, tr.kp_track, tr.num_conflicting)
    with pytest.raises(ValueError, match="outside"):
        triangulate_tracks(g, bad, K, R, t)
    assert bool(triangulate_tracks(g, tr, K, R, t).ok.any())                     # the device is fine afterwards


def test_empty_tracks():
    g, tr, views, K, R, t, X = _scene(10, 3, 400)
    empty = Tracks(torch.zeros(1, dtype=torch.int64, device=DEV), torch.zeros(0, 2, dtype=torch.int32, device=DEV), tr.kp_track, 0)
    res = triangulate_tracks(g, empty, K, R, t)
    assert res.X.shape == (0, 3) and res.ok.shape == (0,) and res.num_inliers.shape == (0,) and res.error.shape == (0,)
    assert res.inlier.shape == (0,) and res.X.device.type == "cuda"
