"""CPU tests of track triangulation (`triangulate_tracks`): the numpy oracle on hand-built cameras (an exact two-view point, a point
behind a camera, min_angle on either side of the true angle, ties to the first hypothesis, same-image pairs skipped), the switch
from every pair to drawn pairs, the camera table, every argument rule (raised before any device work), `synthetic.track_points`,
and the robustness to moved observations on a 16-image `planted_cameras` scene."""
import math

import numpy as np
import pytest
import torch

from oracle.match_graph import consolidate
from oracle.ransac import draw_distinct
from oracle.tracks import tracks as oracle_tracks
from oracle.triangulate import CTR, GN_ITERS, hypothesis_pairs, triangulate
from roma_b200 import cabi, synthetic, triangulate as rb_tri
from roma_b200.match_graph import MatchGraph
from roma_b200.tracks import Tracks

KF = np.array([[500.0, 0.0, 320.0], [0.0, 500.0, 240.0], [0.0, 0.0, 1.0]])


def rig(centres, flip=()):
    """Cameras with K = KF, R = I (or a half turn about y for the indices in `flip`), at the given centres."""
    n = len(centres)
    R = np.stack([np.diag([-1.0, 1.0, -1.0]) if i in flip else np.eye(3) for i in range(n)])
    t = -np.einsum("nij,nj->ni", R, np.asarray(centres, float))
    return np.repeat(KF[None], n, 0), R, t


def project(K, R, t, X):
    p = K @ (R @ X + t)
    return p[:2] / p[2]


def scene(K, R, t, obs):
    """A track per entry of obs: [(image, X), ...], each observation its own keypoint at the exact projection of X (fp32)."""
    N = K.shape[0]
    per = [[] for _ in range(N)]
    elements, offsets = [], [0]
    for track in obs:
        for i, X in track:
            elements.append((i, len(per[i])))
            per[i].append(project(K[i], R[i], t[i], np.asarray(X, float)))
        offsets.append(len(elements))
    kp = np.zeros(N + 1, np.int64)
    kp[1:] = np.cumsum([len(p) for p in per])
    xy = np.array([x for p in per for x in p], np.float32).reshape(-1, 2)
    return kp, xy, np.array(offsets, np.int64), np.array(elements, np.int32).reshape(-1, 2)


def test_noise_free_two_view_point_is_exact():
    K, R, t = rig([(0, 0, 0), (1, 0, 0)])
    X = np.array([0.5, 0.25, 2.0])                                   # projections (445, 302.5) and (195, 302.5): exact in fp32
    kp, xy, off, el = scene(K, R, t, [[(0, X), (1, X)]])
    assert np.array_equal(xy.astype(np.float64), [[445.0, 302.5], [195.0, 302.5]])
    out = triangulate(kp, xy, off, el, K, R, t)
    assert out["ok"][0] and out["num_inliers"][0] == 2 and out["inlier"].all()
    assert np.abs(out["X"][0] - X).max() <= 1e-9 and out["error"][0] <= 1e-9


def test_a_point_behind_a_camera_is_rejected():
    K, R, t = rig([(0, 0, 0), (1, 0, 0), (0, 0, 4)], flip=(2,))
    X = np.array([0.5, 0.25, 2.0])
    Xb = np.array([0.5, 0.25, 6.0])                                 # in front of camera 2 only
    kp, xy, off, el = scene(K, R, t, [[(0, X), (1, X), (2, Xb)], [(0, Xb), (2, Xb)]])
    out = triangulate(kp, xy, off, el, K, R, t)
    assert out["ok"][0] and out["inlier"][:3].tolist() == [True, True, False] and out["num_inliers"][0] == 2
    assert out["depth"][2] > 0 and out["depth"][0] > 0
    X2 = out["X"][0]
    assert np.abs(X2 - X).max() <= 1e-9
    K2, R2, t2 = rig([(0, 0, 0), (1, 0, 0), (0, 0, 1)], flip=(2,))  # camera 2 now stands beyond X, facing away from it
    kp, xy, off, el = scene(K2, R2, t2, [[(0, X), (2, X)], [(0, X), (1, X), (2, X)]])
    out = triangulate(kp, xy, off, el, K2, R2, t2)
    assert not out["ok"][0] and not out["inlier"][:2].any()          # the only pair puts X behind camera 2
    assert out["ok"][1] and out["inlier"][2:].tolist() == [True, True, False]


def test_min_angle_either_side_of_the_true_angle():
    K, R, t = rig([(0, 0, 0), (1, 0, 0)])
    X = np.array([0.5, 0.25, 2.0])
    a, b = X - np.array([0, 0, 0.0]), X - np.array([1.0, 0, 0])
    true = math.degrees(math.atan2(np.linalg.norm(np.cross(a, b)), a @ b))
    kp, xy, off, el = scene(K, R, t, [[(0, X), (1, X)]])
    assert triangulate(kp, xy, off, el, K, R, t, min_angle=true - 1e-6)["ok"][0]
    out = triangulate(kp, xy, off, el, K, R, t, min_angle=true + 1e-6)
    assert not out["ok"][0] and not out["inlier"].any() and (out["X"] == 0).all() and out["num_inliers"][0] == 0
    assert abs(out["angle_margin"][0] + 1e-6 * math.pi / 180) < 1e-12


@pytest.mark.parametrize("L", [5, 8])
def test_every_pair_up_to_max_hypotheses_then_drawn_pairs(L):
    H = L * (L - 1) // 2
    every = hypothesis_pairs(L, 3, H, 7)
    assert every.tolist() == [[p, q] for p in range(L) for q in range(p + 1, L)]
    drawn = hypothesis_pairs(L, 3, H - 1, 7)
    assert drawn.shape == (H - 1, 2) and (drawn[:, 0] != drawn[:, 1]).all() and ((drawn >= 0) & (drawn < L)).all()
    assert drawn.tolist() == [draw_distinct(2, L, 7, lambda s, h=h: (h, s, 3, CTR)) for h in range(H - 1)]
    assert drawn.tolist() != every[:H - 1].tolist()
    # a clean track comes out the same either way
    K, R, t = rig([(i, 0.1 * i, 0) for i in range(L)])
    X = np.array([0.3, -0.2, 5.0])
    kp, xy, off, el = scene(K, R, t, [[(i, X) for i in range(L)]])
    a, b = (triangulate(kp, xy, off, el, K, R, t, max_hypotheses=m) for m in (H, H - 1))
    assert a["ok"][0] and b["ok"][0] and a["num_inliers"][0] == b["num_inliers"][0] == L
    assert np.abs(a["X"][0] - X).max() < 1e-6 and np.abs(b["X"][0] - X).max() < 1e-6


def test_ties_go_to_the_smallest_hypothesis():
    K, R, t = rig([(0, 0, 0), (1, 0, 0), (0, 1, 0), (1, 1, 0)])
    Xa, Xb = np.array([0.5, 0.25, 2.0]), np.array([-0.7, 0.9, 3.0])
    for first, second in ((Xa, Xb), (Xb, Xa)):
        kp, xy, off, el = scene(K, R, t, [[(0, first), (1, first), (2, second), (3, second)]])
        out = triangulate(kp, xy, off, el, K, R, t)
        assert out["ok"][0] and out["inlier"].tolist() == [True, True, False, False]
        assert np.abs(out["X"][0] - first).max() <= 1e-6                # the fp32 keypoints of Xb are rounded


def test_same_image_pairs_are_skipped():
    K, R, t = rig([(0, 0, 0), (1, 0, 0)])
    X, Y = np.array([0.5, 0.25, 2.0]), np.array([0.1, 0.2, 2.0])
    kp, xy, off, el = scene(K, R, t, [[(0, X), (0, Y)], [(0, X), (0, Y), (1, Y)]])
    out = triangulate(kp, xy, off, el, K, R, t)
    assert not out["ok"][0] and out["hyp_margin"][0] == np.inf       # its only pair shares an image: no hypothesis at all
    assert out["ok"][1] and out["inlier"][2:].tolist() == [False, True, True] and np.abs(out["X"][1] - Y).max() <= 1e-9


def test_a_track_that_repeats_images():
    """Two planted tracks merged into one, as drop_conflicts=False leaves a conflicting component: the pairs within an image are
    skipped, and the point of the more observed track wins with only its observations as inliers."""
    g, tr, views, K, R, t, X = oracle_scene(4, 6, 300, size=(192, 256))
    off, el = tr["track_offsets"], tr["elements"]
    L = np.diff(off)
    a = int(np.flatnonzero(L >= 4)[0])
    b = int(np.flatnonzero((L >= 4) & (L != L[a]))[0])                 # different lengths, so that no tie decides
    la, lb = L[a], L[b]
    merged = np.concatenate((el[off[a]:off[a + 1]], el[off[b]:off[b + 1]]))
    order = np.lexsort((merged[:, 1], merged[:, 0]))                # image ascending, as build_tracks orders a track
    m_off = np.array([0, la + lb], np.int64)
    out = triangulate(g["kp_offsets"], g["keypoints"], m_off, merged[order], K, R, t)
    img = merged[order, 0]
    pq = hypothesis_pairs(la + lb, 0, 256, 0)
    assert (img[pq[:, 0]] == img[pq[:, 1]]).any() and np.unique(img).size < la + lb
    winner = a if la >= lb else b
    ref = triangulate(g["kp_offsets"], g["keypoints"], off[winner:winner + 2] - off[winner], el[off[winner]:off[winner + 1]], K, R, t)
    assert out["ok"][0] and out["num_inliers"][0] == ref["num_inliers"][0]
    assert np.abs(out["X"][0] - ref["X"][0]).max() <= 1e-9 * (1 + np.abs(ref["X"][0]).max())
    from_winner = (order >= la) == (winner == b)
    assert np.array_equal(out["inlier"], from_winner & out["inlier"]) and out["inlier"].sum() == ref["inlier"].sum()


def test_camera_table_is_rule_1():
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(0, 3, 10)
    tab = rb_tri.camera_table(K.numpy(), R.numpy(), t.numpy())
    assert tab.shape == (3, cabi.RB_TRI_CAM) and cabi.RB_TRI_CAM == 20 and cabi.RB_TRI_GN_ITERS == GN_ITERS and cabi.RB_TRI_CTR == CTR
    for i in range(3):
        P = K[i].numpy() @ np.c_[R[i].numpy(), t[i].numpy()]
        assert np.array_equal(tab[i, :12], P.reshape(-1)) and np.array_equal(tab[i, 12:15], R[i, 2].numpy())
        assert tab[i, 15] == t[i, 2] and np.allclose(tab[i, 16:19], -R[i].numpy().T @ t[i].numpy(), atol=1e-12) and tab[i, 19] == 0
    assert CTR != 0x46370000                                            # RB_FUND_CTR
    import roma_b200
    assert "romab200_triangulate" in cabi.FUNCTIONS and roma_b200.triangulate_tracks is rb_tri.triangulate_tracks
    assert roma_b200.Points3D is rb_tri.Points3D


# ---- argument rules -------------------------------------------------------------------------------------------------------
def mg(kp_offsets=(0, 2, 4), keypoints=None):
    kp = torch.tensor(kp_offsets, dtype=torch.int64)
    xy = torch.zeros(int(kp[-1]), 2) if keypoints is None else keypoints
    return MatchGraph(kp, xy, torch.zeros(int(kp[-1])), torch.zeros(2, dtype=torch.int64), torch.zeros(0, 2, dtype=torch.int32), torch.zeros(0))


def tk(offsets=(0, 2), elements=((0, 0), (1, 1))):
    el = elements if isinstance(elements, torch.Tensor) else torch.tensor(elements, dtype=torch.int32).reshape(-1, 2)
    off = offsets if isinstance(offsets, torch.Tensor) else torch.tensor(offsets, dtype=torch.int64)
    return Tracks(off, el, torch.zeros(4, dtype=torch.int32), 0)


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


CAM = dict(K=np.repeat(KF[None], 2, 0), R=np.repeat(np.eye(3)[None], 2, 0), t=np.array([[0.0, 0, 0], [-1, 0, 0]]))


@pytest.mark.parametrize("case", [
    dict(graph={"kp_offsets": torch.zeros(1, dtype=torch.int64)}),               # not a MatchGraph
    dict(tracks=(torch.zeros(1, dtype=torch.int64), torch.zeros(0, 2))),          # not Tracks
    dict(graph=mg(kp_offsets=(0, 3, 2))),                                          # decreasing
    dict(graph=mg(kp_offsets=(1, 2, 4))),                                          # not starting at 0
    dict(graph=mg(keypoints=torch.zeros(4, 2, dtype=torch.float64))),
    dict(graph=mg(keypoints=torch.zeros(3, 2))),
    dict(tracks=tk(offsets=(0, 3, 2), elements=((0, 0), (1, 1), (1, 0)))),
    dict(tracks=tk(offsets=(1, 2))),
    dict(tracks=tk(offsets=torch.tensor([0, 2], dtype=torch.int32))),
    dict(tracks=tk(elements=torch.zeros(2, 2, dtype=torch.int64))),
    dict(tracks=tk(elements=torch.zeros(3, 2, dtype=torch.int32))),
    dict(K=np.repeat(KF[None], 3, 0)),                                             # not N cameras
    dict(R=np.eye(3)),
    dict(t=np.zeros((2, 4))),
    dict(t=np.array([[0.0, 0, 0], [np.nan, 0, 0]])),
    dict(K=np.repeat(np.eye(3, dtype=np.int64)[None], 2, 0)),                      # not a float dtype
    dict(R=torch.tensor([[[1.0, 0, 0], [0, 1, 0], [0, 0, math.inf]]] * 2)),
    dict(max_error=0.0), dict(max_error=-1.0), dict(max_error=math.inf), dict(max_error=math.nan), dict(max_error="four"),
    dict(min_angle=-0.1), dict(min_angle=180.0), dict(min_angle=math.nan),
    dict(max_hypotheses=0), dict(max_hypotheses=2.0), dict(max_hypotheses=True), dict(max_hypotheses=1 << 31),
    dict(seed=-1), dict(seed=1.5),
    dict(graph=mg(kp_offsets=(0, 0, 0))),                                          # no keypoints but elements
    {},                                                                             # CPU tensors: the call runs on a CUDA device only
])
def test_argument_errors_before_device_work(no_device, case):
    kw = dict(graph=mg(), tracks=tk(), **CAM)
    kw.update(case)
    with pytest.raises(ValueError) as e:
        rb_tri.triangulate_tracks(kw.pop("graph"), kw.pop("tracks"), kw.pop("K"), kw.pop("R"), kw.pop("t"), **kw)
    assert ("CUDA device" in str(e.value)) == (not case)          # each case fails its own rule, not the device rule


def test_cameras_are_widened_from_any_float_dtype():
    K, R, t = (torch.tensor(v, dtype=torch.float32) for v in (CAM["K"], CAM["R"], CAM["t"]))
    with pytest.raises(ValueError, match="CUDA device"):
        rb_tri.triangulate_tracks(mg(), tk(), K, R, t.half())


def test_oracle_rejects_element_ids_out_of_range():
    K, R, t = rig([(0, 0, 0), (1, 0, 0)])
    kp, xy, off, el = scene(K, R, t, [[(0, np.array([0, 0, 2.0])), (1, np.array([0, 0, 2.0]))]])
    for bad in ((0, 1), (2, 0), (-1, 0), (1, -1)):
        e2 = el.copy()
        e2[1] = bad
        with pytest.raises(ValueError, match="outside"):
            triangulate(kp, xy, off, e2, K, R, t)


# ---- the helper and the robustness bars ------------------------------------------------------------------------------------
def oracle_scene(seed, N, points, cell_size=1, size=(768, 1024)):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cell_size)
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy(), cell_size=cell_size)
    return g, oracle_tracks(pairs.numpy(), g), views, K, R, t, X


def test_track_points_maps_tracks_to_planted_points():
    g, tr, views, K, R, t, X = oracle_scene(5, 5, 300, size=(192, 256))
    args = [torch.from_numpy(a) for a in (tr["track_offsets"], tr["elements"], g["kp_offsets"], g["keypoints"])]
    pts = synthetic.track_points(*args, views, 256)
    T = len(tr["track_offsets"]) - 1
    assert pts.shape == (T,) and (pts >= 0).all() and np.unique(pts).size == T
    v = views.numpy()
    found = synthetic.track_cells(*args, 256)
    assert found == {tuple((i, int(v[p, i])) for i in range(v.shape[1]) if v[p, i] >= 0) for p in pts}
    el = tr["elements"].copy()
    el[[0, 1]] = el[[tr["track_offsets"][1], tr["track_offsets"][2]]]   # track 0 now mixes the first elements of tracks 1 and 2
    pts2 = synthetic.track_points(args[0], torch.from_numpy(el), *args[2:], views, 256)
    assert pts2[0] == -1 and np.array_equal(pts2[3:], pts[3:])
    assert synthetic.track_points(torch.zeros(1, dtype=torch.int64), torch.zeros(0, 2, dtype=torch.int32), *args[2:], views, 256).size == 0


def move_observations(kp_offsets, keypoints, track_offsets, elements, frac, seed):
    """Moves `frac` of the observations of tracks of 3 elements or more by 20-50 px in a uniform direction: (keypoints, moved [E])."""
    rng = np.random.default_rng(seed)
    off, el = np.asarray(track_offsets), np.asarray(elements).astype(np.int64)
    L = np.diff(off)
    eligible = np.repeat(L >= 3, L)
    moved = eligible & (rng.random(el.shape[0]) < frac)
    ang = rng.uniform(0, 2 * np.pi, moved.sum())
    r = rng.uniform(20, 50, moved.sum())
    xy = np.array(keypoints, np.float32, copy=True)
    rows = np.asarray(kp_offsets)[el[moved, 0]] + el[moved, 1]
    xy[rows] += np.stack((r * np.cos(ang), r * np.sin(ang)), 1).astype(np.float32)
    return xy, moved


def test_robustness_to_moved_observations():
    g, tr, views, K, R, t, X = oracle_scene(1, 16, 1000)
    xy, moved = move_observations(g["kp_offsets"], g["keypoints"], tr["track_offsets"], tr["elements"], 0.1, 0)
    out = triangulate(g["kp_offsets"], xy, tr["track_offsets"], tr["elements"], K, R, t)
    rejected, kept, accepted = (~out["inlier"][moved]).mean(), out["inlier"][~moved].mean(), out["ok"].mean()
    print(f"moved {moved.sum()} of {moved.size}: rejected {rejected:.4f}, others kept {kept:.4f}, tracks accepted {accepted:.4f}")
    assert moved.sum() > 500 and rejected >= 0.99 and kept >= 0.995 and accepted >= 0.99
