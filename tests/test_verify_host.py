"""CPU tests of geometric verification (`verify_matches`): the numpy oracle on hand-built graphs (P = 0 and M = 0, a pair of fewer
than 7 matches, num_inliers equal to min_inliers, a rejected pair between accepted ones, match order, the points each pair reads),
the oracle with the numpy estimator on small `planted_cameras` scenes, the chunk planner and its byte formula against the buffers
`geometry._fund_launch` allocates, every argument rule (raised before any device work), and the geometric generator."""
import numpy as np
import pytest
import torch

from oracle.fundamental_ransac import sampson2
from oracle.match_graph import consolidate
from oracle.verify import host_estimator, pair_points, verify
from roma_b200 import cabi, geometry, synthetic, verify as rb_verify
from roma_b200.match_graph import MatchGraph


def graph(kp_counts, pair_matches, keypoints=None):
    """A MatchGraph-like dict: kp_counts[i] keypoints in image i (row r at (r, 2 r) unless given); pair_matches[k] = [(a, b), ...]."""
    kp = np.zeros(len(kp_counts) + 1, np.int64)
    kp[1:] = np.cumsum(kp_counts)
    mo = np.zeros(len(pair_matches) + 1, np.int64)
    mo[1:] = np.cumsum([len(m) for m in pair_matches])
    rows = [m for ms in pair_matches for m in ms]
    K = int(kp[-1])
    xy = np.stack((np.arange(K), 2 * np.arange(K)), 1).astype(np.float32) if keypoints is None else keypoints
    return dict(kp_offsets=kp, keypoints=xy, match_offsets=mo, matches=np.array(rows, np.int32).reshape(-1, 2),
                match_scores=np.arange(len(rows), dtype=np.float32) + 0.5)


def fixed(masks, models=None):
    """An estimator that returns masks[k] (and a model unless models[k] is None) for pair k, recording the calls."""
    calls = []

    def estimate(k, x0, x1):
        calls.append(k)
        F = np.eye(3) if models is None or models[k] is not None else None
        return F, np.asarray(masks[k], bool)

    estimate.calls = calls
    return estimate


def test_no_pairs_and_no_matches():
    r = verify(np.zeros((0, 2)), graph([3, 2], []), fixed([]))
    assert r["match_offsets"].tolist() == [0] and r["matches"].shape == (0, 2) and r["F"].shape == (0, 3, 3)
    est = fixed([[]] * 2)
    r = verify([(0, 1), (1, 0)], graph([3, 2], [[], []]), est)
    assert r["match_offsets"].tolist() == [0, 0, 0] and not r["ok"].any() and not r["accepted"].any() and est.calls == []
    assert r["num_inliers"].tolist() == [0, 0] and (r["F"] == 0).all()


def test_fewer_than_seven_matches_get_no_model():
    ms = [[(a, a) for a in range(6)], [(a, a) for a in range(7)]]
    est = fixed([None, [1] * 7])
    r = verify([(0, 1), (0, 1)], graph([8, 8], ms), est, min_inliers=0)
    assert est.calls == [1] and r["ok"].tolist() == [False, True] and r["accepted"].tolist() == [False, True]
    assert r["match_offsets"].tolist() == [0, 0, 7] and (r["F"][0] == 0).all()


def test_min_inliers_is_inclusive_and_a_rejected_pair_keeps_nothing():
    ms = [[(a, a) for a in range(10)]] * 3
    masks = [[1] * 8 + [0] * 2, [1] * 7 + [0] * 3, [0, 1] * 5]
    r = verify([(0, 1), (1, 2), (0, 2)], graph([10, 10, 10], ms), fixed(masks), min_inliers=5)
    assert r["num_inliers"].tolist() == [8, 7, 5] and r["accepted"].tolist() == [True, True, True]
    r = verify([(0, 1), (1, 2), (0, 2)], graph([10, 10, 10], ms), fixed(masks), min_inliers=8)
    assert r["accepted"].tolist() == [True, False, False] and r["match_offsets"].tolist() == [0, 8, 8, 8]
    masks[2] = [1] * 9 + [0]
    r = verify([(0, 1), (1, 2), (0, 2)], graph([10, 10, 10], ms), fixed(masks), min_inliers=8)
    assert r["accepted"].tolist() == [True, False, True] and r["match_offsets"].tolist() == [0, 8, 8, 17]
    assert r["match_scores"].tolist() == [m + 0.5 for m in list(range(8)) + list(range(20, 29))]


def test_a_pair_without_a_model_is_rejected_whatever_its_mask():
    ms = [[(a, a) for a in range(9)]] * 2
    r = verify([(0, 1), (0, 1)], graph([9, 9], ms), fixed([[1] * 9, [1] * 9], models=[None, 1]), min_inliers=0)
    assert r["ok"].tolist() == [False, True] and r["accepted"].tolist() == [False, True] and r["match_offsets"].tolist() == [0, 0, 9]


def test_matches_keep_their_order_and_scores():
    ms = [[(0, 4), (2, 1), (3, 3), (5, 0), (6, 6), (7, 2), (8, 5), (9, 7)]]
    r = verify([(0, 1)], graph([10, 8], ms), fixed([[0, 1, 1, 0, 1, 1, 0, 1]]), min_inliers=1)
    assert r["matches"].tolist() == [[2, 1], [3, 3], [6, 6], [7, 2], [9, 7]]
    assert r["match_scores"].tolist() == [1.5, 2.5, 4.5, 5.5, 7.5] and r["matches"].dtype == np.int32


def test_pair_points_read_the_keypoints_of_each_side():
    g = graph([3, 2, 4], [[(2, 1), (0, 0)], [(3, 1)], [(1, 1)]])
    pts = pair_points([(0, 1), (2, 1), (2, 2)], g)
    assert pts[0][0].tolist() == [[2, 4], [0, 0]] and pts[0][1].tolist() == [[4, 8], [3, 6]]
    assert pts[1][0].tolist() == [[8, 16]] and pts[1][1].tolist() == [[4, 8]]
    assert pts[2][0].tolist() == pts[2][1].tolist() == [[6, 12]] and pts[2][0].dtype == np.float64
    with pytest.raises(ValueError):
        pair_points([(0, 1)], graph([3, 2], [[(0, 2)]]))


def planted_labels(pairs, g, views, width, cell_size):
    """Per match of g: True when its two keypoints' cells are one planted point's views in the pair's images."""
    kp, xy, mo, m = g["kp_offsets"], g["keypoints"], g["match_offsets"], g["matches"].astype(np.int64)
    gw = -(-width // cell_size)
    cell = (np.floor(xy[:, 1]).astype(np.int64) // cell_size) * gw + np.floor(xy[:, 0]).astype(np.int64) // cell_size
    v = views.cpu().numpy() if hasattr(views, "cpu") else views
    point = [dict((int(c), p) for p, c in enumerate(v[:, i]) if c >= 0) for i in range(v.shape[1])]
    out = np.zeros(m.shape[0], bool)
    for k, (i, j) in enumerate(np.asarray(pairs)):
        for q in range(mo[k], mo[k + 1]):
            pa = point[i].get(int(cell[kp[i] + m[q, 0]]), -1)
            out[q] = pa >= 0 and pa == point[j].get(int(cell[kp[j] + m[q, 1]]), -2)
    return out


@pytest.mark.parametrize("seed, cell_size, threshold", [(0, 1, 2.0), (2, 1, 2.0), (3, 4, 3.0)])
def test_oracle_with_the_numpy_estimator_removes_planted_outliers(seed, cell_size, threshold):
    pairs, m, c, sizes, views = synthetic.planted_cameras(seed, 3, 300, size=(384, 512), cell_size=cell_size, outlier_frac=0.2)[:5]
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy(), cell_size=cell_size)
    inlier = planted_labels(pairs.numpy(), g, views, 512, cell_size)
    assert inlier.sum() > 200 and (~inlier).sum() > 40
    r = verify(pairs.numpy(), g, host_estimator(threshold, 0.999, 10000), min_inliers=15)
    assert r["accepted"].all()
    kept = np.zeros(len(inlier), bool)
    mo = g["match_offsets"]
    for k in range(len(pairs)):
        got = {tuple(x) for x in r["matches"][r["match_offsets"][k]:r["match_offsets"][k + 1]].tolist()}
        kept[mo[k]:mo[k + 1]] = [tuple(x) in got for x in g["matches"][mo[k]:mo[k + 1]].tolist()]
    assert kept[inlier].mean() >= 0.95 and (~kept[~inlier]).mean() >= 0.95


# ---- the chunk planner -----------------------------------------------------------------------------------------------------
def test_chunk_bytes_equal_the_buffers_of_the_estimator(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: None)          # the buffers only: nothing reaches the device
    for ns in ([0], [7], [1, 600, 3], [512, 513], [2000, 0, 0, 1500], [0, 0]):
        total = sum(ns)
        x0, x1 = torch.zeros(max(total, 1), 2, dtype=torch.float64), torch.zeros(max(total, 1), 2, dtype=torch.float64)
        off = torch.tensor(np.r_[0, np.cumsum(ns)], dtype=torch.int64)
        buf = geometry._fund_launch(x0, x1, off, max(ns), 2.0, 0.999, 1, 0)
        got = sum(t.numel() * t.element_size() for t in buf.values()) + sum(t.numel() * t.element_size() for t in (x0, x1, off))
        assert rb_verify.chunk_bytes(ns) == got, ns


@pytest.mark.parametrize("seed", range(5))
def test_chunks_are_consecutive_and_keep_the_budget(seed):
    rng = np.random.default_rng(seed)
    ns = rng.integers(0, 5000, int(rng.integers(1, 60))).tolist()
    if seed == 4:
        ns[3] = 200_000                                                # over the budget alone
    for budget in (1, 3 << 20, 12 << 20, 1 << 30):
        chunks = rb_verify.plan_chunks(ns, budget)
        assert chunks[0][0] == 0 and chunks[-1][1] == len(ns) and all(e0 == b1 for (_, e0), (b1, _) in zip(chunks, chunks[1:]))
        for b, e in chunks:
            assert e > b
            assert rb_verify.chunk_bytes(ns[b:e]) <= budget or e == b + 1
            if e < len(ns):                                            # as long as the budget allows
                assert rb_verify.chunk_bytes(ns[b:e + 1]) > budget
    assert rb_verify.plan_chunks(ns, 1) == [(k, k + 1) for k in range(len(ns))]
    assert len(rb_verify.plan_chunks([10] * 4, 1 << 40)) == 1 and rb_verify.plan_chunks([], 1) == []


# ---- argument rules --------------------------------------------------------------------------------------------------------
def mg(kp_offsets=(0, 2, 4, 6), match_offsets=(0, 1, 2), matches=((0, 1), (1, 0)), scores=(1.0, 1.0), keypoints=None):
    def t(x, dtype):
        return x if isinstance(x, torch.Tensor) else torch.tensor(x, dtype=dtype)

    kp = t(kp_offsets, torch.int64)
    return MatchGraph(kp, torch.zeros(int(kp[-1]), 2) if keypoints is None else keypoints, torch.zeros(1), t(match_offsets, torch.int64),
                      t(matches, torch.int32).reshape(-1, 2), t(scores, torch.float32))


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case, exc", [
    (dict(graph={"kp_offsets": torch.zeros(1, dtype=torch.int64)}), ValueError),   # not a MatchGraph
    (dict(graph=mg(kp_offsets=(0, 2, 1, 6))), ValueError),                          # decreasing
    (dict(graph=mg(kp_offsets=(1, 2, 4, 6))), ValueError),
    (dict(graph=mg(match_offsets=(0, 2, 1))), ValueError),
    (dict(graph=mg(kp_offsets=torch.tensor([0, 2, 4, 6], dtype=torch.int32))), ValueError),
    (dict(graph=mg(matches=((0, 1), (1, 0), (1, 1)))), ValueError),                 # more matches than match_offsets[P]
    (dict(graph=mg(matches=torch.zeros(2, 2, dtype=torch.int64))), ValueError),
    (dict(graph=mg(scores=(1.0,))), ValueError),
    (dict(graph=mg(keypoints=torch.zeros(6, 2, dtype=torch.float64))), ValueError),
    (dict(graph=mg(keypoints=torch.zeros(5, 2))), ValueError),
    (dict(graph=mg(kp_offsets=(0, 0, 0, 0))), ValueError),                          # matches but no keypoints
    (dict(pairs=[(0, 3)]), IndexError),
    (dict(pairs=[(0, 1)]), ValueError),                                             # P mismatch
    (dict(pairs=[(0, 1), (1, 2), (0, 2)]), ValueError),
    (dict(threshold=0.0), ValueError),
    (dict(threshold=-1.0), ValueError),
    (dict(threshold=float("nan")), ValueError),
    (dict(threshold=float("inf")), ValueError),
    (dict(threshold="2x"), ValueError),
    (dict(confidence=0.0), ValueError),
    (dict(confidence=1.0), ValueError),
    (dict(confidence=float("nan")), ValueError),
    (dict(max_iters=0), ValueError),
    (dict(max_iters=2.5), ValueError),
    (dict(min_inliers=-1), ValueError),
    (dict(min_inliers=15.0), ValueError),
    (dict(min_inliers=True), ValueError),
    (dict(workspace_bytes=0), ValueError),
    (dict(workspace_bytes=1.5), ValueError),
    ({}, ValueError),                                                               # CPU tensors: the call runs on a CUDA device only
])
def test_argument_errors_before_device_work(no_device, case, exc):
    kw = dict(pairs=[(0, 1), (1, 2)], graph=mg())
    kw.update(case)
    pairs, g = kw.pop("pairs"), kw.pop("graph")
    with pytest.raises(exc) as e:
        rb_verify.verify_matches(pairs, g, **kw)
    assert ("CUDA device" in str(e.value)) == (not case)          # each case fails its own rule, not the device rule


def test_entry_points_and_exports():
    import roma_b200
    assert {"romab200_verify_check", "romab200_verify_gather", "romab200_verify_count", "romab200_verify_emit"} <= set(cabi.FUNCTIONS)
    assert roma_b200.verify_matches is rb_verify.verify_matches and roma_b200.PairGeometry is rb_verify.PairGeometry
    assert cabi.RB_VERIFY_TILE == 4096 and rb_verify.WORKSPACE_BYTES == 1 << 30


# ---- the geometric generator -----------------------------------------------------------------------------------------------
def test_planted_cameras_shapes_and_outliers():
    out = synthetic.planted_cameras(1, 4, 300, size=(96, 128), outlier_frac=0.2)
    pairs, m, c, sizes, views, K, R, t, X = out
    assert pairs.tolist() == [[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]] and sizes.tolist() == [[96, 128]] * 4
    assert m.shape[:2] == c.shape and views.shape == (300, 4) and K.shape == R.shape == (4, 3, 3) and t.shape == (4, 3)
    assert X.shape == (300, 3) and K.dtype == R.dtype == t.dtype == X.dtype == torch.float64
    inl = ((views[:, pairs[:, 0]] >= 0) & (views[:, pairs[:, 1]] >= 0)).sum(0)
    assert torch.equal((c >= 0.5).sum(1), inl) and inl.min() > 30
    assert torch.equal(((c > 0) & (c < 0.5)).sum(1), torch.round(inl * 0.25).long())
    assert (m.abs() <= 1).all()
    assert torch.allclose(R @ R.transpose(1, 2), torch.eye(3, dtype=torch.float64).expand(4, 3, 3)) and (torch.linalg.det(R) > 0).all()
    a = synthetic.planted_cameras(1, 4, 300, size=(96, 128), outlier_frac=0.2)
    assert all(torch.equal(x, y) for x, y in zip(out, a))


@pytest.mark.parametrize("cell_size", [1, 4])
def test_planted_cameras_cells_are_distinct_and_are_the_match_graph_cells(cell_size):
    pairs, m, c, sizes, views = synthetic.planted_cameras(2, 4, 2000, size=(96, 128), cell_size=cell_size, visibility=0.8)[:5]
    v = views.numpy()
    for i in range(4):
        seen = v[:, i][v[:, i] >= 0]
        assert seen.size > 100 and np.unique(seen).size == seen.size
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy(), cell_size=cell_size)
    gw = -(-128 // cell_size)
    xy = g["keypoints"]
    cell = (np.floor(xy[:, 1]).astype(np.int64) // cell_size) * gw + np.floor(xy[:, 0]).astype(np.int64) // cell_size
    kp = g["kp_offsets"]
    shared = (v >= 0).sum(1) >= 2                                  # points seen by two images or more have samples
    for i in range(4):
        assert sorted(cell[kp[i]:kp[i + 1]].tolist()) == sorted(v[shared, i][v[shared, i] >= 0].tolist())
    assert planted_labels(pairs.numpy(), g, views, 128, cell_size).all()


@pytest.mark.parametrize("noise, cell_size", [(0.5, 1), (1.0, 1), (0.5, 4)])
def test_planted_cameras_inliers_lie_on_the_true_epipolar_geometry(noise, cell_size):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(3, 5, 1500, noise=noise, cell_size=cell_size, outlier_frac=0.2)
    H, W = sizes[0].tolist()
    med, outl = [], []
    for k, (i, j) in enumerate(pairs.tolist()):
        Rr = R[j] @ R[i].T
        tr = t[j] - Rr @ t[i]
        tx = torch.tensor([[0, -tr[2], tr[1]], [tr[2], 0, -tr[0]], [-tr[1], tr[0], 0]], dtype=torch.float64)
        F = (torch.linalg.inv(K[j]).T @ tx @ Rr @ torch.linalg.inv(K[i])).numpy()
        F = F / np.linalg.norm(F)
        mk = m[k].double().numpy()
        x0 = np.stack(((mk[:, 0] + 1) * W / 2, (mk[:, 1] + 1) * H / 2), 1)
        x1 = np.stack(((mk[:, 2] + 1) * W / 2, (mk[:, 3] + 1) * H / 2), 1)
        d = np.sqrt(sampson2(F.reshape(-1), x0, x1))
        inl = c[k].numpy() >= 0.5
        med.append(np.median(d[inl]))
        outl.append(np.median(d[(c[k].numpy() > 0) & ~inl]))
    # the true residual: the noise plus a cell's quantisation and a sample's quarter-cell jitter (about 0.3 cell_size rms)
    bound = noise + 0.35 * cell_size
    assert max(med) < bound and min(med) > 0.2 * noise and min(outl) > 10 * bound
