"""CPU checks of the pose estimator's restatement (oracle/pose_ransac.py) against known geometry and OpenCV, and of the host side
of `roma_b200.estimate_pose` that runs without a GPU."""
import os
import re

import numpy as np
import pytest

from oracle import pose_ransac as pr
from roma_b200 import synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def _unit_E(R, t):
    E = (_skew(t) @ R).ravel()
    E = E / np.linalg.norm(E)
    return -E if E[np.argmax(np.abs(E))] < 0 else E


def _normalised(scene):
    return np.concatenate([pr.normalise(scene["kpts0"], scene["K0"]), pr.normalise(scene["kpts1"], scene["K1"])], axis=1)


def test_philox_known_answers():
    # Random123 kat_vectors, philox4x32 with 10 rounds
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        assert tuple(int(v) for v in pr.philox4x32_10(np.array(ctr, dtype=np.uint64), key)) == want


def test_samples_distinct_and_in_range():
    for h in range(200):
        s = pr.draw_sample(h, 3, 7, seed=11)
        assert len(set(s)) == 5 and all(0 <= v < 7 for v in s)


def test_header_constants_match():
    from roma_b200 import geometry
    text = open(os.path.join(ROOT, "include", "romab200.h")).read()
    got = {k: int(v) for k, v in re.findall(r"#define RB_POSE_(\w+) (\d+)", text)}
    assert (got["ROUND"], got["MAX_SOL"], got["MAX_SPLITS"], got["STATE"]) == (geometry.ROUND, geometry.MAX_SOL, geometry.MAX_SPLITS, geometry.STATE)


def test_five_point_recovers_planted_E():
    # a planted E that sits next to another solution (a near-double root of the degree-10 polynomial) is only determined to
    # ~sqrt(eps): all samples recover it to 1e-5, and all but a few to 1e-9
    close = []
    for seed in range(40):
        sc = synthetic.two_view_scene(seed, 5, 0.0, noise=0.0)
        xn = _normalised(sc)
        sols = pr.solve_five_point(xn[None])[0]
        assert 1 <= len(sols) <= 10
        E0 = _unit_E(sc["R"], sc["t"])
        d = min(np.abs(s - E0).max() for s in sols)
        assert d < 1e-5
        close.append(d < 1e-9)
        _check_solutions(sols, xn, 1e-6 if d < 1e-9 else 1e-3)
    assert np.mean(close) >= 0.9


def _check_solutions(sols, xn, tol):
    for s in sols:
        E = s.reshape(3, 3)
        assert abs(np.linalg.det(E)) < tol
        assert np.abs(2 * E @ E.T @ E - np.trace(E @ E.T) * E).max() < tol
        x0 = np.c_[xn[:, :2], np.ones(5)]
        x1 = np.c_[xn[:, 2:], np.ones(5)]
        assert np.abs(np.einsum("ni,ij,nj->n", x1, E, x0)).max() < tol


@pytest.mark.parametrize("seed", range(5))
def test_recover_pose_matches_cv2(seed):
    cv2 = pytest.importorskip("cv2")
    sc = synthetic.two_view_scene(100 + seed, 2000, 0.3)
    xn = _normalised(sc)
    E = _unit_E(sc["R"], sc["t"]).reshape(3, 3)
    mask = pr.inlier_mask(E.ravel(), xn, 0.5 / 1200)[0]
    m8 = mask.astype(np.uint8)[:, None].copy()
    n_cv, R_cv, t_cv, m_cv = cv2.recoverPose(E, xn[:, :2].copy(), xn[:, 2:].copy(), np.eye(3), 1e9, mask=m8)
    n, R, t, m = pr.recover_pose(E, xn, mask)
    assert n == n_cv
    assert np.abs(R - R_cv).max() < 1e-9 and np.abs(t - t_cv).max() < 1e-9
    assert np.array_equal(m, m_cv.ravel() > 0)


def _reference_estimate_pose(cv2, kpts0, kpts1, K0, K1, norm_thresh, conf=0.99999):
    """romatch/utils/utils.py:30-51, restated with cv2."""
    K0inv, K1inv = np.linalg.inv(K0[:2, :2]), np.linalg.inv(K1[:2, :2])
    k0 = (K0inv @ (kpts0 - K0[None, :2, 2]).T).T
    k1 = (K1inv @ (kpts1 - K1[None, :2, 2]).T).T
    E, mask = cv2.findEssentialMat(k0, k1, np.eye(3), threshold=norm_thresh, prob=conf)
    ret = None
    if E is not None:
        best = 0
        for _E in np.split(E, len(E) / 3):
            n, R, t, _ = cv2.recoverPose(_E, k0, k1, np.eye(3), 1e9, mask=mask)
            if n > best:
                best = n
                ret = (R, t, mask.ravel() > 0)
    return ret


def pose_error(R, t, R_gt, t_gt):
    """Angular errors in degrees as RoMa's pose benchmarks compute them (t up to sign)."""
    ct = np.dot(t.ravel(), t_gt) / (np.linalg.norm(t) * np.linalg.norm(t_gt))
    et = np.rad2deg(np.arccos(np.clip(ct, -1.0, 1.0)))
    et = min(et, 180 - et)
    cr = (np.trace(R.T @ R_gt) - 1) / 2
    return max(et, np.rad2deg(np.abs(np.arccos(np.clip(cr, -1.0, 1.0)))))


def pose_auc(errors, thresholds=(5, 10, 20)):
    errors = np.sort(np.r_[0.0, np.asarray(errors)])
    recall = np.r_[0.0, (np.arange(len(errors) - 1) + 1) / (len(errors) - 1)]
    out = []
    for th in thresholds:
        last = np.searchsorted(errors, th)
        r = np.r_[recall[:last], recall[last - 1]]
        e = np.r_[errors[:last], th]
        out.append(np.trapezoid(r, x=e) / th)
    return out


# Tolerances set from 30 scenes (N = 5 000, outliers 10-60 %, threshold 0.5 px / (f0 + f1), i.e. ~0.25 px against 0.5 px of
# noise, so only about a third of the true matches pass it and the final count depends on which model RANSAC stops at).  The
# restated estimator and OpenCV draw different samples; measured between them: per-scene relative inlier-count difference
# median 4.8 % (largest 42 %), total count -1.4 %, AUC@5/10/20 0.909/0.954/0.977 against 0.922/0.961/0.981.
COUNT_MEDIAN_RTOL = 0.10
COUNT_TOTAL_RTOL = 0.05
AUC_TOL = 0.03


def scene_set():
    return [(s, 0.1 + 0.5 * (s % 6) / 5) for s in range(30)]


def check_statistics(counts, counts_cv2, errs, errs_cv2):
    counts, counts_cv2 = np.asarray(counts, float), np.asarray(counts_cv2, float)
    assert np.median(np.abs(counts - counts_cv2) / counts_cv2) <= COUNT_MEDIAN_RTOL
    assert abs(counts.sum() / counts_cv2.sum() - 1) <= COUNT_TOTAL_RTOL
    auc, auc_cv2 = pose_auc(errs), pose_auc(errs_cv2)
    assert np.abs(np.array(auc) - np.array(auc_cv2)).max() <= AUC_TOL, (auc, auc_cv2)


def test_estimate_pose_statistically_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    errs_o, errs_c, n_o, n_c = [], [], [], []
    for seed, frac in scene_set():
        sc = synthetic.two_view_scene(1000 + seed, 5000, frac)
        thr = 0.5 / (sc["K0"][0, 0] + sc["K1"][0, 0])
        ro = pr.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], thr, seed=seed)
        rc = _reference_estimate_pose(cv2, sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], thr)
        assert ro is not None and rc is not None
        errs_o.append(pose_error(ro[0], ro[1], sc["R"], sc["t"]))
        errs_c.append(pose_error(rc[0], rc[1], sc["R"], sc["t"]))
        n_o.append(int(ro[2].sum()))
        n_c.append(int(rc[2].sum()))
    check_statistics(n_o, n_c, errs_o, errs_c)


def test_edge_cases():
    sc = synthetic.two_view_scene(7, 50, 0.0)
    k0, k1, K0, K1 = sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"]
    assert pr.estimate_pose(k0[:4], k1[:4], K0, K1, 1e-3) is None
    r5 = pr.estimate_pose(k0[:5], k1[:5], K0, K1, 1e-3)
    assert r5 is not None and r5[2].shape == (5,)
    same = np.repeat(k0[:1], 50, axis=0)
    assert pr.estimate_pose(same, same, K0, K1, 1e-3) is None
    k0n = k0.copy()
    k0n[::7] = np.nan
    r = pr.estimate_pose(k0n, k1, K0, K1, 1e-3)
    assert r is not None and not r[2][::7].any()


def test_no_gpu_raises(monkeypatch):
    torch = pytest.importorskip("torch")
    from roma_b200 import geometry
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    sc = synthetic.two_view_scene(0, 20, 0.0)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        geometry.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], 1e-3)
    assert geometry.estimate_pose(sc["kpts0"][:4], sc["kpts1"][:4], sc["K0"], sc["K1"], 1e-3) is None
