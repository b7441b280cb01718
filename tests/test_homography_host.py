"""CPU checks of the homography estimator's restatement (oracle/homography_ransac.py) against OpenCV, and of the host side of
`roma_b200.find_homography` that runs without a GPU."""
import os
import re

import numpy as np
import pytest

from oracle import homography_ransac as hr
from roma_b200 import synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _f32(sc):
    return sc["src"].astype(np.float32), sc["dst"].astype(np.float32)


def _corner_diff(Ha, Hb, size=(640, 480)):
    return float(np.abs(hr.corners(Ha, *size) - hr.corners(Hb, *size)).max())


def test_header_constants_match():
    from roma_b200 import geometry
    text = open(os.path.join(ROOT, "include", "romab200.h")).read()
    got = {k: int(v) for k, v in re.findall(r"#define RB_HOMOG_(\w+) (\d+)", text)}
    assert (got["ROUND"], got["MAX_SPLITS"], got["STATE"], got["MAX_ATTEMPTS"]) == (
        geometry.HOMOG_ROUND, geometry.HOMOG_MAX_SPLITS, geometry.HOMOG_STATE, hr.MAX_ATTEMPTS)
    assert geometry.RANSAC == hr.RANSAC == 8


def test_subsets_distinct_and_in_range():
    sc = synthetic.planar_scene(0, 7, 0.0)
    src, dst = _f32(sc)
    for h in range(100):
        idx, att, found = hr.draw_subset(h, 2, 7, 11, src, dst)
        assert found and len(set(idx)) == 4 and all(0 <= v < 7 for v in idx)
        assert hr.check_subset(src[idx], dst[idx])


def test_check_subset_rejects_collinear_and_flipped():
    sq = np.array([[0, 0], [100, 0], [100, 100], [0, 100]], dtype=np.float32)
    assert hr.check_subset(sq, sq + 5)
    line = np.array([[0, 0], [10, 10], [20, 20], [5, 40]], dtype=np.float32)
    assert hr.check_subset(line, sq)                       # points 0, 1, 2 are collinear, but OpenCV tests the last point only
    line2 = np.array([[0, 0], [10, 10], [5, 40], [20, 20]], dtype=np.float32)
    assert not hr.check_subset(line2, sq)
    assert not hr.check_subset(sq, sq[[0, 1, 3, 2]])          # a bow-tie: the four triples do not keep one orientation


def test_four_point_solver_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    worst = 0.0
    for s in range(20):
        src, dst = _f32(synthetic.planar_scene(200 + s, 4, 0.0))
        Hc, _ = cv2.findHomography(src, dst, 0)
        Ho = hr.solve_four(src, dst)
        worst = max(worst, _corner_diff(Hc, Ho))
    assert worst < 1e-6, worst


def test_refinement_matches_cv2():
    """method 0 is the normalised DLT plus Levenberg-Marquardt over all points; the DLT alone is ~1e-2 px off cv2."""
    cv2 = pytest.importorskip("cv2")
    worst = 0.0
    for s in range(20):
        src, dst = _f32(synthetic.planar_scene(300 + s, 800, 0.0))
        Hc, mc = cv2.findHomography(src, dst, 0)
        Ho, mo = hr.find_homography(src, dst, 0)
        assert mc.ravel().all() and mo.all()
        worst = max(worst, _corner_diff(Hc, Ho))
    assert worst < 1e-4, worst


def scene_set():
    return [(s, (500, 1000, 2000)[s % 3], (0.2, 0.5, 0.7)[(s // 3) % 3]) for s in range(30)]


def test_opencv_stream_replays_cv2():
    """With OpenCV's own sample stream (cv::RNG, getSubset) and solver, the restated loop gives cv2's mask and model on most
    scenes.  cv2's iteration count is not observable, but it is pinned through the model: a different stopping point would draw
    different subsets and refine a different inlier set.  cv2 4.13 returns the inliers of the refined model, not of the best
    hypothesis; `test_returned_mask_is_that_of_the_refined_model` checks that on its own.  The scenes that differ do so because the 4-point model comes from
    numpy's eigh here and from cv::eigen (its own Jacobi) in OpenCV; their last bits differ, which moves points whose float32
    error sits at the threshold, and from then on the two loops run on different counts."""
    cv2 = pytest.importorskip("cv2")
    same, differ = 0, []
    for s, n, frac in scene_set():
        src, dst = _f32(synthetic.planar_scene(400 + s, n, frac))
        Hc, mc = cv2.findHomography(src, dst, cv2.RANSAC, 3.0, confidence=0.99999)
        Ho, mo = hr.find_homography(src, dst, hr.RANSAC, 3.0, 0.99999, stream="opencv")
        if np.array_equal(mo, mc.ravel() > 0) and _corner_diff(Hc, Ho) < 1e-4:
            same += 1
        else:
            differ.append((s, n, frac, int(mo.sum()), int(mc.sum())))
    assert same >= 0.8 * 30, differ


def test_returned_mask_is_that_of_the_refined_model():
    cv2 = pytest.importorskip("cv2")
    for s, n, frac in scene_set()[:10]:
        src, dst = _f32(synthetic.planar_scene(400 + s, n, frac))
        Hc, mc = cv2.findHomography(src, dst, cv2.RANSAC, 3.0, confidence=0.99999)
        assert np.array_equal(hr.inlier_mask(Hc, src, dst, 3.0), mc.ravel() > 0)
    src, dst = _f32(synthetic.planar_scene(3, 300, 0.3))
    for thr in (3.0, 50.0):                                # method 0 too, at ransacReprojThreshold
        Hc, mc = cv2.findHomography(src, dst, 0, thr)
        assert np.array_equal(hr.inlier_mask(Hc, src, dst, thr), mc.ravel() > 0)
        Ho, mo = hr.find_homography(src, dst, 0, thr)       # least squares through 30 % outliers: 10 LM steps do not converge
        assert np.array_equal(mo, mc.ravel() > 0)


# Tolerances set from these 30 scenes (N = 500-2 000, 20-70 % outliers, 3 px threshold, confidence 0.99999, N(0, 0.5 px) noise).
# The Philox estimator and OpenCV draw different samples; measured between them: per-scene relative inlier-count difference
# median 0.0 % (largest 3.3 %), total count within 0.2 %, corner-error AUC@3/5/10 identical to 1e-3.
COUNT_MEDIAN_RTOL = 0.01
COUNT_TOTAL_RTOL = 0.01
AUC_TOL = 0.01


def check_statistics(counts, counts_cv2, errs, errs_cv2):
    counts, counts_cv2 = np.asarray(counts, float), np.asarray(counts_cv2, float)
    assert np.median(np.abs(counts - counts_cv2) / counts_cv2) <= COUNT_MEDIAN_RTOL
    assert abs(counts.sum() / counts_cv2.sum() - 1) <= COUNT_TOTAL_RTOL
    auc, auc_cv2 = synthetic.homography_auc(errs), synthetic.homography_auc(errs_cv2)
    assert np.abs(np.array(auc) - np.array(auc_cv2)).max() <= AUC_TOL, (auc, auc_cv2)


def test_philox_estimator_statistically_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    n_o, n_c, e_o, e_c = [], [], [], []
    for s, n, frac in scene_set():
        sc = synthetic.planar_scene(500 + s, n, frac)
        src, dst = _f32(sc)
        Ho, mo = hr.find_homography(src, dst, hr.RANSAC, 3.0, 0.99999, seed=s)
        Hc, mc = cv2.findHomography(src, dst, cv2.RANSAC, 3.0, confidence=0.99999)
        n_o.append(int(mo.sum()))
        n_c.append(int(mc.sum()))
        e_o.append(synthetic.homography_corner_error(Ho, sc["H"], 640, 480))
        e_c.append(synthetic.homography_corner_error(Hc, sc["H"], 640, 480))
    check_statistics(n_o, n_c, e_o, e_c)


def test_edge_cases_match_cv2():
    cv2 = pytest.importorskip("cv2")
    src, dst = _f32(synthetic.planar_scene(7, 60, 0.0))
    for k in (0, 3):
        with pytest.raises(cv2.error):
            cv2.findHomography(src[:k], dst[:k], cv2.RANSAC, 3.0)
        with pytest.raises(ValueError):
            hr.find_homography(src[:k], dst[:k], hr.RANSAC)
    for k in (4, 5):                                       # N == 4: the 4 points solved directly; N == 5: every point an inlier
        Hc, mc = cv2.findHomography(src[:k], dst[:k], cv2.RANSAC, 3.0)
        Ho, mo = hr.find_homography(src[:k], dst[:k], hr.RANSAC, stream="opencv")
        assert np.array_equal(mo, mc.ravel() > 0) and mo.all()
        assert _corner_diff(Hc, Ho) < 1e-4
    line = np.c_[np.arange(50.0), 2 * np.arange(50.0)].astype(np.float32)
    same = np.repeat(src[:1], 50, axis=0)
    for a, b in ((line, line + 1), (same, same)):
        Hc, mc = cv2.findHomography(a, b, cv2.RANSAC, 3.0)
        Ho, mo = hr.find_homography(a, b, hr.RANSAC)
        assert Hc is None and Ho is None and not mc.any() and not mo.any()
    srcn = src.copy()
    srcn[::7] = np.nan
    Hc, mc = cv2.findHomography(srcn, dst, cv2.RANSAC, 3.0)
    Ho, mo = hr.find_homography(srcn, dst, hr.RANSAC, stream="opencv")
    assert not mc[::7].any() and not mo[::7].any() and np.isfinite(Ho).all()
    assert np.array_equal(mo, mc.ravel() > 0) and _corner_diff(Hc, Ho) < 1e-4
    Ho, mo = hr.find_homography(srcn, dst, hr.RANSAC)
    assert not mo[::7].any() and np.isfinite(Ho).all()
    Hc, mc = cv2.findHomography(src[:, None], dst[:, None], cv2.RANSAC, 3.0)
    Ho, mo = hr.find_homography(src[:, None], dst[:, None], hr.RANSAC, stream="opencv")
    assert mc.shape == (60, 1) and np.array_equal(mo, mc.ravel() > 0) and _corner_diff(Hc, Ho) < 1e-4


def test_arguments_mirror_cv2():
    """What cv2 4.13 does with each argument, and `find_homography`'s host-side handling of it."""
    cv2 = pytest.importorskip("cv2")
    from roma_b200 import geometry
    src, dst = _f32(synthetic.planar_scene(8, 200, 0.2))
    ref, _ = cv2.findHomography(src, dst, cv2.RANSAC, 3.0)
    for thr in (0.0, -1.0):                                # a threshold <= 0 is OpenCV's default, 3
        assert np.array_equal(cv2.findHomography(src, dst, cv2.RANSAC, thr)[0], ref)
        assert geometry._homog_args(8, thr, 0.995, 2000)[1] == 3.0
    for conf in (0.0, 1.0, 1.5):
        with pytest.raises(cv2.error):
            cv2.findHomography(src, dst, cv2.RANSAC, 3.0, confidence=conf)
        with pytest.raises(ValueError):
            geometry._homog_args(8, 3.0, conf, 2000)
    assert geometry._homog_args(0, 3.0, 0.0, 2000)[0] == 0     # method 0 ignores the confidence
    for it in (0, -5):                                          # maxIters < 1 runs one iteration
        assert np.array_equal(cv2.findHomography(src, dst, cv2.RANSAC, 3.0, maxIters=it)[0],
                              cv2.findHomography(src, dst, cv2.RANSAC, 3.0, maxIters=1)[0])
        assert geometry._homog_args(8, 3.0, 0.995, it)[3] == 1
    for m in (cv2.LMEDS, cv2.RHO, cv2.USAC_DEFAULT, cv2.USAC_MAGSAC, cv2.USAC_ACCURATE):
        cv2.findHomography(src, dst, m)                         # cv2 implements them ...
        with pytest.raises(NotImplementedError):               # ... this package does not
            geometry._homog_args(m, 3.0, 0.995, 2000)
    with pytest.raises(cv2.error):
        cv2.findHomography(src, dst, 5)
    with pytest.raises(ValueError):
        geometry._homog_args(5, 3.0, 0.995, 2000)


def test_no_gpu_raises(monkeypatch):
    torch = pytest.importorskip("torch")
    from roma_b200 import geometry
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    src, dst = _f32(synthetic.planar_scene(0, 20, 0.0))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        geometry.find_homography(src, dst, geometry.RANSAC)
    with pytest.raises(ValueError):
        geometry.find_homography(src[:3], dst[:3], geometry.RANSAC)
    with pytest.raises(NotImplementedError):
        geometry.find_homography(src, dst, 4)
