"""Host checks of the fundamental-matrix estimator: the MAGSAC++ tables against the paper's definition, the restated solvers
(oracle/fundamental_ransac.py) against cv2's, cv2's own behaviour that `find_fundamental` copies, and argument handling."""
import math
import os

import cv2
import numpy as np
import pytest
from scipy import integrate, special, stats

from oracle import fundamental_ransac as fr
from roma_b200 import geometry, synthetic

TABLES = geometry.magsac_tables()
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _unit(F):
    F = np.asarray(F, dtype=np.float64).ravel()
    return F / np.linalg.norm(F)


def _close_up_to_sign(a, b):
    a, b = _unit(a), _unit(b)
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def test_constants():
    assert geometry.MAGSAC_K2 == pytest.approx(stats.chi2.ppf(0.99, 4), rel=1e-14) and fr.K2 == geometry.MAGSAC_K2
    header = open(os.path.join(ROOT, "include", "romab200.h")).read()
    assert f"#define RB_FUND_K2 {geometry.MAGSAC_K2!r}" in header
    for name, value in (("USAC_MAGSAC", 38), ("FM_7POINT", 1), ("FM_8POINT", 2), ("FM_LMEDS", 4), ("FM_RANSAC", 8), ("USAC_DEFAULT", 32),
                        ("USAC_PARALLEL", 33), ("USAC_FM_8PTS", 34), ("USAC_FAST", 35), ("USAC_ACCURATE", 36), ("USAC_PROSAC", 37)):
        assert getattr(cv2, name) == value
        assert value == geometry.USAC_MAGSAC or geometry._FUND_UNSUPPORTED[value] == name


def test_loss_and_weight_match_the_paper():
    """The paper's definition with nu = 4: g(r | sigma) = 2 C sigma^-4 exp(-r^2 / 2 sigma^2) r^3 for r < k sigma, C = 1 / (4 Gamma(2)),
    sigma uniform on [0, sigma_max]; the weight is w(r) = int g(r | sigma) / sigma_max dsigma and the loss rho(r) = int_0^r x w(x) dx.
    The tables hold rho / rho(k sigma_max) and w / w(0); the device interpolates them linearly over 1024 intervals of r^2."""
    smax, k = 0.7, math.sqrt(geometry.MAGSAC_K2)

    def w(r):
        if r >= k * smax:
            return 0.0
        f = lambda s: 2 * 0.25 * s ** -4 * math.exp(-r * r / (2 * s * s)) * r ** 3 / smax
        return integrate.quad(f, r / k, smax, epsabs=0, epsrel=1e-12, limit=200)[0]

    def rho(r):
        return integrate.quad(lambda x: x * w(x), 0, r, epsabs=0, epsrel=1e-10, limit=200)[0]

    rmax = rho(k * smax)
    # w(0) = C 2^(3/2) (Gamma(3/2) - Gamma(3/2, k^2 / 2)) / sigma_max
    w0 = 0.25 * 2 ** 1.5 * (1.0 - special.gammaincc(1.5, k * k / 2)) * special.gamma(1.5) / smax
    for r in (0.01, 0.1, 0.35, 0.7, 1.3, 2.0, 2.5):
        q = np.array([r * r])
        loss = float(fr.table_at(TABLES[0], q, smax)[0])
        weight = float(fr.table_at(TABLES[1], q, smax)[0])
        assert loss == pytest.approx(rho(r) / rmax, abs=2e-6), r           # linear interpolation error of the table
        assert weight == pytest.approx(w(r) / w0, abs=1e-4), r              # w has a q^(3/2) term at 0: the coarsest cell
    assert float(fr.point_losses(np.array([(k * smax) ** 2]), smax, TABLES)[0]) == 1.0
    # the table's nodes are the closed form exactly (to rounding)
    i = np.arange(0, 1025, 64)
    x = geometry.MAGSAC_K2 / 2 * i / 1024
    G = lambda a, z: special.gammaincc(a, z) * special.gamma(a)
    g = lambda a, z: special.gammainc(a, z) * special.gamma(a)
    xk = geometry.MAGSAC_K2 / 2
    ref = (g(2.5, x) + x * (G(1.5, x) - G(1.5, xk))) / g(2.5, xk)
    assert np.abs(TABLES[0, i] - ref).max() < 1e-13
    assert np.abs(TABLES[1, i] - (G(1.5, x) - G(1.5, xk)) / (G(1.5, 0) - G(1.5, xk))).max() < 1e-13


def test_seven_point_matches_cv2():
    """As sets of solutions up to scale.  cv2's FM_7POINT solves the un-normalised pixel system, whose algebraic residuals on the 7
    points are about 1e-13 against about 1e-18 here; that limits the agreement to 3e-5 (measured over these seeds)."""
    for seed in range(6):
        sc = synthetic.two_view_scene(seed, 7, 0.0, 0.0)
        nr, xn = fr.normalise(sc["kpts0"], sc["kpts1"])
        nm, Fn = fr.seven_point(xn[None], orient=False)
        mine = [fr.denormalise(Fn[0, m], nr)[0] for m in range(nm[0])]
        Fc, _ = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.FM_7POINT)
        theirs = list(Fc.reshape(-1, 3, 3))
        assert len(mine) == len(theirs)
        for F in mine:
            assert min(_close_up_to_sign(F, c) for c in theirs) < 1e-4, seed
        x0, x1 = np.c_[sc["kpts0"], np.ones(7)], np.c_[sc["kpts1"], np.ones(7)]
        res = lambda F: np.abs(np.einsum("ij,jk,ik->i", x1, _unit(F).reshape(3, 3), x0)).max()
        assert max(res(F) for F in mine) <= max(res(F) for F in theirs)
        # the oriented constraint keeps a subset, in the same order
        nmo, Fo = fr.seven_point(xn[None])
        kept = [m for m in range(nm[0]) if fr.oriented(Fn[0, m][None], xn[None])[0]]
        assert nmo[0] == len(kept) and all(np.array_equal(Fo[0, j], Fn[0, m]) for j, m in enumerate(kept))


def test_unit_weight_eight_point_matches_cv2():
    for seed in range(6):
        sc = synthetic.two_view_scene(seed, 200, 0.0, 0.5)
        nr, xn = fr.normalise(sc["kpts0"], sc["kpts1"])
        F, ok = fr.weighted_eight_point(xn, np.ones(200), nr)
        Fc, _ = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.FM_8POINT)
        assert ok and _close_up_to_sign(F, Fc) < 1e-7, seed             # measured: at most 1.1e-8


def test_cv2_behaviour_that_find_fundamental_copies():
    # the mask of USAC_MAGSAC is the Sampson rule, on cv2's own output (measured agreement 99.97-100 %)
    for seed in range(4):
        sc = synthetic.two_view_scene(seed, 3000, 0.3, 0.5)
        Fc, mc = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.USAC_MAGSAC, 0.2, 0.999999, 10000)
        rule = fr.sampson2(Fc.ravel(), sc["kpts0"], sc["kpts1"]) < 0.04
        assert (rule == mc[:, 0].astype(bool)).mean() >= 0.999
        F2, m2 = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.USAC_MAGSAC, 0.2, 0.999999, 10000)
        assert np.array_equal(Fc, F2) and np.array_equal(mc, m2)            # deterministic across calls
        assert abs(np.linalg.det(_unit(Fc).reshape(3, 3))) < 1e-12          # rank 2, no fixed scale
    # N = 7, 8, 9 clean points: one 3x3 F and an all-ones mask; fewer than 7: an error
    for n in (7, 8, 9):
        sc = synthetic.two_view_scene(1, n, 0.0, 0.0)
        Fc, mc = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.USAC_MAGSAC, 0.2, 0.999999, 10000)
        assert Fc.shape == (3, 3) and mc.shape == (n, 1) and mc.all()
        F, m = fr.find_fundamental(sc["kpts0"], sc["kpts1"], 0.2, 0.999999, 10000, TABLES)
        assert F.shape == (3, 3) and m.all()
    sc = synthetic.two_view_scene(1, 6, 0.0, 0.0)
    with pytest.raises(cv2.error):
        cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.USAC_MAGSAC, 0.2, 0.999999, 10000)


def test_argument_handling():
    sc = synthetic.two_view_scene(0, 50, 0.0)
    x0, x1 = sc["kpts0"], sc["kpts1"]
    for method, name in geometry._FUND_UNSUPPORTED.items():
        with pytest.raises(NotImplementedError, match=name):
            geometry.find_fundamental(x0, x1, method)
    with pytest.raises(ValueError):
        geometry.find_fundamental(x0, x1, 99)
    with pytest.raises(ValueError):                                         # fewer than 7 points: before any device work
        geometry.find_fundamental(x0[:6], x1[:6])
    with pytest.raises(ValueError):
        geometry.find_fundamental(x0, x1[:-1])
    for kw in ({"ransacReprojThreshold": 0}, {"ransacReprojThreshold": float("nan")}, {"confidence": 1.0}, {"maxIters": 0}):
        with pytest.raises(ValueError):
            geometry.find_fundamental(x0, x1, **kw)
    with pytest.raises(ValueError):
        geometry._fund_points(np.zeros((5, 3)), None)
    assert geometry._fund_points(np.zeros((5, 1, 2), np.float32), "cpu").shape == (5, 2)


def test_rules_for_nan_and_degenerate_rows():
    sc = synthetic.two_view_scene(3, 1000, 0.3, 0.1)
    x0 = sc["kpts0"].copy()
    x0[::40] = np.nan
    F, m = fr.find_fundamental(x0, sc["kpts1"], 0.2, 0.999999, 1000, TABLES)
    assert F is not None and not m[::40].any() and m.sum() > 500
    nr, _xn = fr.normalise(x0, sc["kpts1"])
    assert np.isfinite(nr).all()
    same = np.tile([[100.0, 200.0]], (50, 1))
    F, m = fr.find_fundamental(same, same + 1.0, 3.0, 0.99, 1000, TABLES)
    assert F is None and not m.any()
    t = np.linspace(0, 1, 50)[:, None]
    F, m = fr.find_fundamental(np.c_[100 + 500 * t, 200 + 300 * t], np.c_[50 + 400 * t, 300 - 100 * t], 3.0, 0.99, 1000, TABLES)
    assert F is None and not m.any()


def test_oracle_against_cv2_easy_scenes():
    """noise 0.1 px, 30 % outliers, N = 5000, seeds 0-3 at the README's arguments: cv2's max(rotation, translation) error over
    seeds 0-9 was 0.018-0.13 degrees.  The restatement stays inside that range and finds as many inliers as cv2 (within 2 %).  The
    harder settings (0.5 px, up to 50 % outliers, N up to 10 000) take thousands of hypotheses each and run on the device in
    tests/test_fundamental_gpu.py::test_statistics_against_cv2."""
    for seed in range(4):
        sc = synthetic.two_view_scene(seed, 5000, 0.3, 0.1)
        F, m = fr.find_fundamental(sc["kpts0"], sc["kpts1"], 0.2, 0.999999, 10000, TABLES)
        Fc, mc = cv2.findFundamentalMat(sc["kpts0"], sc["kpts1"], cv2.USAC_MAGSAC, 0.2, 0.999999, 10000)
        E = sc["K1"].T @ F @ sc["K0"]
        p0 = cv2.undistortPoints(sc["kpts0"].reshape(-1, 1, 2), sc["K0"], None).reshape(-1, 2)
        p1 = cv2.undistortPoints(sc["kpts1"].reshape(-1, 1, 2), sc["K1"], None).reshape(-1, 2)
        _n, R, t, _m = cv2.recoverPose(E, p0, p1)
        eR = np.degrees(np.arccos(np.clip((np.trace(R.T @ sc["R"]) - 1) / 2, -1, 1)))
        et = np.degrees(np.arccos(np.clip(abs(t.ravel() @ sc["t"]) / np.linalg.norm(t), -1, 1)))
        assert max(eR, et) < 0.13, seed
        assert abs(int(m.sum()) - int(mc.sum())) <= 0.02 * mc.sum(), seed
