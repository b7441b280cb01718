"""`roma_b200.find_fundamental` on the device against the restatement (oracle/fundamental_ransac.py), stage by stage and end to
end, and against cv2's USAC_MAGSAC over seeded scenes."""
import cv2
import numpy as np
import pytest
import torch

from oracle import fundamental_ransac as fr
from roma_b200 import geometry, synthetic

pytestmark = pytest.mark.gpu

TABLES = geometry.magsac_tables()
THR, CONF = 0.2, 0.999999          # the reference's usage example (README.md:62-78)


def _run(x0, x1, max_iters=1024, seed=0, thr=THR, conf=CONF):
    dev = torch.device("cuda")
    a = torch.tensor(x0, dtype=torch.float64, device=dev)
    b = torch.tensor(x1, dtype=torch.float64, device=dev)
    offsets = torch.tensor([0, len(x0)], dtype=torch.int64, device=dev)
    buf = geometry._fund_launch(a, b, offsets, len(x0), thr, conf, max_iters, seed)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in buf.items()}


def _scene(seed, n, frac, noise=0.5):
    sc = synthetic.two_view_scene(seed, n, frac, noise)
    return sc["kpts0"], sc["kpts1"], sc


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


@pytest.mark.parametrize("seed,frac,n", [(0, 0.3, 2000), (1, 0.5, 1500)])
def test_stages_match_oracle(seed, frac, n):
    x0, x1, _ = _scene(seed, n, frac)
    buf = _run(x0, x1, seed=seed)
    nr, xn = fr.normalise(x0, x1)
    assert np.array_equal(buf["norm"][0], nr) and np.array_equal(buf["xn"][:n], xn)
    sample, nmod, F = fr.hypotheses(xn, nr, n, seed, 0, 1024)
    assert np.array_equal(buf["sample"][0], sample)                      # drawn indices identical
    assert np.array_equal(buf["nmod"][0], nmod)
    assert nmod.sum() > 0
    for h in range(1024):
        for m in range(nmod[h]):
            assert _rel(buf["F"][0, h, m], F[h, m]) < 1e-9, (h, m)       # seven-point models
    # the device's losses and counts of its own models are the oracle's fixed-order sums, bit for bit
    L, C = fr.score(buf["F"][0].reshape(-1, 9), x0, x1, THR, TABLES)
    S = L.shape[0]
    live = (np.arange(3)[None, :] < buf["nmod"][0][:, None]).ravel()
    assert np.array_equal(buf["losses"][0, :S][:, live], L[:, live])
    assert np.array_equal(buf["counts"][0, :S][:, live], C[:, live])

    # the warp-parallel select equals the serial replay of the device's losses
    def models(h):
        return [(fr.model_loss(buf["losses"][0, :S, h * 3 + m]), int(buf["counts"][0, :S, h * 3 + m].sum())) for m in range(buf["nmod"][0, h])]

    hyp, slot, best, niters, it = fr.select(models, n, CONF, 1024)
    st = buf["state"][0]
    assert (st[0], st[1], st[2], st[3], st[5]) == (it, niters, hyp, slot, n)
    assert buf["best_loss"][0] == best and np.array_equal(buf["best_F"][0], buf["F"][0, hyp, slot])
    # refinement from the device's best model
    Fo = fr.refine(buf["best_F"][0], x0, x1, xn, nr, THR, TABLES)
    assert buf["ok"][0] == 1 and _rel(buf["out_F"][0], Fo) < 1e-9
    assert np.array_equal(buf["mask"][:n].astype(bool), fr.sampson2(Fo, x0, x1) < THR * THR)


@pytest.mark.parametrize("seed,frac,n,max_iters", [(2, 0.3, 2000, 1000), (3, 0.7, 2000, 10000)])
def test_end_to_end_matches_oracle(seed, frac, n, max_iters):
    x0, x1, _ = _scene(seed, n, frac)
    F, mask = geometry.find_fundamental(x0, x1, geometry.USAC_MAGSAC, THR, CONF, max_iters, seed=seed)
    d = {}
    Fo, mo = fr.find_fundamental(x0, x1, THR, CONF, max_iters, TABLES, seed=seed, details=d)
    if max_iters > 1024:
        assert d["iters"] > 1024                                           # more than one round
    assert _rel(F, Fo) < 1e-9
    assert np.array_equal(mask[:, 0].astype(bool), mo)


def test_batched_equals_single():
    sizes = [(7, 0.0), (2000, 0.3), (513, 0.5), (5000, 0.6), (8, 0.0)]
    scenes = [_scene(10 + i, n, f, 0.5 if n > 8 else 0.0) for i, (n, f) in enumerate(sizes)]
    Fb, ok, masks = geometry.find_fundamental_batched([s[0] for s in scenes], [s[1] for s in scenes], geometry.USAC_MAGSAC, THR, CONF,
                                                      3000, seed=5)
    assert ok.all()
    for b, (x0, x1, _) in enumerate(scenes):
        F, mask = geometry.find_fundamental(x0, x1, geometry.USAC_MAGSAC, THR, CONF, 3000, seed=5)
        assert np.array_equal(Fb[b], F) and np.array_equal(masks[b], mask), b
    assert masks[0].all() and masks[4].all()                               # N = 7, 8 on clean points: every point an inlier


def test_deterministic_and_graph_replay():
    x0, x1, _ = _scene(4, 3000, 0.4)
    a, b = _run(x0, x1, seed=3), _run(x0, x1, seed=3)
    for k in ("out_F", "mask", "ok", "losses", "F"):
        assert np.array_equal(a[k], b[k]), k
    dev = torch.device("cuda")
    t0 = torch.tensor(x0, device=dev)
    t1 = torch.tensor(x1, device=dev)
    offsets = torch.tensor([0, len(x0)], dtype=torch.int64, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        geometry._fund_launch(t0, t1, offsets, len(x0), THR, CONF, 1024, 3)  # warm: the tables are uploaded outside the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        buf = geometry._fund_launch(t0, t1, offsets, len(x0), THR, CONF, 1024, 3)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(buf["out_F"].cpu().numpy(), a["out_F"]) and np.array_equal(buf["mask"].cpu().numpy(), a["mask"])


def test_return_forms_and_rules():
    x0, x1, _ = _scene(6, 1000, 0.3)
    F, mask = geometry.find_fundamental(x0, x1, geometry.USAC_MAGSAC, THR, CONF, 1000)
    assert isinstance(F, np.ndarray) and F.shape == (3, 3) and F.dtype == np.float64
    assert mask.shape == (1000, 1) and mask.dtype == np.uint8
    # float32 and [N, 1, 2] inputs
    F32, m32 = geometry.find_fundamental(x0.astype(np.float32).reshape(-1, 1, 2), x1.astype(np.float32).reshape(-1, 1, 2),
                                         geometry.USAC_MAGSAC, THR, CONF, 1000)
    assert F32.dtype == np.float64 and m32.shape == (1000, 1)
    # tensors in, device tensors out
    Ft, mt = geometry.find_fundamental(torch.tensor(x0, device="cuda"), torch.tensor(x1, device="cuda"), geometry.USAC_MAGSAC, THR, CONF,
                                       1000)
    assert Ft.is_cuda and mt.is_cuda and np.array_equal(Ft.cpu().numpy(), F) and np.array_equal(mt.cpu().numpy(), mask)
    # NaN rows are never inliers and leave the rest alone
    y0 = x0.copy()
    y0[::50] = np.nan
    Fn, mn = geometry.find_fundamental(y0, x1, geometry.USAC_MAGSAC, THR, CONF, 1000)
    assert Fn is not None and not mn[::50].any() and mn.sum() > 0.5 * mask.sum()
    # degenerate inputs: no model
    same = np.tile([[100.0, 200.0]], (50, 1))
    assert geometry.find_fundamental(same, same + 1.0)[0] is None
    t = np.linspace(0, 1, 50)[:, None]
    line0, line1 = np.c_[100 + 500 * t, 200 + 300 * t], np.c_[50 + 400 * t, 300 - 100 * t]
    Fl, ml = geometry.find_fundamental(line0, line1)
    assert Fl is None and not ml.any()


def test_large_pair():
    x0, x1, sc = _scene(7, 100000, 0.5, 0.1)
    F, mask = geometry.find_fundamental(x0, x1, geometry.USAC_MAGSAC, THR, CONF, 10000)
    assert np.array_equal(mask[:, 0].astype(bool), fr.sampson2(F.ravel(), x0, x1) < THR * THR)
    assert mask.sum() > 0.4 * 100000


def _pose_error(F, sc):
    E = sc["K1"].T @ F @ sc["K0"]
    p0 = cv2.undistortPoints(sc["kpts0"].reshape(-1, 1, 2), sc["K0"], None).reshape(-1, 2)
    p1 = cv2.undistortPoints(sc["kpts1"].reshape(-1, 1, 2), sc["K1"], None).reshape(-1, 2)
    _n, R, t, _m = cv2.recoverPose(E, p0, p1)
    ang = lambda c: float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))
    return max(ang((np.trace(R.T @ sc["R"]) - 1) / 2), ang(abs(float(t.ravel() @ sc["t"])) / np.linalg.norm(t)))


@pytest.mark.parametrize("noise,frac,n", [
    (0.1, 0.2, 2000), (0.1, 0.5, 10000), (0.5, 0.5, 10000),
    # measured on an H100: median pose error 0.22 deg against cv2's 0.10 deg (seed-to-seed standard deviation 0.05 deg); outside
    # cv2's spread, and kept as a known gap rather than hidden by a wider tolerance
    pytest.param(0.5, 0.2, 2000, marks=pytest.mark.xfail(strict=True, reason="pose error outside cv2's spread at 0.5 px, 20 % outliers"))])
def test_statistics_against_cv2(noise, frac, n):
    """Over 8 seeded scenes per setting, against cv2 4.13 USAC_MAGSAC with the README's arguments: pose error of E = K1^T F K0 by
    cv2.recoverPose, recall of the planted inliers, and median Sampson distance of the planted inliers.  The device draws its own
    samples, so only the distributions can agree; each tolerance is the spread of cv2's own statistic over the same seeds."""
    ours, theirs = {"err": [], "rec": [], "med": []}, {"err": [], "rec": [], "med": []}
    for seed in range(8):
        x0, x1, sc = _scene(100 + seed, n, frac, noise)
        inl = ~sc["outlier"]
        for F, mask, out in ((*geometry.find_fundamental(x0, x1, geometry.USAC_MAGSAC, THR, CONF, 10000), ours),
                             (*cv2.findFundamentalMat(x0, x1, cv2.USAC_MAGSAC, THR, CONF, 10000), theirs)):
            out["err"].append(_pose_error(F, sc))
            out["rec"].append(float(mask[inl, 0].astype(bool).mean()))
            out["med"].append(float(np.median(np.sqrt(fr.sampson2((F / np.linalg.norm(F)).ravel(), x0[inl], x1[inl])))))
    print({k: (np.median(ours[k]), np.median(theirs[k]), np.std(theirs[k])) for k in ours})
    # pose error: ours is at most cv2's median plus two of cv2's seed-to-seed standard deviations
    assert np.median(ours["err"]) <= np.median(theirs["err"]) + 2 * np.std(theirs["err"]) + 1e-3
    # recall of the planted inliers and their median Sampson distance: within two of cv2's standard deviations (and 2 %)
    assert abs(np.median(ours["rec"]) - np.median(theirs["rec"])) <= 2 * np.std(theirs["rec"]) + 0.02
    assert np.median(ours["med"]) <= np.median(theirs["med"]) + 2 * np.std(theirs["med"]) + 1e-3

