"""`roma_b200.find_homography` on the device against the restatement (oracle/homography_ransac.py), stage by stage and end to end,
and against OpenCV."""
import numpy as np
import pytest
import torch

from oracle import homography_ransac as hr
from roma_b200 import geometry, synthetic

pytestmark = pytest.mark.gpu


def _f32(sc):
    return sc["src"].astype(np.float32), sc["dst"].astype(np.float32)


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def _run(src, dst, max_iters=2000, seed=0, conf=0.99999, thr=3.0, method=hr.RANSAC):
    dev = torch.device("cuda")
    s = torch.tensor(src, device=dev)
    d = torch.tensor(dst, device=dev)
    n = s.shape[0]
    offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
    buf = geometry._homog_launch(s, d, offsets, n, method, thr, conf, max_iters, seed)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in buf.items()}


def _splits(n):
    return max(1, min(32, (n + 511) // 512))


@pytest.mark.parametrize("seed,frac", [(0, 0.3), (1, 0.6)])
def test_stages_match_oracle(seed, frac):
    src, dst = _f32(synthetic.planar_scene(seed, 3000, frac))
    n = len(src)
    buf = _run(src, dst, seed=seed)
    H = 2000
    for h in range(0, H, 5):
        idx, att, found = hr.draw_subset(h, 0, n, seed, src, dst)
        assert found and list(buf["sample"][0, h]) == idx and buf["attempts"][0, h] == att, h
        Ho = hr.solve_four(src[idx], dst[idx])
        assert buf["status"][0, h] == (1 if Ho is not None else 0)
        if Ho is not None:
            assert _rel(buf["H"][0, h], Ho.ravel()) < 1e-9, h
    # the device's counts of its own H are the oracle's counts of those H, bit for bit
    sp = _splits(n)
    for h in range(0, H, 13):
        if buf["status"][0, h] == 1:
            assert int(buf["counts"][0, :sp, h].sum()) == int(hr.inlier_mask(buf["H"][0, h], src, dst, 3.0).sum())
    # the warp-parallel select equals the serial replay of the device's counts

    def hyp(h):
        s = int(buf["status"][0, h])
        return s, (int(buf["counts"][0, :sp, h].sum()) if s == 1 else 0)

    best_h, best, niters, it, nf = hr.select(hyp, n, 0.99999, 2000)
    st = buf["state"][0]
    assert (st[0], st[1], st[2], st[3], st[6]) == (it, niters, best, best_h, int(nf))
    assert np.array_equal(buf["best_H"][0], buf["H"][0, best_h])


@pytest.mark.parametrize("seed", [0, 3])
def test_refine_matches_oracle_and_cv2(seed):
    sc = synthetic.planar_scene(10 + seed, 5000, 0.4)
    src, dst = _f32(sc)
    buf = _run(src, dst, seed=seed)
    Hb = buf["best_H"][0].reshape(3, 3)
    m = hr.inlier_mask(Hb, src, dst, 3.0)
    Ho = hr.refine(Hb, src[m], dst[m])
    Hd = buf["out_H"][0].reshape(3, 3)
    assert _rel(Hd, Ho) < 1e-9
    assert np.array_equal(buf["mask"][:len(src)] > 0, hr.inlier_mask(Hd, src, dst, 3.0))
    cv2 = pytest.importorskip("cv2")
    Hc, _ = cv2.findHomography(src[m], dst[m], 0)
    assert np.abs(hr.corners(Hc, 640, 480) - hr.corners(Hd, 640, 480)).max() < 1e-4


@pytest.mark.parametrize("seed,n,frac", [(0, 2000, 0.2), (1, 5000, 0.5), (2, 1000, 0.7)])
def test_end_to_end_matches_oracle(seed, n, frac):
    src, dst = _f32(synthetic.planar_scene(20 + seed, n, frac))
    d = {}
    Ho, mo = hr.find_homography(src, dst, hr.RANSAC, 3.0, 0.99999, seed=seed, details=d)
    buf = _run(src, dst, seed=seed)
    assert (buf["state"][0, 3], buf["state"][0, 2], buf["state"][0, 1], buf["state"][0, 0]) == (d["hyp"], d["best"], d["niters"], d["iters"])
    Hd, md = geometry.find_homography(src, dst, geometry.RANSAC, 3.0, confidence=0.99999, seed=seed)
    assert _rel(Hd, Ho) < 1e-9
    assert np.array_equal(md.ravel() > 0, mo)


def test_statistically_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    import test_homography_host as th
    n_d, n_c, e_d, e_c = [], [], [], []
    for s, n, frac in th.scene_set():
        sc = synthetic.planar_scene(500 + s, n, frac)
        src, dst = _f32(sc)
        Hd, md = geometry.find_homography(src, dst, geometry.RANSAC, 3.0, confidence=0.99999, seed=s)
        Hc, mc = cv2.findHomography(src, dst, cv2.RANSAC, 3.0, confidence=0.99999)
        n_d.append(int(md.sum()))
        n_c.append(int(mc.sum()))
        e_d.append(synthetic.homography_corner_error(Hd, sc["H"], 640, 480))
        e_c.append(synthetic.homography_corner_error(Hc, sc["H"], 640, 480))
    th.check_statistics(n_d, n_c, e_d, e_c)


def test_batched_equals_per_pair_and_deterministic():
    sizes = [(2000, 0.2), (5000, 0.5), (4, 0.0), (777, 0.3), (3, 0.0), (10000, 0.6)]
    scenes = [_f32(synthetic.planar_scene(30 + i, n, f)) for i, (n, f) in enumerate(sizes)]
    srcs, dsts = [s for s, _ in scenes], [d for _, d in scenes]
    H, ok, masks = geometry.find_homography_batched(srcs, dsts, geometry.RANSAC, 3.0, confidence=0.99999, seed=5)
    H2, ok2, masks2 = geometry.find_homography_batched(srcs, dsts, geometry.RANSAC, 3.0, confidence=0.99999, seed=5)
    assert np.array_equal(H, H2) and np.array_equal(ok, ok2) and all(np.array_equal(a, b) for a, b in zip(masks, masks2))
    assert list(ok) == [True, True, True, True, False, True]
    assert not masks[4].any() and masks[4].shape == (3, 1) and masks[2].all()
    h0, m0 = geometry.find_homography(srcs[0], dsts[0], geometry.RANSAC, 3.0, confidence=0.99999, seed=5)
    assert np.array_equal(h0, H[0]) and np.array_equal(m0, masks[0])
    for b in (0, 1, 3, 5):                                 # each pair against the oracle with its own stream index
        Ho, mo = hr.find_homography(srcs[b], dsts[b], hr.RANSAC, 3.0, 0.99999, seed=5, b=b)
        assert _rel(H[b], Ho) < 1e-9 and np.array_equal(masks[b].ravel() > 0, mo)
    H4 = hr.solve_four(srcs[2], dsts[2])
    assert np.array_equal(H[2], H4)


def test_cuda_graph_replay_equals_eager():
    src, dst = _f32(synthetic.planar_scene(60, 5000, 0.5))
    dev = torch.device("cuda")
    s = torch.tensor(src, device=dev)
    d = torch.tensor(dst, device=dev)
    offsets = torch.tensor([0, len(src)], dtype=torch.int64, device=dev)
    args = (s, d, offsets, len(src), hr.RANSAC, 3.0, 0.995, 2000, 3)
    eager = geometry._homog_launch(*args)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        geometry._homog_launch(*args)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = geometry._homog_launch(*args)
    g.replay()
    torch.cuda.synchronize()
    for k in ("out_H", "ok", "mask", "state", "best_H"):
        assert torch.equal(out[k], eager[k]), k


def test_more_rounds_than_one():
    src, dst = _f32(synthetic.planar_scene(70, 2000, 0.85))
    d = {}
    Ho, mo = hr.find_homography(src, dst, hr.RANSAC, 3.0, 0.99999, max_iters=5000, seed=1, details=d)
    buf = _run(src, dst, max_iters=5000, seed=1)
    st = buf["state"][0]
    assert (st[3], st[2], st[1], st[0]) == (d["hyp"], d["best"], d["niters"], d["iters"])
    assert d["iters"] > geometry.HOMOG_ROUND
    assert _rel(buf["out_H"][0], Ho.ravel()) < 1e-9


def test_forms_method0_and_large_n():
    cv2 = pytest.importorskip("cv2")
    sc = synthetic.planar_scene(80, 3000, 0.3)
    src, dst = sc["src"], sc["dst"]                        # float64 in: rounded to float32 first, as cv2 does
    H, m = geometry.find_homography(src, dst, geometry.RANSAC, 3.0, seed=2)
    assert isinstance(H, np.ndarray) and H.dtype == np.float64 and H.shape == (3, 3) and abs(H[2, 2] - 1) < 1e-15
    assert m.dtype == np.uint8 and m.shape == (3000, 1)
    H2, m2 = geometry.find_homography(src.astype(np.float32)[:, None], dst.astype(np.float32)[:, None], geometry.RANSAC, 3.0, seed=2)
    assert np.array_equal(H, H2) and np.array_equal(m, m2)
    Ht, mt = geometry.find_homography(torch.tensor(src, device="cuda"), torch.tensor(dst, device="cuda"), geometry.RANSAC, 3.0, seed=2)
    assert Ht.is_cuda and Ht.dtype == torch.float64 and mt.dtype == torch.uint8 and tuple(mt.shape) == (3000, 1)
    assert np.array_equal(Ht.cpu().numpy(), H) and np.array_equal(mt.cpu().numpy(), m)
    # method 0 on the inliers: least squares over all points, against the oracle and cv2
    s32, d32 = src.astype(np.float32)[sc["inlier"]], dst.astype(np.float32)[sc["inlier"]]
    H0, m0 = geometry.find_homography(s32, d32)
    Ho, mo = hr.find_homography(s32, d32, 0)
    Hc, mc = cv2.findHomography(s32, d32, 0)
    assert _rel(H0, Ho) < 1e-9 and np.array_equal(m0.ravel() > 0, mo) and np.array_equal(m0, mc)
    assert np.abs(hr.corners(Hc, 640, 480) - hr.corners(H0, 640, 480)).max() < 1e-4
    import roma_b200
    assert roma_b200.find_homography is geometry.find_homography and roma_b200.RANSAC == 8
    # 100 000 points: buffers linear in N
    big = synthetic.planar_scene(81, 100_000, 0.5)
    Hb, mb = geometry.find_homography(big["src"], big["dst"], geometry.RANSAC, 3.0, confidence=0.99999)
    assert Hb is not None and mb.shape == (100_000, 1)
    assert synthetic.homography_corner_error(Hb, big["H"], 640, 480) < 0.5
    assert abs(int(mb.sum()) - int(big["inlier"].sum())) < 0.02 * big["inlier"].sum()


def test_edge_cases():
    src, dst = _f32(synthetic.planar_scene(90, 60, 0.0))
    with pytest.raises(ValueError):
        geometry.find_homography(src[:3], dst[:3], geometry.RANSAC)
    H4, m4 = geometry.find_homography(src[:4], dst[:4], geometry.RANSAC)
    assert m4.all() and _rel(H4, hr.solve_four(src[:4], dst[:4])) == 0.0
    H5, m5 = geometry.find_homography(src[:5], dst[:5], geometry.RANSAC)
    Ho5, mo5 = hr.find_homography(src[:5], dst[:5], hr.RANSAC)
    assert _rel(H5, Ho5) < 1e-9 and np.array_equal(m5.ravel() > 0, mo5)
    line = np.c_[np.arange(50.0), 2 * np.arange(50.0)].astype(np.float32)
    same = np.repeat(src[:1], 50, axis=0)
    for a, b in ((line, line + 1), (same, same)):
        H, m = geometry.find_homography(a, b, geometry.RANSAC)
        assert H is None and m.shape == (50, 1) and not m.any()
    srcn = src.copy()
    srcn[::7] = np.nan
    H, m = geometry.find_homography(srcn, dst, geometry.RANSAC)
    assert H is not None and np.isfinite(H).all() and not m[::7].any()
