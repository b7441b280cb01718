"""`roma_b200.estimate_pose` on the device against the numpy restatement (oracle/pose_ransac.py), stage by stage and end to end,
and against OpenCV."""
import numpy as np
import pytest
import torch

from oracle import pose_ransac as pr
from roma_b200 import geometry, synthetic

pytestmark = pytest.mark.gpu


def _scene(seed, n=5000, frac=0.3):
    sc = synthetic.two_view_scene(seed, n, frac)
    sc["thr"] = 0.5 / (sc["K0"][0, 0] + sc["K1"][0, 0])
    return sc


def _run(sc, max_iters=1000, seed=0):
    dev = torch.device("cuda")
    x0 = torch.tensor(sc["kpts0"], device=dev)
    x1 = torch.tensor(sc["kpts1"], device=dev)
    n = x0.shape[0]
    offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
    K = torch.tensor(np.stack([sc["K0"], sc["K1"]])[None], device=dev)
    buf = geometry._launch(x0, x1, offsets, K, n, sc["thr"], 0.99999, max_iters, seed)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in buf.items()}


def _xn(sc):
    return np.concatenate([pr.normalise(sc["kpts0"], sc["K0"]), pr.normalise(sc["kpts1"], sc["K1"])], axis=1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_stages_match_oracle(seed):
    sc = _scene(seed)
    buf = _run(sc, seed=seed)
    xn = _xn(sc)
    n = xn.shape[0]
    assert np.array_equal(buf["xn"], xn)
    H = 1000
    for h in range(H):
        assert list(buf["sample"][0, h]) == pr.draw_sample(h, 0, n, seed)
    # solutions within 1e-9 (relative to the unit norm) of the oracle's.  A sample whose degree-10 polynomial has a near-double
    # root gets its roots from the Sturm bisection on the device and from eigenvalues (np.roots) in the oracle, which may then
    # disagree beyond 1e-9 or on whether the pair is real; that happens for a few percent of samples.
    sols = pr.solve_five_point(xn[buf["sample"][0, :H]])
    match = 0
    for h in range(H):
        d = buf["E"][0, h, :buf["nsol"][0, h]]
        o = sols[h]
        if len(d) == len(o) and (len(d) == 0 or np.abs(d - o).max() < 1e-9):
            match += 1
    assert match >= 0.95 * H, match
    # the device's counts of its own E are the oracle's counts of those E, bit for bit
    st = buf["state"][0]
    for h in range(0, H, 7):
        for s in range(buf["nsol"][0, h]):
            want = int(pr.inlier_mask(buf["E"][0, h, s], xn, sc["thr"]).sum())
            got = int(buf["counts"][0, :, s, h][:max(1, min(16, (n + 1023) // 1024))].sum())
            assert got == want
    # selection replay over the device's counts
    splits = max(1, min(16, (n + 1023) // 1024))

    def counts_of(h):
        return [int(buf["counts"][0, :splits, s, h].sum()) for s in range(buf["nsol"][0, h])]

    hyp, sol, best, niters, it = pr.select(counts_of, n, 0.99999, 1000)
    assert (st[3], st[4], st[2], st[1], st[0]) == (hyp, sol, best, niters, it)
    assert np.array_equal(buf["best_E"][0, 0], buf["E"][0, hyp, sol])


@pytest.mark.parametrize("seed", [0, 3])
def test_recover_matches_cv2(seed):
    cv2 = pytest.importorskip("cv2")
    sc = _scene(seed)
    buf = _run(sc, seed=seed)
    xn = _xn(sc)
    E = buf["best_E"][0, 0].reshape(3, 3)
    m8 = pr.inlier_mask(E.ravel(), xn, sc["thr"])[0].astype(np.uint8)[:, None].copy()
    n_cv, R_cv, t_cv, m_cv = cv2.recoverPose(E, xn[:, :2].copy(), xn[:, 2:].copy(), np.eye(3), 1e9, mask=m8)
    assert buf["ok"][0] == 1
    assert np.abs(buf["R"][0] - R_cv).max() < 1e-9 and np.abs(buf["t"][0] - t_cv.ravel()).max() < 1e-9
    assert np.array_equal(buf["mask"][:len(xn)] > 0, m_cv.ravel() > 0)


@pytest.mark.parametrize("seed,frac", [(0, 0.2), (1, 0.5), (2, 0.3)])
def test_end_to_end_matches_oracle(seed, frac):
    sc = _scene(10 + seed, frac=frac)
    d = {}
    ro = pr.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], sc["thr"], seed=seed, details=d)
    buf = _run(sc, seed=seed)
    assert (buf["state"][0, 3], buf["state"][0, 4]) == (d["hyp"], d["sol"])
    assert np.abs(buf["best_E"][0, 0] - d["E"]).max() < 1e-9
    R, t, mask = geometry.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], sc["thr"], seed=seed)
    # the two E agree to 1e-9; the decomposition amplifies that by up to ~10 (the recover stage alone is pinned to cv2 at 1e-9)
    assert np.abs(R - ro[0]).max() < 1e-8 and np.abs(t - ro[1]).max() < 1e-8
    assert np.array_equal(mask, ro[2])


def test_statistically_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    import test_pose_host as th
    errs_d, errs_c, n_d, n_c = [], [], [], []
    for seed, frac in th.scene_set():
        sc = synthetic.two_view_scene(1000 + seed, 5000, frac)
        thr = 0.5 / (sc["K0"][0, 0] + sc["K1"][0, 0])
        rd = geometry.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], thr, seed=seed)
        rc = th._reference_estimate_pose(cv2, sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], thr)
        errs_d.append(th.pose_error(rd[0], rd[1], sc["R"], sc["t"]))
        errs_c.append(th.pose_error(rc[0], rc[1], sc["R"], sc["t"]))
        n_d.append(int(rd[2].sum()))
        n_c.append(int(rc[2].sum()))
    th.check_statistics(n_d, n_c, errs_d, errs_c)


def test_batched_equals_per_pair_and_deterministic():
    scenes = [_scene(20 + i, n=n, frac=f) for i, (n, f) in enumerate([(2000, 0.2), (5000, 0.5), (777, 0.3), (10000, 0.4)])]
    thr = 0.5 / 2400
    K0 = np.stack([s["K0"] for s in scenes])
    K1 = np.stack([s["K1"] for s in scenes])
    R, t, ok, masks = geometry.estimate_pose_batched([s["kpts0"] for s in scenes], [s["kpts1"] for s in scenes], K0, K1, thr, seed=5)
    R2, t2, ok2, masks2 = geometry.estimate_pose_batched([s["kpts0"] for s in scenes], [s["kpts1"] for s in scenes], K0, K1, thr, seed=5)
    assert np.array_equal(R, R2) and np.array_equal(t, t2) and all(np.array_equal(a, b) for a, b in zip(masks, masks2))
    assert ok.all()
    # pair 0 alone draws the same stream (b = 0)
    r0 = geometry.estimate_pose(scenes[0]["kpts0"], scenes[0]["kpts1"], K0[0], K1[0], thr, seed=5)
    assert np.array_equal(r0[0], R[0]) and np.array_equal(r0[1], t[0]) and np.array_equal(r0[2], masks[0])
    # every pair against the oracle run with its own stream index
    for b, s in enumerate(scenes):
        ro = pr.estimate_pose(s["kpts0"], s["kpts1"], K0[b], K1[b], thr, seed=5, b=b)
        assert np.abs(R[b] - ro[0]).max() < 1e-9 and np.array_equal(masks[b], ro[2])


def test_numpy_and_tensor_forms():
    sc = _scene(30, n=3000)
    r = geometry.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], sc["thr"])
    R, t, mask = r
    assert isinstance(R, np.ndarray) and R.dtype == np.float64 and R.shape == (3, 3)
    assert t.dtype == np.float64 and t.shape == (3, 1)
    assert mask.dtype == bool and mask.shape == (3000,)
    k0 = torch.tensor(sc["kpts0"], dtype=torch.float32, device="cuda")
    k1 = torch.tensor(sc["kpts1"], dtype=torch.float32, device="cuda")
    Rt, tt, mt = geometry.estimate_pose(k0, k1, sc["K0"], sc["K1"], sc["thr"])
    assert Rt.is_cuda and Rt.dtype == torch.float64 and tt.shape == (3, 1) and mt.dtype == torch.bool and mt.shape == (3000,)
    import roma_b200
    assert roma_b200.estimate_pose is geometry.estimate_pose


def test_edge_cases():
    sc = _scene(40, n=50, frac=0.0)
    k0, k1, K0, K1 = sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"]
    assert geometry.estimate_pose(k0[:4], k1[:4], K0, K1, 1e-3) is None
    r5 = geometry.estimate_pose(k0[:5], k1[:5], K0, K1, 1e-3)
    o5 = pr.estimate_pose(k0[:5], k1[:5], K0, K1, 1e-3)
    assert (r5 is None) == (o5 is None)
    if r5 is not None:                  # a minimal sample: its solutions are only as well conditioned as the five points
        assert np.abs(r5[0] - o5[0]).max() < 1e-6 and np.array_equal(r5[2], o5[2])
    same = np.repeat(k0[:1], 50, axis=0)
    assert geometry.estimate_pose(same, same, K0, K1, 1e-3) is None
    k0n = k0.copy()
    k0n[::7] = np.nan
    r = geometry.estimate_pose(k0n, k1, K0, K1, 1e-3)
    assert r is not None and not r[2][::7].any()
    # a pair of fewer than 5 points inside a batch
    R, t, ok, masks = geometry.estimate_pose_batched([k0[:3], k0], [k1[:3], k1], K0, K1, 1e-3)
    assert not ok[0] and ok[1] and not masks[0].any()


def test_more_rounds_than_one():
    sc = _scene(50, n=2000, frac=0.75)
    d = {}
    ro = pr.estimate_pose(sc["kpts0"], sc["kpts1"], sc["K0"], sc["K1"], sc["thr"], max_iters=3000, seed=1, details=d)
    buf = _run(sc, max_iters=3000, seed=1)
    assert (buf["state"][0, 3], buf["state"][0, 4], buf["state"][0, 1]) == (d["hyp"], d["sol"], d["niters"])
    assert (ro is not None) == bool(buf["ok"][0])


def test_cuda_graph_replay_equals_eager():
    sc = _scene(60)
    dev = torch.device("cuda")
    x0 = torch.tensor(sc["kpts0"], device=dev)
    x1 = torch.tensor(sc["kpts1"], device=dev)
    n = x0.shape[0]
    offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
    K = torch.tensor(np.stack([sc["K0"], sc["K1"]])[None], device=dev)
    eager = geometry._launch(x0, x1, offsets, K, n, sc["thr"], 0.99999, 1000, 3)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        geometry._launch(x0, x1, offsets, K, n, sc["thr"], 0.99999, 1000, 3)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = geometry._launch(x0, x1, offsets, K, n, sc["thr"], 0.99999, 1000, 3)
    g.replay()
    torch.cuda.synchronize()
    for k in ("R", "t", "ok", "mask", "state", "best_E"):
        assert torch.equal(out[k], eager[k]), k
