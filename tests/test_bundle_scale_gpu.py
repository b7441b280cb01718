"""`bundle_adjust` at the sizes the benchmark runs, stage by stage: the blocked Cholesky (`romab200_ba_cholesky`) called directly on
synthetic systems of order n = 6F up to 2400 (several trsm CTAs, more than one pass of the substitutions' 1024-strided loops, long
panel sequences, failing pivots) against Higham's backward-error bounds; the reduced camera system S, its right-hand side, factor
and step captured from real runs at N = 30, 60 and 200 against `oracle/bundle.py`'s fp64 systems with summation-error bars; gauges
with several fixed_tx cameras, gaps in the free cameras and a fixed_tx camera that is also fixed; and more tracks than one launch
of the track kernels covers."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.bundle import bundle_adjust as oracle_ba  # noqa: E402
from roma_b200 import MatchGraph, Points3D, Tracks, build_tracks, bundle_adjust, cabi, consolidate_matches, synthetic  # noqa: E402
from roma_b200 import triangulate_tracks, verify_matches  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}
U = 2.0 ** -53                    # unit roundoff of float64
# S and b of the device against the oracle: |dS| <= TAU S_abs, where S_abs sums the absolute value of every term.  The worst ratio
# measured on an H100 was 143 u (290 529 tracks over 4 cameras, so about 2e5 terms per entry); 71 u at N = 30 with the Cauchy loss.
# Dropping one observation moves S by more than 1e13 u S_abs.
TAU = 256 * U


def gamma(n):
    return n * U / (1 - n * U)


def _scene(seed, N, points, cs=1, outlier_frac=0.0, size=(384, 512), rot_deg=0.3, centre=0.05, drop_conflicts=True):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cs, outlier_frac=outlier_frac,
                                                                      device=DEV)
    g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    if outlier_frac > 0:
        g = verify_matches(pairs, g, threshold=THR[cs])[0]
    tr = build_tracks(pairs, g, drop_conflicts=drop_conflicts)
    R1, t1 = synthetic.perturb_cameras(seed, R, t, rot_deg, centre)
    pts = triangulate_tracks(g, tr, K, R1, t1, max_error=20.0)
    return g, tr, pts, K, R1, t1, R, t, X


def _oracle(g, tr, pts, K, R, t, **kw):
    return oracle_ba(g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.X, pts.ok, pts.inlier, K, R, t, **kw)


# ---- checks of a factor and a solve -----------------------------------------------------------------------------------------
def _full(S):
    """The symmetric matrix whose lower triangle is S's."""
    L = np.tril(S)
    return L + np.tril(L, -1).T


def _factor_ratios(S, L, b, x):
    """Worst ratios of the backward errors of L = chol(S) and of x = S^-1 b to Higham's bounds (S symmetric, L lower):
    |S - L L^T| <= gamma_{n+1} |L| |L^T| and |S x - b| <= gamma_n |L| |L^T| |x|, element by element (where a bound is 0 the error
    must be 0 too: an infinite ratio), and of |x - numpy.linalg.solve(S, b)|_inf / |x|_inf to n u cond(S)."""
    n = S.shape[0]
    aL = np.abs(L)
    LLt = aL @ aL.T
    with np.errstate(divide="ignore", invalid="ignore"):
        e1 = np.abs(S - L @ L.T)
        r1 = np.where(e1 == 0, 0.0, e1 / (gamma(n + 1) * LLt))
        e2 = np.abs(S @ x - b)
        r2 = np.where(e2 == 0, 0.0, e2 / (gamma(n) * (LLt @ np.abs(x))))
    ref = np.linalg.solve(S, b)
    ev = np.abs(np.linalg.eigvalsh(S))
    r3 = np.abs(x - ref).max() / np.abs(ref).max() / (n * U * ev.max() / ev.min())
    return np.tril(r1).max(), r2.max(), r3


def _check_factor(S, L, b, x, what):
    """Higham's bounds with c = 3 for the factor and c = 5 for the solve: the checking products in float64 add up to gamma_n
    |L| |L^T| (|x|) of their own."""
    r1, r2, r3 = _factor_ratios(S, L, b, x)
    print(f"{what}: backward error {r1:.3f} of gamma_(n+1) |L||L^T|, residual {r2:.3f} of gamma_n |L||L^T||x|, "
          f"x vs numpy {r3:.2e} of n u cond(S)")
    assert r1 <= 3 and r2 <= 5 and r3 <= 10, (what, r1, r2, r3)


# ---- the Cholesky stage, called directly ------------------------------------------------------------------------------------
def _cholesky(S, b):
    """romab200_ba_cholesky on float64 S [n, n] and b [n] (n = 6F) with a one-track, one-element geometry of F images: returns the
    factored S, the solution and result[3] (the pivot flag; result is zeroed first)."""
    n = S.shape[0]
    F = n // 6
    i64, i32 = torch.int64, torch.int32
    z = lambda k, dt=torch.float64: torch.zeros(k, dtype=dt, device=DEV)  # noqa: E731
    S_d, b_d, result = torch.from_numpy(S.copy()).to(DEV).reshape(-1), torch.from_numpy(b.copy()).to(DEV), z(cabi.RB_BA_RESULT)
    cabi.call("romab200_ba_cholesky", "rb_ba_args", num_tracks=1, num_images=F, num_free=F, num_elements=1, num_rows=1,
              loss_scale2=0.0, track_offsets=torch.tensor([0, 1], dtype=i64, device=DEV), elements=z(2, i32), kp_offsets=z(F + 1, i64),
              keypoints=z(2, torch.float32), track_ok=z(1, torch.uint8), inlier=z(1, torch.uint8), info=z(2, i64),
              cams=z(F * cabi.RB_BA_CAM), X=z(3), S=S_d, rhs=b_d, result=result, **{"lambda": 1.0})
    torch.cuda.synchronize()
    return S_d.view(n, n).cpu().numpy(), b_d.cpu().numpy(), float(result[3])


def _spd(n, cond, seed):
    """Q diag(sigma) Q^T with sigma log-spaced from 1 to 1 / cond, its strict upper triangle NaN; and b."""
    rng = np.random.default_rng(seed)
    Q = np.linalg.qr(rng.normal(size=(n, n)))[0]
    S = (Q * np.logspace(0, -np.log10(cond), n)) @ Q.T
    S = _full(S)
    S[np.triu_indices(n, 1)] = np.nan
    return S, rng.normal(size=n)


# one panel, a partial last panel, a second trsm CTA (n > NB + 128), a second pass of both substitution loops (n > NB + 1024)
CHOL_F = [1, 5, 6, 11, 26, 27, 60, 170, 171, 176, 177, 200, pytest.param(400, marks=pytest.mark.slow)]


@pytest.mark.parametrize("F", CHOL_F)
@pytest.mark.parametrize("cond", [1e2, 1e10])
def test_cholesky_backward_error(F, cond):
    n = 6 * F
    S, b = _spd(n, cond, F)
    L_out, x, pivot = _cholesky(S, b)
    assert pivot == 0
    up = np.triu_indices(n, 1)
    # the factor reads and writes only the lower triangle: ba_cameras_kernel leaves the upper one undefined
    assert L_out[up].tobytes() == S[up].tobytes()
    _check_factor(_full(S), np.tril(L_out), b, x, f"n={n} cond={cond:.0e}")
    L2, x2, _ = _cholesky(S, b)
    assert L2.tobytes() == L_out.tobytes() and x2.tobytes() == x.tobytes()


@pytest.mark.parametrize("F", [27, 200])
def test_cholesky_flags_a_failing_pivot(F):
    """S = L0 D L0^T with D = I but one -1 at p: a pivot that fails in the first panel, a middle one and the last partial one."""
    n = 6 * F
    rng = np.random.default_rng(F)
    L0 = np.eye(n) + np.tril(rng.normal(size=(n, n)), -1) / np.sqrt(n)
    b = rng.normal(size=n)
    _, _, pivot = _cholesky(L0 @ L0.T, b)
    assert pivot == 0
    assert (n - 2) // cabi.RB_BA_NB == (n - 1) // cabi.RB_BA_NB and n % cabi.RB_BA_NB != 0
    for p in (3, 40, n - 2):
        D = np.ones(n)
        D[p] = -1.0
        S = (L0 * D) @ L0.T
        S[np.triu_indices(n, 1)] = np.nan
        assert _cholesky(S, b)[2] == 1.0, p


@pytest.mark.parametrize("value", [np.nan, np.inf])
def test_cholesky_flags_a_value_that_is_not_finite(value):
    n = 6 * 30
    S0, b = _spd(n, 1e2, 0)
    for i, j in ((0, 0), (n - 1, 0), (40, 3), (n - 1, n - 1), (100, 99)):
        S = S0.copy()
        S[i, j] = value
        assert _cholesky(S, b)[2] == 1.0, (i, j)


# ---- the reduced camera system inside real runs -----------------------------------------------------------------------------
def _captured(monkeypatch, *args, **kw):
    """bundle_adjust with S and rhs copied after every romab200_ba_cameras and romab200_ba_cholesky call: the result and, per trial
    with free cameras, (S, b, factor, step) as float64 arrays, S [n, n] with only the lower triangle defined."""
    caps = []
    orig = cabi.call

    def spy(fn, struct, **a):
        orig(fn, struct, **a)
        if fn in ("romab200_ba_cameras", "romab200_ba_cholesky"):
            n = 6 * a["num_free"]
            if fn == "romab200_ba_cameras":
                caps.append([])
            caps[-1] += [a["S"].view(n, n).cpu().numpy().copy(), a["rhs"].cpu().numpy().copy()]

    monkeypatch.setattr(cabi, "call", spy)
    try:
        res = bundle_adjust(*args, **kw)
    finally:
        monkeypatch.setattr(cabi, "call", orig)
    return res, caps


def _system_ratio(S_dev, b_dev, sy):
    """Worst |S - S_oracle| / S_abs over the lower triangle and |b - b_oracle| / b_abs (an entry whose bar is 0 must be equal)."""
    lo = np.tril_indices(S_dev.shape[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        dS, dB = np.abs(S_dev[lo] - sy["S"][lo]), np.abs(b_dev - sy["b"])
        rS = np.where(dS == 0, 0.0, dS / sy["S_abs"][lo]).max()
        rB = np.where(dB == 0, 0.0, dB / sy["b_abs"]).max()
    return rS, rB


def _compare(res, caps, ref, systems, what, final_cost=True):
    """The whole-run rules of test_bundle_gpu.test_device_matches_the_oracle, then every trial's captured system: S and b against
    the oracle's while both runs are still at the same linearization point (up to and including the first kept trial), and the
    device's factor and step against the backward-error bounds of its own S."""
    tri = ref["trials"]
    assert abs(res.cost[0] - ref["cost"][0]) <= 1e-10 * ref["cost"][0]
    assert abs(res.pred[0] - tri[0]["pred"]) <= 1e-10 * abs(tri[0]["pred"])
    assert abs(res.cost[1] - ref["cost"][1]) <= 1e-10 * ref["cost"][1]
    n = min(res.accepted.size, ref["accepted"].size)
    for k in range(n):
        if abs(tri[k]["margin"]) <= 1e-6 + 1e-10 * tri[k]["F"] / abs(tri[k]["pred"]):
            break
        assert res.accepted[k] == ref["accepted"][k], k
    if final_cost:
        assert abs(res.cost[-1] - ref["cost"][-1]) <= 1e-8 * ref["cost"][-1]
    assert all(len(c) == 4 for c in caps)
    for k, (S, b, Lf, x) in enumerate(caps):
        if k < len(systems) and not ref["accepted"][:k].any():
            rS, rB = _system_ratio(S, b, systems[k])
            print(f"{what} trial {k}: |S - S_oracle| {rS / U:.2f} u S_abs, |b - b_oracle| {rB / U:.2f} u b_abs (bar {TAU / U:.0f} u)")
            assert rS <= TAU and rB <= TAU, (k, rS / U, rB / U)
        _check_factor(_full(S), np.tril(Lf), b, x, f"{what} trial {k}")


def _free_inlier(g, tr, pts, fixed_poses):
    """An inlier element of an ok track in a free camera."""
    off = tr.track_offsets.cpu().numpy()
    used = np.repeat(pts.ok.cpu().numpy(), np.diff(off)) & pts.inlier.cpu().numpy()
    img = tr.elements[:, 0].cpu().numpy()
    return int(np.flatnonzero(used & ~np.isin(img, fixed_poses))[0])


def _bar_bites(g, tr, pts, K, R, t, systems, kw):
    """The bar of S is tight enough to see one observation: without one inlier flag the oracle's S moves by more than TAU S_abs."""
    e = _free_inlier(g, tr, pts, kw.get("fixed_poses", (0,)))
    inl = pts.inlier.clone()
    inl[e] = False
    sys1 = []
    _oracle(g, tr, Points3D(pts.X, pts.ok, pts.num_inliers, pts.error, inl), K, R, t, **{**kw, "max_iterations": 1}, systems=sys1)
    rS, _ = _system_ratio(sys1[0]["S"], sys1[0]["b"], systems[0])
    print(f"one observation fewer moves S by {rS / U:.3g} u S_abs")
    assert rS > 1e3 * TAU


@pytest.mark.parametrize("seed, N, points, gauge, max_iterations", [
    (20, 30, 600, {}, 100),
    (21, 60, 600, dict(fixed_poses=(3, 4, 31), fixed_tx=(0, 5, 59)), 4),
    pytest.param(22, 200, 1000, {}, 3, marks=pytest.mark.slow)])
def test_system_factor_and_step_match_the_oracle(monkeypatch, seed, N, points, gauge, max_iterations):
    g, tr, pts, K, R, t, *_ = _scene(seed, N, points)
    kw = dict(max_iterations=max_iterations, function_tolerance=1e-12, **gauge)
    res, caps = _captured(monkeypatch, g, tr, pts, K, R, t, **kw)
    systems = []
    ref = _oracle(g, tr, pts, K, R, t, **kw, systems=systems)
    print(f"N={N}: {len(tr)} tracks, {int(pts.inlier.sum())} inliers, n = {6 * (N - len(gauge.get('fixed_poses', (0,))))}; "
          f"F {res.cost[0]:.6g} -> {res.cost[-1]:.10g} in {res.accepted.size} trials; oracle {ref['cost'][-1]:.10g}")
    assert len(caps) == res.accepted.size
    _compare(res, caps, ref, systems, f"N={N}", final_cost=max_iterations == 100)
    if N < 200:                                   # one more oracle trial at N = 200 costs half a minute; N = 30 and 60 show the reach
        _bar_bites(g, tr, pts, K, R, t, systems, kw)


# ---- gauges -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("loss_scale", [None, 1.0])
def test_gauge_with_several_fixed_tx_and_gaps(monkeypatch, loss_scale):
    fixed_poses, fixed_tx = (0, 7, 19), (1, 7, 12, 29)               # camera 7 is in both
    g, tr, pts, K, R, t, *_ = _scene(23, 30, 600)
    kw = dict(fixed_poses=fixed_poses, fixed_tx=fixed_tx, loss_scale=loss_scale, max_iterations=10, function_tolerance=1e-12)
    res, caps = _captured(monkeypatch, g, tr, pts, K, R, t, **kw)
    systems = []
    ref = _oracle(g, tr, pts, K, R, t, **kw, systems=systems)
    assert res.accepted.any() and len(caps) == res.accepted.size
    _compare(res, caps, ref, systems, f"gauge loss={loss_scale}")
    free = [i for i in range(30) if i not in fixed_poses]
    tx = [6 * fi + 3 for fi, i in enumerate(free) if i in fixed_tx]
    assert len(tx) == 3
    for S, b, _, x in caps:
        for j in tx:
            assert (S[j, :j] == 0).all() and S[j, j] == 1.0 and (S[j + 1:, j] == 0).all() and b[j] == 0.0 and x[j] == 0.0
    R0, t0 = R.double(), t.double()
    for i in fixed_poses:
        assert torch.equal(res.R[i], R0[i]) and torch.equal(res.t[i], t0[i])
    for i in fixed_tx:
        assert res.t[i, 0] == t0[i, 0]
    moved = [i for i in free if i not in fixed_tx]
    assert all(not torch.equal(res.t[i], t0[i]) for i in moved)


# ---- more tracks than one launch covers ---------------------------------------------------------------------------------------
def _many_tracks(seed, points, visibility=0.7, noise=0.5, size=(768, 1024)):
    """4 cameras of `planted_cameras`'s geometry and `points` scene points in its box, each seen in 2-4 of them (visibility per
    camera, inside the image and in front), with `noise` px Gaussian noise; one track per point seen twice or more, every element an
    inlier, X the planted point moved by up to 0.01 units.  The graph has no matches (bundle_adjust reads keypoints only)."""
    _, _, _, _, _, K, R, t, _ = synthetic.planted_cameras(seed, 4, 10, size=size)
    K, R, t = K.numpy(), R.numpy(), t.numpy()
    H, W = size
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.0, 1.0, (points, 3)) * np.array([4.0, 3.0, 3.0])
    p = np.einsum("cij,cjk,pk->cpi", K, R, X) + np.einsum("cij,cj->ci", K, t)[:, None]
    xy = p[..., :2] / p[..., 2:3] + rng.normal(scale=noise, size=(4, points, 2))
    vis = (p[..., 2] > 0) & (xy[..., 0] >= 0) & (xy[..., 0] < W) & (xy[..., 1] >= 0) & (xy[..., 1] < H)
    vis &= rng.random(vis.shape) < visibility
    keep = vis.sum(0) >= 2
    vis, xy, X = vis[:, keep], xy[:, keep], X[keep]
    T = X.shape[0]
    kp_off = np.concatenate(([0], np.cumsum(vis.sum(1))))
    ids = np.cumsum(vis, 1) - 1                                              # keypoint id of point k in image i
    keypoints = np.concatenate([xy[i][vis[i]] for i in range(4)]).astype(np.float32)
    trk, img = np.nonzero(vis.T)                                             # track-major, image ascending
    elements = np.stack((img, ids[img, trk]), 1).astype(np.int32)
    track_off = np.concatenate(([0], np.cumsum(vis.sum(0))))
    kp_track = np.full(kp_off[-1], -1, np.int32)
    kp_track[kp_off[img] + elements[:, 1]] = trk
    d = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(DEV)         # noqa: E731
    g = MatchGraph(d(kp_off), d(keypoints), d(np.ones(kp_off[-1], np.float32)), d(np.zeros(1, np.int64)), d(np.zeros((0, 2), np.int32)),
                   d(np.zeros(0, np.float32)))
    tr = Tracks(d(track_off), d(elements), d(kp_track), 0)
    Xs = X + rng.uniform(-0.01, 0.01, X.shape)
    pts = Points3D(d(Xs), d(np.ones(T, bool)), d(vis.sum(0).astype(np.int32)), d(np.zeros(T)), d(np.ones(img.size, bool)))
    R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
    return g, tr, pts, d(K), d(R1), d(t1)


@pytest.mark.slow
def test_more_tracks_than_one_launch_covers(monkeypatch):
    g, tr, pts, K, R, t = _many_tracks(24, 320_000)
    T = len(tr)
    L = np.diff(tr.track_offsets.cpu().numpy())
    print(f"{T} tracks of {L.min()}-{L.max()} views, {L.sum()} observations")
    assert T > 64 * 1024 * 4 and L.min() == 2 and L.max() == 4
    for gauge in (dict(fixed_poses=range(4)), {}):
        kw = dict(max_iterations=2, **gauge)
        res, caps = _captured(monkeypatch, g, tr, pts, K, R, t, **kw)
        systems = []
        ref = _oracle(g, tr, pts, K, R, t, **kw, systems=systems)
        print(f"gauge {gauge}: F {res.cost[0]:.10g} -> {res.cost[-1]:.10g}, accepted {res.accepted}; oracle {ref['cost'][-1]:.10g}")
        _compare(res, caps, ref, systems, f"{T} tracks", final_cost=False)
        assert len(caps) == (0 if gauge else 2)
        again = bundle_adjust(g, tr, pts, K, R, t, **kw)
        for x, y in ((res.R, again.R), (res.t, again.t), (res.points.X, again.points.X), (res.points.error, again.points.error)):
            assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
        assert np.array_equal(res.cost, again.cost) and np.array_equal(res.pred, again.pred)
