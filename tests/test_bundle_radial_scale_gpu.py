"""Self-calibrating `bundle_adjust` (camera_model="SIMPLE_RADIAL") at the sizes the benchmarks run, stage by stage: the per-image
camera system (8 rows per camera), the fold onto shared cameras (`romab200_ba_fold`: S' = P^T S P, b' = P^T b, order n' = 6F + 2G),
the factor and solve of the folded system (`romab200_ba_groups_cholesky`), and the unfold d = P d' (`romab200_ba_unfold`), captured
from real runs at N = 50 and 200 images:
- the fold against a `math.fsum` of the device's own S, with one camera of 200 images, 200 singleton cameras, and uneven groups
  that are not contiguous in image order (one of more than 128 members), fixed poses, fixed t_x, a fixed camera and unobserved
  images inside the groups, and the refine switches; and called directly on random systems whose pinned rows are not zero;
- the unfold and the trial cameras bit for bit, for every member of every group;
- the factor and solve of S' (n' = 1202 and 1600) and of the per-image 8F system (n = 1600) against Higham's backward-error bounds;
- S and b (per-image) and S' and b' (shared) against `oracle/bundle_radial.py` and `oracle/bundle_shared.py` with summation-error
  bars, and whole runs against the same oracles;
- at N = 200, reruns that are byte-identical and cameras past the first 128 that move."""
import functools
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import bundle_radial as orad  # noqa: E402
from oracle import bundle_shared as osh  # noqa: E402
from roma_b200 import MatchGraph, Points3D, Tracks, bundle_adjust, cabi, synthetic  # noqa: E402
from roma_b200 import bundle as rb_ba  # noqa: E402

DEV = "cuda"
U = 2.0 ** -53                    # unit roundoff of float64
# S and b of the device against the oracle: |dS| <= TAU S_abs, where S_abs sums the absolute value of every term (as in
# test_bundle_scale_gpu.py).
TAU = 256 * U


def gamma(n):
    return n * U / (1 - n * U)


# ---- scenes ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def _cameras(seed, N, size):
    """planted_cameras' SIMPLE_RADIAL geometry of N images (k in +-0.05), as float64 numpy arrays."""
    _, _, _, _, _, intr, R, t, _ = synthetic.planted_cameras(seed, N, 10, size=size, radial=(-0.05, 0.05))
    return intr.numpy(), R.numpy(), t.numpy()


def _scene(seed, ids, points, visibility, unobserved=(), noise=0.5, size=(768, 1024), ferr=0.03):
    """N = len(ids) SIMPLE_RADIAL cameras of planted_cameras' geometry, every image of a camera id taking the intrinsics of the id's
    first image, and `points` scene points in its box, each seen by every camera in front of it that has it inside the image, with
    probability `visibility`, plus `noise` px Gaussian noise.  One track per point seen twice or more, every element an inlier but
    those of the images in `unobserved`; X the planted point moved by up to 0.01 units; perturbed poses; a prior whose f is off by
    ferr (sign random) per camera id and k = 0.  The graph has no matches (bundle_adjust reads keypoints only).  Returns the graph,
    tracks, points, prior [N, 4] (numpy), R and t on the device."""
    ids = np.asarray(ids)
    N = ids.size
    intr, R, t = _cameras(seed, N, size)
    first = np.array([np.flatnonzero(ids == ids[i])[0] for i in range(N)])
    intr = intr[first]
    H, W = size
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.0, 1.0, (points, 3)) * np.array([4.0, 3.0, 3.0])
    p = np.einsum("cij,pj->cpi", R, X) + t[:, None]
    x, y = p[..., 0] / p[..., 2], p[..., 1] / p[..., 2]
    d = 1.0 + intr[:, 3:4] * (x * x + y * y)
    xy = np.stack((intr[:, 0:1] * d * x + intr[:, 1:2], intr[:, 0:1] * d * y + intr[:, 2:3]), -1)
    xy += rng.normal(scale=noise, size=xy.shape)
    vis = (p[..., 2] > 0) & (xy[..., 0] >= 0) & (xy[..., 0] < W) & (xy[..., 1] >= 0) & (xy[..., 1] < H)
    vis &= rng.random(vis.shape) < visibility
    keep = vis.sum(0) >= 2
    vis, xy, X = vis[:, keep], xy[:, keep], X[keep]
    T = X.shape[0]
    kp_off = np.concatenate(([0], np.cumsum(vis.sum(1))))
    kid = np.cumsum(vis, 1) - 1                                              # keypoint id of point k in image i
    keypoints = np.concatenate([xy[i][vis[i]] for i in range(N)]).astype(np.float32)
    trk, img = np.nonzero(vis.T)                                             # track-major, image ascending
    elements = np.stack((img, kid[img, trk]), 1).astype(np.int32)
    track_off = np.concatenate(([0], np.cumsum(vis.sum(0))))
    kp_track = np.full(kp_off[-1], -1, np.int32)
    kp_track[kp_off[img] + elements[:, 1]] = trk
    dv = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(DEV)        # noqa: E731
    g = MatchGraph(dv(kp_off), dv(keypoints), dv(np.ones(kp_off[-1], np.float32)), dv(np.zeros(1, np.int64)),
                   dv(np.zeros((0, 2), np.int32)), dv(np.zeros(0, np.float32)))
    tr = Tracks(dv(track_off), dv(elements), dv(kp_track), 0)
    Xs = X + rng.uniform(-0.01, 0.01, X.shape)
    inlier = ~np.isin(img, list(unobserved))
    pts = Points3D(dv(Xs), dv(np.ones(T, bool)), dv(vis.sum(0).astype(np.int32)), dv(np.zeros(T)), dv(inlier))
    R1, t1 = synthetic.perturb_cameras(seed, torch.from_numpy(R), torch.from_numpy(t), 0.3, 0.05)
    prior = intr.copy()
    C = ids.max() + 1
    prior[:, 0] *= (1 + rng.choice([-1.0, 1.0], C) * ferr)[ids]
    prior[:, 3] = 0.0
    return g, tr, pts, prior, R1.to(DEV), t1.to(DEV)


def _uneven_ids(seed, sizes=(1, 2, 30, 37, 130)):
    """Camera ids of sum(sizes) images, id j held by sizes[j] images interleaved in a random order."""
    return np.random.default_rng(seed).permutation(np.repeat(np.arange(len(sizes)), sizes))


# ---- capture ------------------------------------------------------------------------------------------------------------------
def _host(v, shape=None):
    a = v.cpu().numpy().copy()
    return a.reshape(shape) if shape is not None else a


def _captured(monkeypatch, *args, **kw):
    """bundle_adjust with its buffers copied to the host, per trial with free cameras: S and rhs after romab200_ba_cameras (S [8F,
    8F], only its lower triangle defined); after romab200_ba_cholesky the factor L and the step d; with camera_ids, S' and b' after
    romab200_ba_fold (Sg [n', n'], lower triangle), the factor Lg and step dg after romab200_ba_groups_cholesky, the group layout,
    and the per-camera step d after romab200_ba_unfold; then cams and cams_trial [N, 16] after romab200_ba_step."""
    caps = []
    orig = cabi.call

    def spy(fn, struct, **a):
        orig(fn, struct, **a)
        name = fn[len("romab200_ba_"):]
        if name == "cameras":
            n = 8 * a["num_free"]
            caps.append(dict(S=_host(a["S"], (n, n)), rhs=_host(a["rhs"])))
        elif name == "cholesky":
            n = 8 * a["num_free"]
            caps[-1].update(L=_host(a["S"], (n, n)), d=_host(a["rhs"]))
        elif name in ("fold", "groups_cholesky"):
            n = 6 * a["num_free"] + 2 * a["num_groups"]
            S, b = _host(a["S_groups"], (n, n)), _host(a["rhs_groups"])
            if name == "fold":
                caps[-1].update(Sg=S, bg=b, offsets=_host(a["group_offsets"]), members=_host(a["group_members"]),
                                group_pin=_host(a["group_pin"], (-1, 2)).astype(bool))
            else:
                caps[-1].update(Lg=S, dg=b)
        elif name == "unfold":
            caps[-1].update(d=_host(a["rhs"]))
        elif name == "step" and caps and "trial" not in caps[-1]:
            N = a["num_images"]
            caps[-1].update(cams=_host(a["cams"], (N, cabi.RB_BA_CAM1)), trial=_host(a["cams_trial"], (N, cabi.RB_BA_CAM1)))

    monkeypatch.setattr(cabi, "call", spy)
    try:
        res = bundle_adjust(*args, **kw)
    finally:
        monkeypatch.setattr(cabi, "call", orig)
    return res, caps


def _full(S):
    """The symmetric matrix whose lower triangle is S's."""
    L = np.tril(S)
    return L + np.tril(L, -1).T


# ---- checks of a factor and a solve (those of test_bundle_scale_gpu.py) ---------------------------------------------------------
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


# ---- the fold and the unfold against the device's own S ---------------------------------------------------------------------
def _fsum_ratio(dev, terms, chain):
    """Worst |dev - fsum(terms)| / (gamma_chain sum |terms|) over the columns of terms [k, m] (dev [m]); a zero bar needs equality."""
    ref = np.array([math.fsum(c) for c in terms.T])
    err = np.abs(dev - ref)
    bar = gamma(chain) * np.abs(terms).sum(0)
    assert ((err == 0) | (bar > 0)).all(), "an entry with a zero bar differs"
    return float(np.where(err == 0, 0.0, err / np.where(bar > 0, bar, 1.0)).max(initial=0.0))


def _check_fold(c):
    """S' and b' of romab200_ba_fold against P^T S P and P^T b from the lower triangle of the captured S: pose-pose entries and pose
    rows of b' bit for bit; group-pose entries and group rows of b' within gamma_(|g| - 1) of fsum, group-group entries within
    gamma_(ceil(|g| |h| / 256) + 8) (a strided slice per thread of 256, then an 8-level tree); pinned groups exactly e_r with b' = 0.
    Returns the worst ratios (group-pose, group-group, b')."""
    S, rhs, Sg, bg = _full(c["S"]), c["rhs"], c["Sg"], c["bg"]
    off, mem, gpin = c["offsets"], c["members"], c["group_pin"]
    F, G = S.shape[0] // 8, off.size - 1
    P6 = 6 * F
    assert Sg.shape == (P6 + 2 * G,) * 2 and off[0] == 0 and off[-1] == F and sorted(mem.tolist()) == list(range(F))
    pose = (8 * np.arange(F)[:, None] + np.arange(6)).reshape(-1)
    lo = np.tril_indices(P6)
    assert Sg[:P6, :P6][lo].tobytes() == S[np.ix_(pose, pose)][lo].tobytes()
    assert bg[:P6].tobytes() == rhs[pose].tobytes()
    worst = [0.0, 0.0, 0.0]
    for g in range(G):
        mg = mem[off[g]:off[g + 1]]
        for j in range(2):
            R = P6 + 2 * g + j
            if gpin[g, j]:
                assert (Sg[R, :R] == 0).all() and Sg[R, R] == 1.0 and (Sg[R + 1:, R] == 0).all() and bg[R] == 0.0, (g, j)
                continue
            rows = 8 * mg + 6 + j
            worst[0] = max(worst[0], _fsum_ratio(Sg[R, :P6], S[np.ix_(rows, pose)], mg.size - 1))
            worst[2] = max(worst[2], _fsum_ratio(bg[R:R + 1], rhs[rows][:, None], mg.size - 1))
            for h in range(g + 1):
                mh = mem[off[h]:off[h + 1]]
                for l in range(2):
                    C = P6 + 2 * h + l
                    if C > R or gpin[h, l]:
                        continue
                    terms = S[np.ix_(rows, 8 * mh + 6 + l)].reshape(-1, 1)
                    worst[1] = max(worst[1], _fsum_ratio(Sg[R, C:C + 1], terms, -(-mg.size * mh.size // 256) + 8))
    assert max(worst) <= 1.0, worst
    return worst


def _check_unfold_and_trial(c, pins, free):
    """The per-camera step after romab200_ba_unfold is P d' bit for bit, and the trial cameras of romab200_ba_step take it: t and
    (f, k) of every free camera are cams + d (cams where pinned), the rotation and everything of a camera that is not free are
    copies where pinned, and the trial intrinsics of every image of a camera id are equal bit for bit."""
    F = len(free)
    off, mem, dg, d = c["offsets"], c["members"], c["dg"], c["d"]
    want = np.empty(8 * F)
    grp = np.empty(F, np.int64)
    for g in range(off.size - 1):
        grp[mem[off[g]:off[g + 1]]] = g
    d8 = want.reshape(F, 8)
    d8[:, :6] = dg[:6 * F].reshape(F, 6)
    d8[:, 6] = dg[6 * F + 2 * grp]
    d8[:, 7] = dg[6 * F + 2 * grp + 1]
    assert d.tobytes() == want.tobytes(), np.flatnonzero(d != want)[:10]
    _check_trial(c, pins, free, d8)


def _check_trial(c, pins, free, d8):
    cams, trial = c["cams"], c["trial"]
    N = cams.shape[0]
    fidx = np.full(N, -1)
    fidx[free] = np.arange(len(free))
    for i in range(N):
        fi = fidx[i]
        if fi < 0:
            assert trial[i].tobytes() == cams[i].tobytes(), i
            continue
        pin = pins[fi].astype(bool)
        want = cams[i].copy()
        want[9:12] = np.where(pin[3:6], cams[i, 9:12], cams[i, 9:12] + d8[fi, 3:6])
        want[12] = cams[i, 12] if pin[6] else cams[i, 12] + d8[fi, 6]
        want[15] = cams[i, 15] if pin[7] else cams[i, 15] + d8[fi, 7]
        sel = np.r_[9:16] if not pin[:3].all() else np.r_[0:16]
        assert trial[i, sel].tobytes() == want[sel].tobytes(), (i, trial[i, sel], want[sel])


def _group_rows_equal(intr, ids):
    """The intrinsics [N, 4] of every image of a camera id are equal bit for bit."""
    for gid in np.unique(ids):
        rows = intr[ids == gid]
        assert (rows == rows[0]).all() and rows.tobytes() == np.tile(rows[0], (rows.shape[0], 1)).tobytes(), gid


N_BIG, POINTS_BIG, VIS_BIG = 200, 40_000, 0.15


def _layout(name):
    """(camera ids, unobserved images, gauge) of the N = 200 fold cases."""
    N = N_BIG
    if name == "one camera":
        return np.zeros(N, np.int64), (), {}
    if name == "singletons":
        return np.arange(N), (), {}
    ids = _uneven_ids(30)
    # in the 30-image camera (id 2, fixed): two images with fixed poses drop out, the rest stay free for their poses; in the
    # 130-image camera (id 4): fixed poses, a fixed t_x and unobserved images, one of them with a free pose
    c2, c4 = np.flatnonzero(ids == 2), np.flatnonzero(ids == 4)
    c3 = np.flatnonzero(ids == 3)
    fixed_poses = (0, int(c2[0]), int(c2[1]), int(c4[5]), int(c4[140 - 20]), int(c4[-1]))
    fixed_tx = (1, int(c3[3]), int(c4[7]), int(c4[-2]))
    unobserved = (int(c4[-1]), int(c4[-3]), int(c4[60]))
    gauge = dict(fixed_poses=fixed_poses, fixed_tx=fixed_tx, fixed_intrinsics=(2,))
    if name == "uneven, no f":
        gauge.update(refine_focal_length=False)
    elif name == "uneven, no k":
        gauge.update(refine_extra_params=False)
    return ids, unobserved, gauge


FOLD_LAYOUTS = ["one camera", "singletons", "uneven", "uneven, no f", "uneven, no k"]


@pytest.mark.parametrize("layout", FOLD_LAYOUTS)
def test_fold_and_unfold_at_200_images(monkeypatch, layout):
    ids, unobserved, gauge = _layout(layout)
    g, tr, pts, prior, R, t = _scene(31, ids, POINTS_BIG, VIS_BIG, unobserved)
    kw = dict(camera_model="SIMPLE_RADIAL", camera_ids=ids, max_iterations=1, **gauge)
    res, caps = _captured(monkeypatch, g, tr, pts, prior, R, t, **kw)
    assert len(caps) == 1
    c = caps[0]
    sizes = np.diff(c["offsets"])
    print(f"{layout}: {len(tr)} tracks, {int(pts.inlier.sum())} inliers, F = {c['S'].shape[0] // 8}, G = {sizes.size} of "
          f"{sorted(sizes.tolist())[-5:]} (largest), n' = {c['Sg'].shape[0]}, pinned group columns {c['group_pin'].sum(0).tolist()}")
    worst = _check_fold(c)
    print(f"{layout}: fold worst of the bar: group-pose {worst[0]:.3f}, group-group {worst[1]:.3f}, b' {worst[2]:.3f}")
    free, pins = rb_ba._free_and_pins(N_BIG, kw.get("fixed_poses", (0,)), kw.get("fixed_tx", (1,)), True,
                                      kw.get("refine_focal_length", True), kw.get("refine_extra_params", True),
                                      kw.get("fixed_intrinsics", ()), ids)
    assert c["S"].shape[0] == 8 * len(free)
    _check_unfold_and_trial(c, pins, free)
    _group_rows_equal(c["trial"][:, 12:16], ids)
    if layout == "one camera":
        assert sizes.tolist() == [N_BIG]
    if layout == "uneven":
        assert sizes.max() > 128 and c["group_pin"].any() and not c["group_pin"].all()
    if layout in ("one camera", "singletons"):
        n = c["Sg"].shape[0]
        assert n == {"one camera": 6 * N_BIG + 2, "singletons": 8 * N_BIG}[layout]
        _check_factor(_full(c["Sg"]), np.tril(c["Lg"]), c["bg"], c["dg"], f"{layout}: S' n'={n}")


@pytest.mark.parametrize("sizes, pinned", [((200,), ()), ((1, 2, 30, 37, 130), ((2, 0), (2, 1), (4, 1), (0, 0)))])
def test_fold_and_unfold_called_directly(sizes, pinned):
    """romab200_ba_fold and romab200_ba_unfold on a random S (its strict upper triangle NaN, which the fold must not read) and rhs
    whose pinned rows are not zero, so the fold's own pin rule shows: pinned group rows and columns of S' become e_r and their b'
    entries 0 whatever the members hold.  Then the unfold of a random d'."""
    F, G = sum(sizes), len(sizes)
    rng = np.random.default_rng(F + G)
    ids = _uneven_ids(G, sizes)
    members = np.concatenate([np.flatnonzero(ids == g) for g in range(G)]).astype(np.int32)
    offsets = np.concatenate(([0], np.cumsum(sizes))).astype(np.int32)
    gpin = np.zeros((G, 2), np.uint8)
    for g, j in pinned:
        gpin[g, j] = 1
    S = rng.normal(size=(8 * F, 8 * F))
    S[np.triu_indices(8 * F, 1)] = np.nan
    rhs = rng.normal(size=8 * F)
    n = 6 * F + 2 * G
    dv = lambda v: torch.from_numpy(np.ascontiguousarray(v)).to(DEV)        # noqa: E731
    b = dict(group_offsets=dv(offsets), group_members=dv(members), group_pin=dv(gpin.reshape(-1)), S=dv(S.reshape(-1)), rhs=dv(rhs),
             S_groups=torch.full((n * n,), np.nan, dtype=torch.float64, device=DEV), rhs_groups=torch.empty(n, dtype=torch.float64, device=DEV),
             result=torch.zeros(cabi.RB_BA_RESULT, dtype=torch.float64, device=DEV))
    cabi.call("romab200_ba_fold", "rb_ba_groups_args", num_free=F, num_groups=G, **b)
    torch.cuda.synchronize()
    c = dict(S=S, rhs=rhs, Sg=_host(b["S_groups"], (n, n)), bg=_host(b["rhs_groups"]), offsets=offsets, members=members,
             group_pin=gpin.astype(bool))
    assert np.isfinite(c["Sg"][np.tril_indices(n)]).all() and np.isfinite(c["bg"]).all()
    worst = _check_fold(c)
    print(f"groups {sizes}, pinned {pinned}: fold worst of the bar: group-pose {worst[0]:.3f}, group-group {worst[1]:.3f}, "
          f"b' {worst[2]:.3f}")
    dg = rng.normal(size=n)
    b["rhs_groups"].copy_(dv(dg))
    cabi.call("romab200_ba_unfold", "rb_ba_groups_args", num_free=F, num_groups=G, **b)
    torch.cuda.synchronize()
    d = _host(b["rhs"]).reshape(F, 8)
    grp = ids.copy()
    want = np.c_[dg[:6 * F].reshape(F, 6), dg[6 * F + 2 * grp], dg[6 * F + 2 * grp + 1]]
    assert d.tobytes() == want.tobytes(), np.flatnonzero((d != want).any(1))[:10]


def test_per_image_system_factor_at_200_images(monkeypatch):
    """The per-image 8F system of N = 200 (n = 1600): factor and solve against Higham's bounds, and the trial cameras."""
    g, tr, pts, prior, R, t = _scene(32, np.arange(N_BIG), POINTS_BIG, VIS_BIG)
    res, caps = _captured(monkeypatch, g, tr, pts, prior, R, t, camera_model="SIMPLE_RADIAL", max_iterations=1)
    c = caps[0]
    n = c["S"].shape[0]
    assert n == 8 * N_BIG and "Sg" not in c
    _check_factor(_full(c["S"]), np.tril(c["L"]), c["rhs"], c["d"], f"per-image S n={n}")
    free, pins = rb_ba._free_and_pins(N_BIG, (0,), (1,), True, True, True, ())
    _check_trial(c, pins, free, c["d"].reshape(-1, 8))


# ---- systems and whole runs against the oracles ---------------------------------------------------------------------------------
def _system_ratio(S_dev, b_dev, sy):
    """Worst |S - S_oracle| / S_abs over the lower triangle and |b - b_oracle| / b_abs (an entry whose bar is 0 must be equal)."""
    lo = np.tril_indices(S_dev.shape[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        dS, dB = np.abs(S_dev[lo] - sy["S"][lo]), np.abs(b_dev - sy["b"])
        rS = np.where(dS == 0, 0.0, dS / sy["S_abs"][lo]).max()
        rB = np.where(dB == 0, 0.0, dB / sy["b_abs"]).max()
    return rS, rB


def _oracle(g, tr, pts, prior, R, t, ids, **kw):
    a = (g.kp_offsets, g.keypoints, tr.track_offsets, tr.elements, pts.X, pts.ok, pts.inlier, prior, R, t)
    return osh.bundle_adjust(*a, ids, **kw) if ids is not None else orad.bundle_adjust(*a, **kw)


def _close(res, ref, tol):
    """Parameters within tol of the oracle's, relative to each quantity's largest magnitude (at least 1)."""
    for name, a in (("R", res.R), ("t", res.t), ("intrinsics", res.intrinsics), ("X", res.points.X)):
        b = ref[name]
        err = np.abs(a.cpu().numpy() - b).max()
        assert err <= tol * max(1.0, np.abs(b).max()), (name, err)


def _mixed_ids(N):
    """Four cameras of uneven sizes, interleaved."""
    return np.random.default_rng(N).permutation(np.repeat(np.arange(4), [1, 3, N // 4, N - 4 - N // 4]))


ORACLE_CASES = [
    # (seed, N, ids: None (per image), "one" or "mixed", loss_scale, gauge, max_iterations)
    # the shared oracle takes seconds per trial at N = 50 (its Jacobian is dense in the n' parameters), so its runs are shorter
    (40, 50, None, None, {}, 10),
    (41, 50, "one", None, {}, 4),
    (42, 50, "mixed", None, dict(fixed_poses=(0, 7), fixed_tx=(1, 9), fixed_intrinsics=(1,)), 4),
    (43, 50, "one", 1.0, {}, 4),
    (44, 50, None, 1.0, dict(fixed_poses=(0, 3), fixed_tx=(1, 30), refine_extra_params=False), 10),
    pytest.param(45, 200, None, None, {}, 2, marks=pytest.mark.slow),
    pytest.param(46, 200, "one", None, {}, 1, marks=pytest.mark.slow),
]
POINTS_ORACLE = {50: (400, 0.3), 200: (300, 0.08)}          # points, visibility


@pytest.mark.parametrize("seed, N, kind, loss_scale, gauge, max_iterations", ORACLE_CASES)
def test_systems_and_runs_match_the_oracle(monkeypatch, seed, N, kind, loss_scale, gauge, max_iterations):
    """Every trial's system while the device and the oracle share the linearization point (up to and including the first kept
    trial) entry by entry within TAU of its summation scale: the per-image S and b against oracle/bundle_radial.py, the folded S'
    and b' against oracle/bundle_shared.py (which never folds); then the whole run with the rules of test_self_calibration_gpu.py and
    test_shared_intrinsics_gpu.py, bit-identical gauges, and one observation fewer moving the oracle's S past the bar."""
    ids = None if kind is None else (np.zeros(N, np.int64) if kind == "one" else _mixed_ids(N))
    points, vis = POINTS_ORACLE[N]
    g, tr, pts, prior, R, t = _scene(seed, np.arange(N) if ids is None else ids, points, vis, size=(384, 512))
    kw = dict(loss_scale=loss_scale, max_iterations=max_iterations, function_tolerance=0.0, **gauge)
    extra = {} if ids is None else dict(camera_ids=ids)
    res, caps = _captured(monkeypatch, g, tr, pts, prior, R, t, camera_model="SIMPLE_RADIAL", **extra, **kw)
    systems = []
    ref = _oracle(g, tr, pts, prior, R, t, ids, systems=systems, **kw)
    what = f"N={N} {kind or 'per-image'} loss={loss_scale}"
    print(f"{what}: {len(tr)} tracks, {int(pts.inlier.sum())} inliers; F {res.cost[0]:.6g} -> {res.cost[-1]:.10g} "
          f"({res.accepted.sum()} of {res.accepted.size} kept); oracle {ref['cost'][-1]:.10g}")
    assert len(caps) == res.accepted.size
    worst = [0.0, 0.0]
    checked = 0
    for k, c in enumerate(caps):
        if k >= len(systems) or ref["accepted"][:k].any() or res.accepted[:k].any():
            break
        S, b = (c["Sg"], c["bg"]) if ids is not None else (c["S"], c["rhs"])
        rS, rB = _system_ratio(S, b, systems[k])
        print(f"{what} trial {k}: |S - S_oracle| {rS / U:.2f} u S_abs, |b - b_oracle| {rB / U:.2f} u b_abs (bar {TAU / U:.0f} u)")
        assert rS <= TAU and rB <= TAU, (k, rS / U, rB / U)
        worst = [max(worst[0], rS / U), max(worst[1], rB / U)]
        checked += 1
    assert checked >= 1
    # whole run: kept/rejected and pred agree up to the first trial whose rho lies within rounding of 1e-3, the costs at every trial
    tri = ref["trials"]
    for k in range(min(res.accepted.size, len(tri))):
        if abs(tri[k]["margin"]) <= 1e-6 + 1e-10 * tri[k]["F"] / abs(tri[k]["pred"]):
            break
        assert res.accepted[k] == ref["accepted"][k], k
        assert abs(res.pred[k] - tri[k]["pred"]) <= 1e-9 * abs(tri[k]["pred"]), k
    assert res.cost.size == ref["cost"].size and np.abs(res.cost - ref["cost"]).max() <= 1e-9 * ref["cost"].max()
    assert res.accepted.any()
    _close(res, ref, 1e-8)
    intr = res.intrinsics.cpu().numpy()
    assert (intr[:, 1:3] == prior[:, 1:3]).all()
    if ids is not None:
        _group_rows_equal(intr, ids)
        for gid in gauge.get("fixed_intrinsics", ()):
            assert (intr[ids == gid] == prior[ids == gid]).all()
    if not gauge.get("refine_extra_params", True):
        assert (intr[:, 3] == prior[:, 3]).all()
    R0, t0 = R.double(), t.double()
    for i in gauge.get("fixed_poses", (0,)):
        assert torch.equal(res.R[i], R0[i]) and torch.equal(res.t[i], t0[i])
    for i in gauge.get("fixed_tx", (1,)):
        assert res.t[i, 0] == t0[i, 0]
    if N < 200:                      # the bar sees one observation: without one inlier flag the oracle's S moves past it
        el = tr.elements[:, 0].cpu().numpy()
        e = int(np.flatnonzero(pts.inlier.cpu().numpy() & ~np.isin(el, gauge.get("fixed_poses", (0,))))[0])
        inl = pts.inlier.clone()
        inl[e] = False
        sys1 = []
        _oracle(g, tr, Points3D(pts.X, pts.ok, pts.num_inliers, pts.error, inl), prior, R, t, ids, systems=sys1,
                **{**kw, "max_iterations": 1})
        rS, _ = _system_ratio(sys1[0]["S"], sys1[0]["b"], systems[0])
        print(f"{what}: one observation fewer moves S by {rS / U:.3g} u S_abs")
        assert rS > 1e3 * TAU


# ---- whole runs at 200 images -----------------------------------------------------------------------------------------------------
@pytest.mark.slow
@pytest.mark.parametrize("kind", ["per-image", "one camera"])
def test_runs_at_200_images_move_every_camera_and_repeat(kind):
    """Ten trials at N = 200 with 40 000 points: every free camera moves, including those at index 128 and above (the second CTA of
    the trial-camera kernel, the second member pass of the unfold), the gauges come back bit for bit, and a rerun is byte-identical."""
    ids = np.zeros(N_BIG, np.int64) if kind == "one camera" else np.arange(N_BIG)
    g, tr, pts, prior, R, t = _scene(33, ids, POINTS_BIG, VIS_BIG)
    kw = dict(camera_model="SIMPLE_RADIAL", max_iterations=10, function_tolerance=0.0)
    if kind == "one camera":
        kw["camera_ids"] = ids
    a = bundle_adjust(g, tr, pts, prior, R, t, **kw)
    b = bundle_adjust(g, tr, pts, prior, R, t, **kw)
    print(f"{kind}: F {a.cost[0]:.6g} -> {a.cost[-1]:.10g} ({a.accepted.sum()} of {a.accepted.size} kept)")
    assert a.accepted.any() and a.cost[-1] < a.cost[0]
    for x, y in ((a.R, b.R), (a.t, b.t), (a.intrinsics, b.intrinsics), (a.points.X, b.points.X), (a.points.error, b.points.error)):
        assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()
    assert a.cost.tobytes() == b.cost.tobytes() and a.pred.tobytes() == b.pred.tobytes()
    R0, t0, intr = R.double(), t.double(), a.intrinsics.cpu().numpy()
    assert torch.equal(a.R[0], R0[0]) and torch.equal(a.t[0], t0[0]) and a.t[1, 0] == t0[1, 0]
    for i in range(1, N_BIG):
        assert not torch.equal(a.R[i], R0[i]) and not torch.equal(a.t[i, 1:], t0[i, 1:]), i
    assert (intr[:, 1:3] == prior[:, 1:3]).all() and (intr[:, 0] != prior[:, 0]).all() and (intr[:, 3] != prior[:, 3]).all()
    if kind == "one camera":
        assert (intr == intr[0]).all()
