"""numpy statement of `roma_b200.mapper`: the ranking of the candidate pairs, rules 1-6 of romab200_twoview_score with the margin of
every decision, the acceptance of a candidate, and the whole `reconstruct` loop built from the oracles of the stages
(`oracle.pose_ransac.estimate_pose(..., b=c)`, `oracle.register.triangulate`, `oracle.absolute_pose` and `oracle.bundle`)."""
from __future__ import annotations

import numpy as np

from oracle import absolute_pose as ap
from oracle import pose_ransac
from oracle.bundle import bundle_adjust
from oracle.register import triangulate
from oracle.triangulate import _arr


def rank(match_offsets, min_num_inliers, num_candidates):
    """The pairs k with n_k >= min_num_inliers matches, by n_k descending, then k ascending, the first num_candidates."""
    ns = np.diff(_arr(match_offsets, np.int64))
    ks = [k for k in range(ns.size) if ns[k] >= min_num_inliers]
    return sorted(ks, key=lambda k: (-ns[k], k))[:num_candidates]


def dlt(R, t, xn):
    """Rule 1: the homogeneous DLT point Q [n, 4] of every normalised match xn [n, 4] = (x0, y0, x1, y1) with P0 = [I | 0] and
    P1 = [R | t]: the right singular vector of the smallest singular value of A (recoverPose's rows)."""
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)
    P1 = np.c_[R, t]
    n = xn.shape[0]
    A = np.zeros((n, 4, 4))
    A[:, 0] = xn[:, 0:1] * np.array([0, 0, 1.0, 0]) - np.array([1.0, 0, 0, 0])
    A[:, 1] = xn[:, 1:2] * np.array([0, 0, 1.0, 0]) - np.array([0, 1.0, 0, 0])
    A[:, 2] = xn[:, 2:3] * P1[2] - P1[0]
    A[:, 3] = xn[:, 3:4] * P1[2] - P1[1]
    return np.linalg.svd(A)[2][:, -1, :] if n else np.zeros((0, 4))


def score(x0, x1, K0, K1, R, t, mask, max_error):
    """Rules 1-4 for one candidate: its pixels x0, x1 [n, 2], intrinsics, pose (R, t) and mask [n].  Returns dict(num_good,
    median_angle, forward, good [n], angle [n] degrees (nan where not good), X [n, 3], and the margins of every decision: err2 [n, 2]
    = each squared reprojection error minus max_error^2, depth [n, 2] = X.z and (R X + t).z, nan where the point is not masked or
    not finite)."""
    x0, x1 = np.asarray(x0, np.float64), np.asarray(x1, np.float64)
    K0, K1 = np.asarray(K0, np.float64), np.asarray(K1, np.float64)
    R, t = np.asarray(R, np.float64).reshape(3, 3), np.asarray(t, np.float64).reshape(3)
    mask = np.asarray(mask, bool)
    n = x0.shape[0]
    xn = np.concatenate([pose_ransac.normalise(x0, K0), pose_ransac.normalise(x1, K1)], axis=1)
    X = np.full((n, 3), np.nan)
    err2 = np.full((n, 2), np.nan)
    depth = np.full((n, 2), np.nan)
    good = np.zeros(n, bool)
    angle = np.full(n, np.nan)
    idx = np.flatnonzero(mask)
    with np.errstate(all="ignore"):
        Q = dlt(R, t, xn[idx])
        Xm = Q[:, :3] / Q[:, 3:4]
        fin = (Q[:, 3] != 0) & np.isfinite(Xm).all(1)
        Y = Xm @ R.T + t
        p0, p1 = Xm @ K0.T, Y @ K1.T
        e0 = ((p0[:, :2] / p0[:, 2:3] - x0[idx]) ** 2).sum(1)
        e1 = ((p1[:, :2] / p1[:, 2:3] - x1[idx]) ** 2).sum(1)
        me2 = max_error * max_error
        g = fin & (Xm[:, 2] > 0) & (Y[:, 2] > 0) & (e0 <= me2) & (e1 <= me2)
        C1 = -R.T @ t
        a, b = Xm, Xm - C1
        ang = np.degrees(np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), (a * b).sum(1)))
    f = idx[fin]
    X[f] = Xm[fin]
    depth[f] = np.c_[Xm[fin, 2], Y[fin, 2]]
    err2[f] = np.c_[e0[fin] - me2, e1[fin] - me2]
    good[idx] = g
    angle[idx[g]] = ang[g]
    num_good = int(good.sum())
    return dict(num_good=num_good, median_angle=float(np.median(angle[good])) if num_good else 0.0, forward=abs(float(t[2])), good=good,
                angle=angle, X=X, err2=err2, depth=depth)


def accept(ok, s, min_num_inliers, min_tri_angle, max_forward_motion):
    """The acceptance rule of a candidate, and whether every decision in it is clear of rounding: each squared error more than
    1e-6 px^2 from max_error^2, each depth more than 1e-9 from 0, the median more than 1e-9 degrees from min_tri_angle and forward more
    than 1e-12 from max_forward_motion (num_good is an integer, so its comparison is exact once the points are)."""
    if not ok:
        return False, True
    acc = s["num_good"] >= min_num_inliers and s["median_angle"] >= min_tri_angle and s["forward"] <= max_forward_motion
    clear = bool(np.nan_to_num(np.abs(s["err2"]), nan=np.inf).min(initial=np.inf) > 1e-6
                 and np.nan_to_num(np.abs(s["depth"]), nan=np.inf).min(initial=np.inf) > 1e-9
                 and abs(s["median_angle"] - min_tri_angle) > 1e-9 and abs(s["forward"] - max_forward_motion) > 1e-12)
    return acc, clear


def _pair_points(kp_offsets, keypoints, match_offsets, matches, pairs, k):
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    mo, mm, p = _arr(match_offsets, np.int64), _arr(matches, np.int64).reshape(-1, 2), _arr(pairs, np.int64).reshape(-1, 2)
    m = mm[mo[k]:mo[k + 1]]
    return xy[kpo[p[k, 0]] + m[:, 0]], xy[kpo[p[k, 1]] + m[:, 1]]


def initialize(pairs, kp_offsets, keypoints, match_offsets, matches, K, init_pair=None, num_candidates=256, min_num_inliers=100,
               max_error=4.0, min_tri_angle=16.0, max_forward_motion=0.95, confidence=0.999, max_iters=10000, seed=0, first_only=False):
    """`initialize_reconstruction` restated: returns dict(cand, images [C, 2], ok, R, t, mask (list), stats (list of `score` dicts),
    accepted, clear, chosen).  With first_only, the candidates after the chosen one are not evaluated (their lists stop there)."""
    p, K = _arr(pairs, np.int64).reshape(-1, 2), _arr(K, np.float64)
    if init_pair is None:
        cand = rank(match_offsets, min_num_inliers, num_candidates)
    else:
        i, j = init_pair
        cand = [int(np.flatnonzero(((p[:, 0] == i) & (p[:, 1] == j)) | ((p[:, 0] == j) & (p[:, 1] == i)))[0])]
    norm_thresh = max_error / np.mean((K[:, 0, 0] + K[:, 1, 1]) / 2)
    out = dict(cand=cand, images=p[cand], ok=[], R=[], t=[], mask=[], stats=[], accepted=[], clear=[], chosen=-1)
    for c, k in enumerate(cand):
        x0, x1 = _pair_points(kp_offsets, keypoints, match_offsets, matches, p, k)
        i, j = p[k]
        res = pose_ransac.estimate_pose(x0, x1, K[i], K[j], norm_thresh, confidence, max_iters, seed, b=c)
        ok = res is not None
        R, t, mask = (res[0], res[1].ravel(), res[2]) if ok else (np.zeros((3, 3)), np.zeros(3), np.zeros(len(x0), bool))
        s = score(x0, x1, K[i], K[j], R, t, mask, max_error)
        acc, clear = accept(ok, s, min_num_inliers, min_tri_angle, max_forward_motion)
        for name, v in (("ok", ok), ("R", R), ("t", t), ("mask", mask), ("stats", s), ("accepted", acc), ("clear", clear)):
            out[name].append(v)
        if acc and out["chosen"] < 0:
            out["chosen"] = c
            if first_only:
                break
    return out


def reconstruct(pairs, kp_offsets, keypoints, match_offsets, matches, track_offsets, elements, K, *, init_pair=None, init_num_candidates=256,
                init_min_num_inliers=100, init_max_error=4.0, init_min_tri_angle=16.0, init_max_forward_motion=0.95, tri_max_error=4.0,
                tri_min_angle=1.5, abs_max_error=12.0, abs_min_inliers=30, ba_loss_scale=None, ba_max_iterations=50, seed=0):
    """The loop of `reconstruct` with the oracles alone.  Returns dict(init, registered (sorted list), R, t, points, rounds,
    termination)."""
    K = _arr(K, np.float64)
    N = K.shape[0]
    init = initialize(pairs, kp_offsets, keypoints, match_offsets, matches, K, init_pair, init_num_candidates, init_min_num_inliers,
                      init_max_error, init_min_tri_angle, init_max_forward_motion, seed=seed, first_only=True)
    R, t = np.zeros((N, 3, 3)), np.zeros((N, 3))
    if init["chosen"] < 0:
        return dict(init=init, registered=[], R=R, t=t, points=None, rounds=[], termination="no_initial_pair")
    c = init["chosen"]
    a, b = (int(v) for v in init["images"][c])
    R[a], R[b], t[b] = np.eye(3), init["R"][c], init["t"][c]
    reg, rounds = sorted((a, b)), []

    def tri(R, t):
        return triangulate(kp_offsets, keypoints, track_offsets, elements, K, R, t, reg, max_error=tri_max_error, min_angle=tri_min_angle,
                           seed=seed)

    while True:
        rest = [i for i in range(N) if i not in reg]
        pts = tri(R, t)
        ba = bundle_adjust(kp_offsets, keypoints, track_offsets, elements, pts["X"], pts["ok"], pts["inlier"], K, R, t,
                           fixed_poses=[a] + rest, fixed_tx=[b], loss_scale=ba_loss_scale, max_iterations=ba_max_iterations)
        R, t = ba["R"].copy(), ba["t"].copy()
        pts = tri(R, t)
        rnd = dict(registered=list(reg), ba_termination=ba["termination"], ba_cost=(float(ba["cost"][0]), float(ba["cost"][-1])),
                   ok_tracks=int(np.sum(pts["ok"])), added=[])
        rounds.append(rnd)
        if not rest:
            termination = "all_registered"
            break
        corr = ap.gather(kp_offsets, keypoints, track_offsets, elements, pts["ok"], pts["X"], rest)
        for i, (x, X) in zip(rest, corr):
            res = ap.estimate(x, X, K[i], max_error=abs_max_error, seed=seed)
            if res["ok"] and res["num_inliers"] >= abs_min_inliers:
                R[i], t[i] = res["R"], res["t"]
                rnd["added"].append(i)
        if not rnd["added"]:
            termination = "no_image_added"
            break
        reg = sorted(reg + rnd["added"])
    return dict(init=init, registered=reg, R=R, t=t, points=pts, rounds=rounds, termination=termination)
