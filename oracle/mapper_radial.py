"""The loop of `roma_b200.reconstruct(..., intrinsics=...)` with the numpy oracles alone: `oracle/mapper.py`'s loop with the stages
that take pinhole cameras run on keypoints undistorted under the current SIMPLE_RADIAL intrinsics (`oracle/camera.py`) and each
round's bundle adjustment in SIMPLE_RADIAL on the raw keypoints (`oracle/bundle_radial.py`).  It restates the pinhole loop rather
than sharing it, so the two must be kept in step by hand."""
from __future__ import annotations

import numpy as np

from oracle import absolute_pose as ap
from oracle.bundle_radial import bundle_adjust
from oracle.camera import undistort_graph_keypoints
from oracle.mapper import initialize
from oracle.register import triangulate
from oracle.triangulate import _arr

MIN_REGISTERED_TO_REFINE = 3


def pinhole_K(intr):
    K = np.zeros((intr.shape[0], 3, 3))
    K[:, 0, 0] = K[:, 1, 1] = intr[:, 0]
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = intr[:, 1], intr[:, 2], 1.0
    return K


def reconstruct(pairs, kp_offsets, keypoints, match_offsets, matches, track_offsets, elements, intrinsics, *, refine_intrinsics=False,
                init_pair=None, init_num_candidates=256, init_min_num_inliers=100, init_max_error=4.0, init_min_tri_angle=16.0,
                init_max_forward_motion=0.95, tri_max_error=4.0, tri_min_angle=1.5, abs_max_error=12.0, abs_min_inliers=30,
                ba_loss_scale=None, ba_max_iterations=50, seed=0):
    """Returns dict(init, registered (sorted list), R, t, intrinsics, points, rounds, termination)."""
    cur = _arr(intrinsics, np.float64).copy()
    N = cur.shape[0]
    kpo = _arr(kp_offsets, np.int64)
    und = undistort_graph_keypoints(kpo, keypoints, cur)[0]
    K = pinhole_K(cur)
    init = initialize(pairs, kpo, und, match_offsets, matches, K, init_pair, init_num_candidates, init_min_num_inliers, init_max_error,
                      init_min_tri_angle, init_max_forward_motion, seed=seed, first_only=True)
    R, t = np.zeros((N, 3, 3)), np.zeros((N, 3))
    if init["chosen"] < 0:
        return dict(init=init, registered=[], R=R, t=t, intrinsics=cur, points=None, rounds=[], termination="no_initial_pair")
    c = init["chosen"]
    a, b = (int(v) for v in init["images"][c])
    R[a], R[b], t[b] = np.eye(3), init["R"][c], init["t"][c]
    reg, rounds = sorted((a, b)), []

    def tri(R, t):
        return triangulate(kpo, und, track_offsets, elements, K, R, t, reg, max_error=tri_max_error, min_angle=tri_min_angle, seed=seed)

    while True:
        rest = [i for i in range(N) if i not in reg]
        pts = tri(R, t)
        free = refine_intrinsics and len(reg) >= MIN_REGISTERED_TO_REFINE
        ba = bundle_adjust(kpo, keypoints, track_offsets, elements, pts["X"], pts["ok"], pts["inlier"], cur, R, t, fixed_poses=[a] + rest,
                           fixed_tx=[b], refine_focal_length=free, refine_extra_params=free, fixed_intrinsics=rest,
                           loss_scale=ba_loss_scale, max_iterations=ba_max_iterations)
        R, t = ba["R"].copy(), ba["t"].copy()
        if free:
            cur = ba["intrinsics"].copy()
            K = pinhole_K(cur)
            und = undistort_graph_keypoints(kpo, keypoints, cur)[0]
        pts = tri(R, t)
        rnd = dict(registered=list(reg), ba_termination=ba["termination"], ba_cost=(float(ba["cost"][0]), float(ba["cost"][-1])),
                   ok_tracks=int(np.sum(pts["ok"])), added=[])
        rounds.append(rnd)
        if not rest:
            termination = "all_registered"
            break
        corr = ap.gather(kpo, und, track_offsets, elements, pts["ok"], pts["X"], rest)
        for i, (x, X) in zip(rest, corr):
            res = ap.estimate(x, X, K[i], max_error=abs_max_error, seed=seed)
            if res["ok"] and res["num_inliers"] >= abs_min_inliers:
                R[i], t[i] = res["R"], res["t"]
                rnd["added"].append(i)
        if not rnd["added"]:
            termination = "no_image_added"
            break
        reg = sorted(reg + rnd["added"])
    return dict(init=init, registered=reg, R=R, t=t, intrinsics=cur, points=pts, rounds=rounds, termination=termination)
