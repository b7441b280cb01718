"""numpy statement of `roma_b200.triangulate_tracks(..., images=...)` and of the incremental loop it serves.

`triangulate` restates the registered-images rule through `oracle.triangulate.triangulate` itself, without a second copy of rules 1-6.
Each image that is not listed gets the camera K = I, R = diag(1, 1, 0), t = (0, 0, -1).  Every depth (R X + t)_z is then -1, so its
elements are never inliers (rule 4).  A pair that contains one is skipped but keeps its index h (rule 3 skips a hypothesis with a
depth <= 0), and they never enter the refinement or the angle test.  That is exactly the rule of include/romab200.h.  The stand-in
camera adds only decisions that cannot flip (depth -1) to the margins, so the margins stay conservative.  oracle/triangulate.py
remains the statement of the images=None path.

`incremental` runs the loop of tests/test_absolute_pose_gpu.py with the oracles alone: triangulate with the registered cameras,
register the rest (`oracle.absolute_pose`), repeat, then bundle-adjust (`oracle.bundle`) with the never-registered images fixed."""
from __future__ import annotations

import numpy as np

from oracle import absolute_pose as ap
from oracle.bundle import bundle_adjust
from oracle.triangulate import _arr
from oracle.triangulate import triangulate as _triangulate


def triangulate(kp_offsets, keypoints, track_offsets, elements, K, R, t, images, max_error=4.0, min_angle=1.5, max_hypotheses=256,
                seed=0):
    """oracle.triangulate.triangulate with only `images` registered; the same outputs and margins (the margins of an element of an
    unlisted image describe the stand-in camera and need no check)."""
    K, R, t = _arr(K, np.float64).copy(), _arr(R, np.float64).copy(), _arr(t, np.float64).copy()
    out = np.ones(K.shape[0], bool)
    out[list(images)] = False
    K[out], R[out], t[out] = np.eye(3), np.diag([1.0, 1.0, 0.0]), (0.0, 0.0, -1.0)
    return _triangulate(kp_offsets, keypoints, track_offsets, elements, K, R, t, max_error=max_error, min_angle=min_angle,
                        max_hypotheses=max_hypotheses, seed=seed)


def incremental(kp_offsets, keypoints, track_offsets, elements, K, R, t, start=(0, 1), candidates=None, tri_max_error=4.0,
                max_error=12.0, min_inliers=30, seed=0):
    """From the true cameras of `start`: triangulate with the registered cameras, register the `candidates` not yet registered
    (all images by default), keep the accepted ones, and repeat until none is added; then bundle_adjust with the images never
    registered added to fixed_poses (their cameras zero).  Returns dict(registered, R, t) with the adjusted cameras."""
    K, Rt, tt = _arr(K, np.float64), _arr(R, np.float64), _arr(t, np.float64)
    N = K.shape[0]
    cand = list(range(N)) if candidates is None else list(candidates)
    Rw, tw = np.zeros((N, 3, 3)), np.zeros((N, 3))
    reg = sorted(start)
    Rw[reg], tw[reg] = Rt[reg], tt[reg]
    while True:
        pts = triangulate(kp_offsets, keypoints, track_offsets, elements, K, Rw, tw, reg, max_error=tri_max_error, seed=seed)
        rest = [i for i in cand if i not in reg]
        corr = ap.gather(kp_offsets, keypoints, track_offsets, elements, pts["ok"], pts["X"], rest)
        new = []
        for i, (x, X) in zip(rest, corr):
            res = ap.estimate(x, X, K[i], max_error=max_error, seed=seed)
            if res["ok"] and res["num_inliers"] >= min_inliers:
                Rw[i], tw[i] = res["R"], res["t"]
                new.append(i)
        if not new:
            break
        reg = sorted(reg + new)
    fixed = sorted({min(start)} | {i for i in range(N) if i not in reg})
    ba = bundle_adjust(kp_offsets, keypoints, track_offsets, elements, pts["X"], pts["ok"], pts["inlier"], K, Rw, tw, fixed_poses=fixed)
    return dict(registered=reg, R=ba["R"], t=ba["t"])
