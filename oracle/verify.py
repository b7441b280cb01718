"""numpy statement of `roma_b200.verify_matches` (include/romab200.h, INTEGRATION.md) around a fundamental-matrix estimator it is
given: rules 1 (points), 3 (accept) and 4 (output).  Rule 2 is the estimator itself: on the host `oracle.fundamental_ransac.
find_fundamental` (see `host_estimator`), in GPU tests the device's `find_fundamental_batched` called pair by pair."""
from __future__ import annotations

import numpy as np


def _arr(graph, name, dtype):
    v = graph[name] if isinstance(graph, dict) else getattr(graph, name)
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype)


def pair_points(pairs, graph):
    """Rule 1: per pair k = (i, j), (x0, x1) float64 [M_k, 2]: keypoints[kp_offsets[i] + a] and keypoints[kp_offsets[j] + b] of its
    matches (a, b), in match order.  ValueError for a match id outside its image's keypoints."""
    kp = _arr(graph, "kp_offsets", np.int64)
    xy = _arr(graph, "keypoints", np.float32).reshape(-1, 2)
    mo = _arr(graph, "match_offsets", np.int64)
    m = _arr(graph, "matches", np.int64).reshape(-1, 2)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    out = []
    for k, (i, j) in enumerate(pairs):
        a, b = m[mo[k]:mo[k + 1], 0], m[mo[k]:mo[k + 1], 1]
        if ((a < 0) | (a >= kp[i + 1] - kp[i]) | (b < 0) | (b >= kp[j + 1] - kp[j])).any():
            raise ValueError("verify: a match id lies outside its image's keypoints")
        out.append((xy[kp[i] + a].astype(np.float64), xy[kp[j] + b].astype(np.float64)))
    return out


def verify(pairs, graph, estimate, min_inliers=15):
    """pairs [P, 2], a match graph (a dict or object with kp_offsets, keypoints, match_offsets, matches, match_scores) and
    estimate(k, x0, x1) -> (F [3, 3] or None, mask bool [M_k]), rule 2 for pair k; it is not called for pairs of fewer than 7
    matches, which get no model.  Returns a dict of numpy arrays: F [P, 3, 3] float64 (zero without a model), ok, num_inliers int64,
    accepted [P], and the verified match_offsets [P + 1] int64, matches [M', 2] int32, match_scores [M'] fp32."""
    mo = _arr(graph, "match_offsets", np.int64)
    m = _arr(graph, "matches", np.int32).reshape(-1, 2)
    s = _arr(graph, "match_scores", np.float32).reshape(-1)
    pts = pair_points(pairs, graph)
    P = len(pts)
    F = np.zeros((P, 3, 3))
    ok = np.zeros(P, bool)
    num_inliers = np.zeros(P, np.int64)
    keep = np.zeros(m.shape[0], bool)
    for k, (x0, x1) in enumerate(pts):
        if len(x0) < 7:
            continue
        Fk, mask = estimate(k, x0, x1)
        mask = np.asarray(mask, bool).reshape(-1)
        if Fk is not None:
            F[k], ok[k] = np.asarray(Fk, np.float64).reshape(3, 3), True
        num_inliers[k] = int(mask.sum())                                  # rule 3
        if ok[k] and num_inliers[k] >= min_inliers:
            keep[mo[k]:mo[k + 1]] = mask                                  # rule 4
    accepted = ok & (num_inliers >= min_inliers)
    out_offsets = np.zeros(P + 1, np.int64)
    out_offsets[1:] = np.cumsum(np.where(accepted, num_inliers, 0))
    return dict(F=F, ok=ok, num_inliers=num_inliers, accepted=accepted, match_offsets=out_offsets, matches=m[keep].reshape(-1, 2),
                match_scores=s[keep])


def host_estimator(threshold, confidence, max_iters, seed=0):
    """estimate(k, x0, x1) of `verify` by the numpy restatement of the device estimator (oracle/fundamental_ransac.py)."""
    from oracle.fundamental_ransac import find_fundamental
    from roma_b200.geometry import magsac_tables

    tables = magsac_tables()
    return lambda k, x0, x1: find_fundamental(x0, x1, threshold, confidence, max_iters, tables, seed)
