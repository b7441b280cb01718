"""numpy statement of `roma_b200.triangulate_tracks` (include/romab200.h, INTEGRATION.md), rules 1-6 in float64: `np.linalg.eigh`
for every DLT, `oracle.ransac.draw_distinct` for the drawn pairs, `np.linalg.solve` for the Gauss-Newton steps.  The device's
Jacobi solver and sums round differently, so the result agrees with it to a tolerance, and the decisions (inlier, ok) agree
wherever they are not within rounding of a threshold: each track also reports its decision margins."""
from __future__ import annotations

import math
from itertools import combinations

import numpy as np

from oracle.ransac import draw_distinct

CTR = 0x54524900            # RB_TRI_CTR
GN_ITERS = 10               # RB_TRI_GN_ITERS


def _arr(v, dtype):
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype)


def _dlt(x, P):
    """Rule 3 for a stack of observation sets: x [..., n, 2], P [..., n, 3, 4] -> the dehomogenised smallest eigenvector of A^T A."""
    rows = np.concatenate((x[..., 0:1, None] * P[..., 2:3, :] - P[..., 0:1, :], x[..., 1:2, None] * P[..., 2:3, :] - P[..., 1:2, :]), -2)
    rows = rows.reshape(*rows.shape[:-3], -1, 4)
    _, V = np.linalg.eigh(np.einsum("...ri,...rj->...ij", rows, rows))
    with np.errstate(divide="ignore", invalid="ignore"):
        return V[..., :3, 0] / V[..., 3:4, 0]


def _project(X, P, Rz, tz, x):
    """(err2, depth) of points X [..., 3] in observations x [L, 2] with cameras P [L, 3, 4]: shapes [..., L]."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        p = np.einsum("lij,...j->...li", P[:, :, :3], X) + P[:, :, 3]
        du, dv = p[..., 0] / p[..., 2] - x[:, 0], p[..., 1] / p[..., 2] - x[:, 1]
        return du * du + dv * dv, np.einsum("lj,...j->...l", Rz, X) + tz


def _gauss_newton(X, P, x):
    """Rule 5's Gauss-Newton on the summed squared reprojection error over observations x [n, 2] with cameras P [n, 3, 4].  Returns
    (X, the length of the first step whose cost comparison lies within rounding, 0 if none).  A residual is the difference of two
    coordinates of hundreds of px, so its rounding is about 1e-13 px and the cost's about 1e-13 px^2 per observation: a step whose
    cost change is below 1e-11 px^2 per observation may be kept by one implementation and rejected by another, and the point is
    then determined only to about that step's length."""
    contested = 0.0
    def sums(X):
        p = P[:, :, :3] @ X + P[:, :, 3]
        uv = p[:, :2] / p[:, 2:3]
        r = uv - x
        J = (P[:, :2, :3] - uv[:, :, None] * P[:, 2:3, :3]) / p[:, 2, None, None]        # [n, 2, 3]
        return np.einsum("nki,nkj->ij", J, J), np.einsum("nki,nk->i", J, r), float((r * r).sum())

    with np.errstate(all="ignore"):
        JJ, Jr, cost = sums(X)
        for _ in range(GN_ITERS):
            try:
                d = np.linalg.solve(JJ, -Jr)
            except np.linalg.LinAlgError:
                break
            if not np.isfinite(d).all():
                break
            X1 = X + d
            JJ1, Jr1, cost1 = sums(X1)
            if not contested and abs(cost1 - cost) <= 1e-11 * len(x):
                contested = float(np.linalg.norm(d))
            if not cost1 < cost:
                break
            X, JJ, Jr, cost = X1, JJ1, Jr1, cost1
    return X, contested


def hypothesis_pairs(L, k, max_hypotheses, seed):
    """Rule 2: the element pairs (p, q) of track k's hypotheses, [H, 2]."""
    if L * (L - 1) // 2 <= max_hypotheses:
        return np.array(list(combinations(range(L), 2)), np.int64).reshape(-1, 2)
    return np.array([draw_distinct(2, L, seed, lambda s, h=h: (h, s, k, CTR)) for h in range(max_hypotheses)], np.int64)


def triangulate(kp_offsets, keypoints, track_offsets, elements, K, R, t, max_error=4.0, min_angle=1.5, max_hypotheses=256, seed=0):
    """Rules 1-6 per track.  Returns a dict of numpy arrays: X [T, 3], ok [T], num_inliers [T] int32, error [T], inlier [E] (zero
    where not ok), and the decision margins: err2_margin [E] = max_error^2 - err^2 and depth [E] at the final point (NaN where the
    track has no final point), angle_margin [T] (the largest angle minus min_angle, radians; inf where it was not decided) and
    hyp_margin [T], the smallest |max_error^2 - err^2| and |depth| over every hypothesis and element (inf without hypotheses), and
    gn_step [T], the length of the first Gauss-Newton step whose keep-or-stop decision lies within rounding (0 if none; X is
    determined only to about that length, see `_gauss_newton`).
    ValueError for an element id outside its image's keypoints."""
    kp = _arr(kp_offsets, np.int64)
    xy = _arr(keypoints, np.float32).reshape(-1, 2).astype(np.float64)
    off = _arr(track_offsets, np.int64)
    el = _arr(elements, np.int64).reshape(-1, 2)
    K, R, t = _arr(K, np.float64), _arr(R, np.float64), _arr(t, np.float64)
    N, T, E = kp.size - 1, off.size - 1, el.shape[0]
    img, ids = el[:, 0], el[:, 1]
    if ((img < 0) | (img >= N)).any() or ((ids < 0) | (ids >= kp[np.clip(img, 0, N - 1) + 1] - kp[np.clip(img, 0, N - 1)])).any():
        raise ValueError("triangulate: a track element lies outside its image's keypoints")
    P_all = K @ np.concatenate((R, t[:, :, None]), 2)                               # rule 1
    C_all = -np.einsum("nji,nj->ni", R, t)
    thr2, amin = float(max_error) ** 2, float(min_angle) * (math.pi / 180.0)
    out = dict(X=np.zeros((T, 3)), ok=np.zeros(T, bool), num_inliers=np.zeros(T, np.int32), error=np.zeros(T), inlier=np.zeros(E, bool),
               err2_margin=np.full(E, np.nan), depth=np.full(E, np.nan), angle_margin=np.full(T, np.inf), hyp_margin=np.full(T, np.inf),
               gn_step=np.zeros(T))
    for k in range(T):
        b, L = int(off[k]), int(off[k + 1] - off[k])
        if L < 2:
            continue
        im = img[b:b + L]
        x, P, Rz, tz = xy[kp[im] + ids[b:b + L]], P_all[im], R[im, 2], t[im, 2]
        pq = hypothesis_pairs(L, k, max_hypotheses, seed)
        Xh = _dlt(x[pq], P[pq])                                                     # [H, 3]
        err2, depth = _project(Xh, P, Rz, tz, x)                                    # [H, L]
        hidx = np.arange(len(pq))
        cand = (im[pq[:, 0]] != im[pq[:, 1]]) & np.isfinite(Xh).all(1)
        valid = cand & (depth[hidx, pq[:, 0]] > 0) & (depth[hidx, pq[:, 1]] > 0)
        if cand.any():
            with np.errstate(invalid="ignore"):
                m = np.nan_to_num(np.abs(thr2 - err2[cand]), nan=np.inf)
            out["hyp_margin"][k] = min(m.min(), np.abs(depth[cand]).min())
        if not valid.any():
            continue
        inl = (depth > 0) & (err2 <= thr2)
        cnt = np.where(valid, inl.sum(1), -1)
        h = int(np.argmax(cnt))                                                     # rule 4: first of the most inliers
        if cnt[h] < 2:
            continue
        S = inl[h]
        X = _dlt(x[S], P[S])                                                        # rule 5
        if not np.isfinite(X).all():
            X = Xh[h]
        X, out["gn_step"][k] = _gauss_newton(X, P[S], x[S])
        e2, d = _project(X, P, Rz, tz, x)
        out["err2_margin"][b:b + L], out["depth"][b:b + L] = thr2 - e2, d
        fin = (d > 0) & (e2 <= thr2)
        # rule 6: the largest angle over inlier pairs in distinct images
        idx = np.flatnonzero(fin)
        ok = False
        if idx.size >= 2:
            ray = X - C_all[im[idx]]
            i1, i2 = np.triu_indices(idx.size, 1)
            dist = im[idx][i1] != im[idx][i2]
            if dist.any():
                a, c = ray[i1[dist]], ray[i2[dist]]
                ang = np.arctan2(np.linalg.norm(np.cross(a, c), axis=1), (a * c).sum(1))
                out["angle_margin"][k] = ang.max() - amin
                ok = bool(ang.max() >= amin)
        if ok:
            out["X"][k], out["ok"][k], out["num_inliers"][k] = X, True, idx.size
            out["error"][k] = np.sqrt(e2[fin]).mean()
            out["inlier"][b:b + L] = fin
    return out
