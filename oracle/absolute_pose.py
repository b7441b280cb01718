"""numpy statement of `roma_b200.estimate_absolute_pose_batched` (include/romab200.h, INTEGRATION.md), rules 1-7 in float64:
Lambda Twist P3P (Persson & Nordberg, ECCV 2018) on three bearings, plain RANSAC with OpenCV's stopping rule replayed one
hypothesis at a time, and Gauss-Newton on the inliers' reprojection error.  `np.linalg.eigh` and `np.linalg.solve` round
differently from the device's Jacobi and Cholesky, so the result agrees with it to a tolerance, and the decisions agree wherever
they are not within rounding of a threshold: every call also reports its decision margins.  `gather` restates the
correspondences of `register_images`."""
from __future__ import annotations

import math

import numpy as np

from oracle.ransac import draw_distinct, ransac_update_num_iters

CTR = 0x41425300            # RB_ABS_CTR
GN_ITERS = 10               # RB_ABS_GN_ITERS
POLISH_ITERS = 5            # RB_ABS_POLISH_ITERS


def _arr(v, dtype):
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype)


def bearings(x, K):
    """Rule 1: f = normalise(K^-1 [x, y, 1]) for x [n, 2]."""
    h = np.concatenate((x, np.ones((len(x), 1))), 1) @ np.linalg.inv(K).T
    return h / np.linalg.norm(h, axis=1, keepdims=True)


def _cubic_roots(b, c, d):
    """The real roots of g^3 + b g^2 + c g + d, in descending order: Cardano or the trigonometric form, then two Newton steps each."""
    p, q = c - b * b / 3.0, 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    disc = q * q / 4.0 + p * p * p / 27.0
    if disc > 0.0:
        s = math.sqrt(disc)
        roots = [math.copysign(abs(-q / 2.0 + s) ** (1.0 / 3.0), -q / 2.0 + s) +
                 math.copysign(abs(-q / 2.0 - s) ** (1.0 / 3.0), -q / 2.0 - s) - b / 3.0]
    else:
        r = math.sqrt(max(-p / 3.0, 0.0))
        arg = 0.0 if r == 0.0 else min(max(-q / (2.0 * r * r * r), -1.0), 1.0)
        phi = math.acos(arg)
        roots = [2.0 * r * math.cos((phi - 2.0 * math.pi * k) / 3.0) - b / 3.0 for k in range(3)]
    out = []
    for g in roots:
        for _ in range(2):
            f, df = ((g + b) * g + c) * g + d, (3.0 * g + 2.0 * b) * g + c
            if df != 0.0:
                g1 = g - f / df
                if math.isfinite(g1):
                    g = g1
        out.append(g)
    return sorted(out, reverse=True)


def _canonical(u):
    """u with the sign that makes its first largest-magnitude entry positive."""
    return -u if u[int(np.argmax(np.abs(u)))] < 0 else u


def p3p(f, X):
    """Rule 3: Lambda Twist on bearings f [3, 3] and world points X [3, 3].  Returns the list of (R [3, 3], t [3]) with x ~ R X + t,
    in the order of the header: among the real roots g of the cubic (descending) whose D0 = D1 + g D2 is indefinite, the one with the
    largest ratio |sigma2| / |sigma1| (the first on a tie); its two lines (u1 - s u2 first), on each the roots tau > 0 ascending."""
    a12, a13, a23 = (float(np.dot(X[i] - X[j], X[i] - X[j])) for i, j in ((0, 1), (0, 2), (1, 2)))
    b12, b13, b23 = float(f[0] @ f[1]), float(f[0] @ f[2]), float(f[1] @ f[2])
    M12 = np.array([[1.0, -b12, 0.0], [-b12, 1.0, 0.0], [0.0, 0.0, 0.0]])
    M13 = np.array([[1.0, 0.0, -b13], [0.0, 0.0, 0.0], [-b13, 0.0, 1.0]])
    M23 = np.array([[0.0, 0.0, 0.0], [0.0, 1.0, -b23], [0.0, -b23, 1.0]])
    D1, D2 = M12 * a23 - M23 * a12, M13 * a23 - M23 * a13
    c3 = np.linalg.det(D2)
    c2 = sum(np.linalg.det(np.stack([D1[:, k] if k == j else D2[:, k] for k in range(3)], 1)) for j in range(3))
    c1 = sum(np.linalg.det(np.stack([D2[:, k] if k == j else D1[:, k] for k in range(3)], 1)) for j in range(3))
    c0 = np.linalg.det(D1)
    if not (c3 != 0.0 and math.isfinite(c3)):
        return []
    best = None                    # the root whose D0 is indefinite with the largest |sigma| ratio, ties to the first
    for g in _cubic_roots(c2 / c3, c1 / c3, c0 / c3):
        w, V = np.linalg.eigh(D1 + g * D2)
        order = np.argsort(-np.abs(w), kind="stable")
        (s1, s2), (u1, u2) = w[order[:2]], (_canonical(V[:, order[0]]), _canonical(V[:, order[1]]))
        if not s1 * s2 < 0.0:
            continue
        ratio = abs(s2) / abs(s1)
        if best is None or ratio > best[0]:
            best = (ratio, s1, s2, u1, u2)
    sols = []
    if best is not None:
        _, s1, s2, u1, u2 = best
        if s1 < 0.0:
            s1, s2, u1, u2 = s2, s1, u2, u1
        s = math.sqrt(-s2 / s1)
        for n in (u1 - s * u2, u1 + s * u2):
            if n[0] == 0.0:
                continue
            w0, w1 = -n[1] / n[0], -n[2] / n[0]
            al, be = np.array([w0, 1.0, 0.0]), np.array([w1, 0.0, 1.0])
            A, B, C = be @ D2 @ be, 2.0 * (al @ D2 @ be), al @ D2 @ al
            disc = B * B - 4.0 * A * C
            if not (A != 0.0 and disc >= 0.0):
                continue
            qq = -0.5 * (B + math.copysign(math.sqrt(disc), B))
            taus = sorted((qq / A, C / qq)) if qq != 0.0 else []
            for tau in taus:
                if not tau > 0.0:
                    continue
                l2 = math.sqrt(a23 / (tau * tau - 2.0 * b23 * tau + 1.0))
                lam = np.array([w0 * l2 + w1 * tau * l2, l2, tau * l2])
                if not lam[0] > 0.0:
                    continue
                lam = _polish(lam, (a12, a13, a23), (b12, b13, b23))
                Y = lam[:, None] * f
                Xm = np.stack((X[0] - X[1], X[0] - X[2], np.cross(X[0] - X[1], X[0] - X[2])), 1)
                Ym = np.stack((Y[0] - Y[1], Y[0] - Y[2], np.cross(Y[0] - Y[1], Y[0] - Y[2])), 1)
                with np.errstate(all="ignore"):
                    R = Ym @ np.linalg.inv(Xm)
                    t = Y[0] - R @ X[0]
                if np.isfinite(R).all() and np.isfinite(t).all():
                    sols.append((R, t))
    return sols


def _polish(lam, a, b):
    """Lambda Twist's Gauss-Newton on the depths: at most POLISH_ITERS Newton steps on the three distance residuals
    l_i^2 + l_j^2 - 2 b_ij l_i l_j - a_ij, a step kept only when it lowers their sum of squares."""
    pairs = ((0, 1), (0, 2), (1, 2))

    def res(l):
        return np.array([l[i] * l[i] + l[j] * l[j] - 2.0 * b[k] * l[i] * l[j] - a[k] for k, (i, j) in enumerate(pairs)])

    r = res(lam)
    for _ in range(POLISH_ITERS):
        J = np.zeros((3, 3))
        for k, (i, j) in enumerate(pairs):
            J[k, i], J[k, j] = 2.0 * lam[i] - 2.0 * b[k] * lam[j], 2.0 * lam[j] - 2.0 * b[k] * lam[i]
        try:
            d = np.linalg.solve(J, r)
        except np.linalg.LinAlgError:
            break
        l1 = lam - d
        r1 = res(l1)
        if not (np.isfinite(l1).all() and r1 @ r1 < r @ r):
            break
        lam, r = l1, r1
    return lam


def exp_so3(w):
    """Bundle rule 3's Exp: Rodrigues, with the small-angle branch I + [w]x for theta^2 <= 2^-52."""
    t2 = float(w @ w)
    Kx = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if t2 > 2.0 ** -52:
        th = math.sqrt(t2)
        k = w / th
        Kk = Kx / th
        return math.cos(th) * np.eye(3) + (1.0 - math.cos(th)) * np.outer(k, k) + math.sin(th) * Kk
    return np.eye(3) + Kx


def reprojection(R, t, K, x, X):
    """(err2 [n], depth [n]) of world points X [n, 3] against pixels x [n, 2] under x ~ K (R X + t)."""
    Y = X @ R.T + t
    p = Y @ K.T
    with np.errstate(all="ignore"):
        d = p[:, :2] / p[:, 2:3] - x
    return (d * d).sum(1), Y[:, 2]


def _sums(R, t, K, x, X):
    """Gauss-Newton sums of rule 5 at (R, t): J^T J [6, 6], J^T r [6], cost, and the depths."""
    Y = X @ R.T + t
    p = Y @ K.T
    with np.errstate(all="ignore"):
        uv = p[:, :2] / p[:, 2:3]
        r = uv - x
        G = (K[None, :2, :] - uv[:, :, None] * K[None, 2:3, :]) / p[:, 2, None, None]          # d uv / d Y  [n, 2, 3]
        Jw = np.cross((X @ R.T)[:, None, :], G)                                                  # (R X) x g, the d omega part
    J = np.concatenate((Jw, G), 2)                                                               # [n, 2, 6]
    return np.einsum("nki,nkj->ij", J, J), np.einsum("nki,nk->i", J, r), float((r * r).sum()), Y[:, 2]


def refine(R, t, K, x, X):
    """Rule 5's Gauss-Newton over the used points.  Returns (R, t, the cost changes cost - cost1 of every trial, the length of the
    first step whose cost change lies within rounding, 0 if none)."""
    changes, contested = [], 0.0
    with np.errstate(all="ignore"):
        H, g, cost, _ = _sums(R, t, K, x, X)
        for _ in range(GN_ITERS):
            try:
                d = np.linalg.solve(H, -g)
            except np.linalg.LinAlgError:
                break
            if not np.isfinite(d).all():
                break
            R1, t1 = exp_so3(d[:3]) @ R, t + d[3:]
            H1, g1, cost1, depth1 = _sums(R1, t1, K, x, X)
            changes.append(cost - cost1)
            if not contested and abs(cost1 - cost) <= 1e-11 * max(len(x), 1):
                contested = float(np.linalg.norm(d))
            if not (cost1 < cost and (depth1 > 0).all()):
                break
            R, t, H, g, cost = R1, t1, H1, g1, cost1
    return R, t, changes, contested


def estimate(x, X, K, max_error=12.0, confidence=0.9999, max_iters=10000, seed=0):
    """Rules 1-6 for one set of pixels x [n, 2] and world points X [n, 3] under intrinsics K [3, 3].  Returns a dict: R [3, 3], t [3],
    ok, num_inliers, mask [n] (zero where not ok), the hypotheses run (`iters`), and the margins: count_margin = best count minus the
    runner-up over every model scored (inf with one model), hyp_margin = the smallest |max_error^2 - err^2| and |depth| over every
    scored model and point (inf without models), err2_margin [n] = max_error^2 - err^2 and depth [n] at the returned pose (NaN when
    not ok), gn_changes = the cost change of every Gauss-Newton trial, gn_step = the length of the first step whose keep-or-stop
    decision lies within rounding (0 if none)."""
    x, X, K = _arr(x, np.float64).reshape(-1, 2), _arr(X, np.float64).reshape(-1, 3), _arr(K, np.float64).reshape(3, 3)
    n = len(x)
    thr2 = float(max_error) ** 2
    out = dict(R=np.zeros((3, 3)), t=np.zeros(3), ok=False, num_inliers=0, mask=np.zeros(n, bool), iters=0, count_margin=math.inf,
               hyp_margin=math.inf, err2_margin=np.full(n, np.nan), depth=np.full(n, np.nan), gn_changes=[], gn_step=0.0)
    if n < 3:
        return out
    f = bearings(x, K)
    best, best_model, counts = 0, None, []
    it, niters = 0, int(max_iters)
    while it < niters and (n > 3 or it == 0):            # an item of exactly 3 points draws hypothesis 0 only
        ids = draw_distinct(3, n, seed, lambda s, h=it: (h, s, 0, CTR))
        for R, t in p3p(f[ids], X[ids]):
            err2, depth = reprojection(R, t, K, x, X)
            with np.errstate(invalid="ignore"):
                m = np.nan_to_num(np.abs(thr2 - err2), nan=np.inf)
            out["hyp_margin"] = min(out["hyp_margin"], float(m.min()), float(np.abs(depth).min()))
            cnt = int(((depth > 0) & (err2 <= thr2)).sum())
            counts.append(cnt)
            if cnt > max(best, 2):
                best, best_model = cnt, (R, t)
                niters = ransac_update_num_iters(confidence, (n - cnt) / n, niters, 3)
        it += 1
    out["iters"] = it
    if best_model is None:
        return out
    c = sorted(counts, reverse=True)
    out["count_margin"] = c[0] - c[1] if len(c) > 1 else math.inf
    R, t = best_model
    err2, depth = reprojection(R, t, K, x, X)
    used = (depth > 0) & (err2 <= thr2)
    R, t, out["gn_changes"], out["gn_step"] = refine(R, t, K, x[used], X[used])
    err2, depth = reprojection(R, t, K, x, X)
    mask = (depth > 0) & (err2 <= thr2)
    out.update(R=R, t=t, ok=True, num_inliers=int(mask.sum()), mask=mask, err2_margin=thr2 - err2, depth=depth)
    return out


def gather(kp_offsets, keypoints, track_offsets, elements, points_ok, points_X, images):
    """The correspondences of `register_images` for every image of `images`: the elements (i, a) of ok tracks k in element order,
    x = keypoints[kp_offsets[i] + a] widened to float64 and X = points_X[k].  Returns a list of (x [n, 2], X [n, 3]).
    ValueError for an element id outside its image's keypoints."""
    kp = _arr(kp_offsets, np.int64)
    xy = _arr(keypoints, np.float32).reshape(-1, 2).astype(np.float64)
    off = _arr(track_offsets, np.int64)
    el = _arr(elements, np.int64).reshape(-1, 2)
    ok, P = _arr(points_ok, bool), _arr(points_X, np.float64).reshape(-1, 3)
    N = kp.size - 1
    img, ids = el[:, 0], el[:, 1]
    if ((img < 0) | (img >= N)).any() or ((ids < 0) | (ids >= kp[np.clip(img, 0, N - 1) + 1] - kp[np.clip(img, 0, N - 1)])).any():
        raise ValueError("register_images: a track element lies outside its image's keypoints")
    track = np.repeat(np.arange(off.size - 1), np.diff(off))
    use = ok[track]
    out = []
    for i in images:
        e = np.flatnonzero(use & (img == int(i)))
        out.append((xy[kp[img[e]] + ids[e]], P[track[e]]))
    return out
