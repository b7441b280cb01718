"""numpy float64 restatement of `roma_b200.estimate_pose` (roma_b200/csrc/pose.cu), for the tests only.

Steps, as in include/romab200.h:
  1. xn = inv(K[:2,:2]) (x - K[:2,2]) with the closed-form 2x2 inverse, every operation rounded separately;
  2. hypothesis h of pair b: 5 distinct indices from Philox4x32-10, key (seed lo, seed hi), counter (h, b, s, 0), words in order,
     index (w * n) >> 32, repeats skipped; Nister's five-point solver (null space of the 5x9 system by Gauss-Jordan with
     partial pivoting, orthonormalised by modified Gram-Schmidt; 10x20 constraint matrix, Gauss-Jordan, degree-10 polynomial in z) with `np.roots` for the real roots;
     each E at unit Frobenius norm with its first largest-magnitude entry positive;
  3. OpenCV's E error (Sampson) in float64 without contraction, rounded to float32, <= float32(thresh^2);
  4. OpenCV's sequential RANSAC replay with RANSACUpdateNumIters;
  5. cv::recoverPose (SVD decomposition, DLT triangulation, chirality and distance tests).
"""
from __future__ import annotations

import math

import numpy as np

from oracle.ransac import draw_distinct, philox4x32_10, ransac_update_num_iters  # noqa: F401  (philox4x32_10 stays importable here)


def draw_sample(h, b, n, seed):
    """The 5 distinct indices of hypothesis h of pair b (n > 5 points)."""
    return draw_distinct(5, n, seed, lambda sub: (h, b, sub, 0))


def normalise(x, K):
    x = np.asarray(x, dtype=np.float64)
    det = K[0, 0] * K[1, 1] - K[0, 1] * K[1, 0]
    i00, i01, i10, i11 = K[1, 1] / det, -K[0, 1] / det, -K[1, 0] / det, K[0, 0] / det
    dx, dy = x[:, 0] - K[0, 2], x[:, 1] - K[1, 2]
    return np.stack([i00 * dx + i01 * dy, i10 * dx + i11 * dy], axis=1)


# ---- five-point solver --------------------------------------------------------------------------------------------------
def _mono2(u, v):
    return (0, 4, 7, 9)[u] + (v - u)


_MONO3 = {(3, 0, 0): 0, (0, 3, 0): 1, (2, 1, 0): 2, (1, 2, 0): 3, (2, 0, 1): 4, (2, 0, 0): 5, (0, 2, 1): 6, (0, 2, 0): 7, (1, 1, 1): 8,
          (1, 1, 0): 9, (1, 0, 2): 10, (1, 0, 1): 11, (1, 0, 0): 12, (0, 1, 2): 13, (0, 1, 1): 14, (0, 1, 0): 15, (0, 0, 3): 16,
          (0, 0, 2): 17, (0, 0, 1): 18, (0, 0, 0): 19}


def _mono3(*vs):
    return _MONO3[tuple(sum(v == k for v in vs) for k in range(3))]


def _mul11(a, b):
    out = np.zeros(a.shape[:-1] + (10,))
    for u in range(4):
        for v in range(4):
            out[..., _mono2(min(u, v), max(u, v))] += a[..., u] * b[..., v]
    return out


def _mul21(p, b):
    out = np.zeros(p.shape[:-1] + (20,))
    for u in range(4):
        for v in range(u, 4):
            for w in range(4):
                out[..., _mono3(u, v, w)] += p[..., _mono2(u, v)] * b[..., w]
    return out


def _gauss_jordan(M):
    """In place on M [H, R, C]: reduce the first R columns to the identity with partial pivoting; returns the ok mask [H]
    (False on a non-finite pivot or one below 1e-12 of the first)."""
    H, R, _ = M.shape
    ok = np.ones(H, bool)
    ar = np.arange(H)
    p0 = None
    for k in range(R):
        piv = k + np.argmax(np.abs(M[:, k:, k]), axis=1)
        rows = M[ar, piv].copy()
        M[ar, piv] = M[:, k]
        M[:, k] = rows
        p = M[:, k, k].copy()
        p0 = np.abs(p) if p0 is None else p0
        ok &= (np.abs(p) > 1e-12 * p0) & np.isfinite(p)
        p = np.where(ok, p, 1.0)
        M[:, k] = M[:, k] / p[:, None]
        for r in range(R):
            if r != k:
                M[:, r] = M[:, r] - M[:, r, k:k + 1] * M[:, k]
    return ok


def solve_five_point(pts):
    """pts [H, 5, 4] normalised (x0, y0, x1, y1).  Returns a list of H arrays [m, 9] (row-major E, ascending z)."""
    pts = np.asarray(pts, dtype=np.float64)
    H = pts.shape[0]
    x0, y0, x1, y1 = (pts[..., i] for i in range(4))
    one = np.ones_like(x0)
    Q = np.stack([x1 * x0, x1 * y0, x1, y1 * x0, y1 * y0, y1, x0, y0, one], axis=-1)
    ok = _gauss_jordan(Q)
    basis = np.zeros((H, 4, 9))
    for c in range(5, 9):
        basis[:, c - 5, :5] = -Q[:, :, c]
        basis[:, c - 5, c] = 1.0
    for i in range(4):                                   # modified Gram-Schmidt: an orthonormal basis conditions the solver
        for j in range(i):
            basis[:, i] -= np.sum(basis[:, i] * basis[:, j], axis=1, keepdims=True) * basis[:, j]
        basis[:, i] /= np.sqrt(np.sum(basis[:, i] * basis[:, i], axis=1, keepdims=True))
    e = np.transpose(basis, (0, 2, 1))                   # [H, 9 entries, 4 coefficients (x, y, z, 1)]
    M = np.zeros((H, 10, 20))
    cof = [(0, 4, 8, 5, 7, 1.0), (1, 3, 8, 5, 6, -1.0), (2, 3, 7, 4, 6, 1.0)]
    for j0, a1, b1, a2, b2, s in cof:
        m2 = _mul11(e[:, a1], e[:, b1]) - _mul11(e[:, a2], e[:, b2])
        M[:, 0] += s * _mul21(m2, e[:, j0])
    tr = sum(_mul11(e[:, k], e[:, k]) for k in range(9))
    for i in range(3):
        for j in range(3):
            row = -_mul21(tr, e[:, 3 * i + j])
            for k in range(3):
                A = sum(_mul11(e[:, 3 * i + l], e[:, 3 * k + l]) for l in range(3))
                row = row + 2.0 * _mul21(A, e[:, 3 * k + j])
            M[:, 1 + 3 * i + j] = row
    ok &= _gauss_jordan(M)
    out = []
    for h in range(H):
        if not ok[h]:
            out.append(np.zeros((0, 9)))
            continue
        Bm = M[h]
        px, py, p1 = np.zeros((3, 4)), np.zeros((3, 4)), np.zeros((3, 5))
        for k in range(3):
            ra, rb = 4 + 2 * k, 5 + 2 * k
            for p in range(3):
                px[k, 2 - p] -= Bm[ra, 10 + p]; px[k, 3 - p] += Bm[rb, 10 + p]
                py[k, 2 - p] -= Bm[ra, 13 + p]; py[k, 3 - p] += Bm[rb, 13 + p]
            for p in range(4):
                p1[k, 3 - p] -= Bm[ra, 16 + p]; p1[k, 4 - p] += Bm[rb, 16 + p]
        pm = np.polynomial.polynomial
        poly = (pm.polymul(px[0], pm.polysub(pm.polymul(py[1], p1[2]), pm.polymul(p1[1], py[2])))
                - pm.polymul(py[0], pm.polysub(pm.polymul(px[1], p1[2]), pm.polymul(p1[1], px[2])))
                + np.pad(pm.polymul(p1[0], pm.polysub(pm.polymul(px[1], py[2]), pm.polymul(py[1], px[2]))), (0, 0)))
        poly = np.pad(poly, (0, max(0, 11 - len(poly))))[:11]
        if not np.any(poly[1:] != 0) or not np.all(np.isfinite(poly)):
            out.append(np.zeros((0, 9)))
            continue
        roots = np.roots(poly[::-1])
        zs = np.sort(roots[roots.imag == 0].real)
        dpoly = pm.polyder(poly)
        sols = []
        for z in zs:
            for _ in range(2):                                    # Newton polish, as the device does
                d = pm.polyval(z, dpoly)
                zn = z - pm.polyval(z, poly) / d
                if np.isfinite(zn):
                    z = zn
            Bz = np.array([[pm.polyval(z, px[k]), pm.polyval(z, py[k]), pm.polyval(z, p1[k])] for k in range(3)])
            best = None
            for r0, r1 in ((0, 1), (0, 2), (1, 2)):
                v = np.cross(Bz[r0], Bz[r1])
                if best is None or abs(v[2]) > abs(best[2]):
                    best = v
            x, y = best[0] / best[2], best[1] / best[2]
            E = x * basis[h, 0] + y * basis[h, 1] + z * basis[h, 2] + basis[h, 3]
            nrm = math.sqrt(float(np.sum(E * E)))
            if not (nrm > 0 and math.isfinite(nrm)):
                continue
            E = E / nrm
            E = -E if E[np.argmax(np.abs(E))] < 0 else E
            if np.all(np.isfinite(E)):
                sols.append(E)
        out.append(np.array(sols).reshape(-1, 9))
    return out


# ---- scoring and selection ---------------------------------------------------------------------------------------------
def inlier_mask(E, xn, thresh):
    """OpenCV's E error of every point under E (9 or [M, 9]) with the device's operation order; returns bool [M, N]."""
    E = np.atleast_2d(np.asarray(E, dtype=np.float64))
    e = [E[:, i:i + 1] for i in range(9)]
    x0, y0, x1, y1 = (xn[None, :, i] for i in range(4))
    ex0 = e[0] * x0 + e[1] * y0 + e[2]
    ex1 = e[3] * x0 + e[4] * y0 + e[5]
    ex2 = e[6] * x0 + e[7] * y0 + e[8]
    et0 = e[0] * x1 + e[3] * y1 + e[6]
    et1 = e[1] * x1 + e[4] * y1 + e[7]
    v = x1 * ex0 + y1 * ex1 + ex2
    den = ex0 * ex0 + ex1 * ex1 + et0 * et0 + et1 * et1
    with np.errstate(all="ignore"):
        err = ((v * v) / den).astype(np.float32)
    return err <= np.float32(thresh * thresh)


def select(counts_of, n, conf, max_iters):
    """OpenCV's loop over hypotheses: counts_of(h) -> list of inlier counts of hypothesis h's solutions.
    Returns (best hypothesis, best solution, best count, final niters, iterations run)."""
    best, hyp, sol, niters, it = 0, -1, -1, max_iters, 0
    while it < niters:
        for s, c in enumerate(counts_of(it)):
            if c > max(best, 4):
                best, hyp, sol = c, it, s
                niters = ransac_update_num_iters(conf, (n - c) / n, niters, 5)
        it += 1
    return hyp, sol, best, niters, it


# ---- recoverPose ---------------------------------------------------------------------------------------------------------
def decompose_essential(E):
    U, _, Vt = np.linalg.svd(np.asarray(E, dtype=np.float64).reshape(3, 3))
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, 1, 0], [-1, 0, 0], [0, 0, 1]])
    return U @ W @ Vt, U @ W.T @ Vt, U[:, 2].copy()


def recover_pose(E, xn, mask=None, dist=1e9):
    """cv2.recoverPose(E, xn[:, :2], xn[:, 2:], I, dist, mask): returns (count, R, t [3, 1], mask bool [N])."""
    R1, R2, t = decompose_essential(E)
    n = xn.shape[0]
    x0, y0, x1, y1 = (xn[:, i] for i in range(4))
    inm = np.ones(n, bool) if mask is None else np.asarray(mask).ravel() > 0
    goods = []
    for R, tt in ((R1, t), (R2, t), (R1, -t), (R2, -t)):
        P1 = np.c_[R, tt]
        A = np.zeros((n, 4, 4))
        A[:, 0] = x0[:, None] * np.array([0, 0, 1.0, 0]) - np.array([1.0, 0, 0, 0])
        A[:, 1] = y0[:, None] * np.array([0, 0, 1.0, 0]) - np.array([0, 1.0, 0, 0])
        A[:, 2] = x1[:, None] * P1[2] - P1[0]
        A[:, 3] = y1[:, None] * P1[2] - P1[1]
        ok = np.isfinite(A).all(axis=(1, 2))
        A[~ok] = 0
        Q = np.linalg.svd(A)[2][:, -1, :]
        with np.errstate(all="ignore"):
            m = Q[:, 2] * Q[:, 3] > 0
            Qn = Q / Q[:, 3:4]
            m &= Qn[:, 2] < dist
            z2 = Qn @ P1[2]
            m &= (z2 > 0) & (z2 < dist)
        goods.append(m & inm & ok)
    g = [int(m.sum()) for m in goods]
    if g[0] >= g[1] and g[0] >= g[2] and g[0] >= g[3]:
        c = 0
    elif g[1] >= g[0] and g[1] >= g[2] and g[1] >= g[3]:
        c = 1
    elif g[2] >= g[0] and g[2] >= g[1] and g[2] >= g[3]:
        c = 2
    else:
        c = 3
    R = (R1, R2, R1, R2)[c]
    tt = (t, t, -t, -t)[c]
    return g[c], R, tt.reshape(3, 1), goods[c]


# ---- the whole estimate --------------------------------------------------------------------------------------------------
def estimate_pose(kpts0, kpts1, K0, K1, norm_thresh, conf=0.99999, max_iters=1000, seed=0, b=0, details=None):
    """The device estimator restated; returns None or (R, t [3, 1], mask).  `details` (a dict) receives the best hypothesis,
    solution, count, final niters and the best E."""
    n = len(kpts0)
    if n < 5:
        return None
    K0, K1 = np.asarray(K0, dtype=np.float64), np.asarray(K1, dtype=np.float64)
    xn = np.concatenate([normalise(kpts0, K0), normalise(kpts1, K1)], axis=1)
    if n == 5:
        Es = solve_five_point(xn[None])[0]
        mask = np.ones(n, bool)
    else:
        cache = {}

        def counts_of(h):
            if h not in cache:                    # solve the next 128 hypotheses at once
                hs = list(range(h, min(h + 128, max_iters)))
                for g, E in zip(hs, solve_five_point(xn[np.array([draw_sample(g, b, n, seed) for g in hs])])):
                    cache[g] = (E, None)
            E, c = cache[h]
            if c is None:
                c = [int(v) for v in inlier_mask(E, xn, norm_thresh).sum(axis=1)] if len(E) else []
                cache[h] = (E, c)
            return c

        hyp, sol, best, niters, _ = select(counts_of, n, conf, max_iters)
        if details is not None:
            details.update(hyp=hyp, sol=sol, best=best, niters=niters)
        if hyp < 0:
            return None
        Es = cache[hyp][0][sol:sol + 1]
        mask = inlier_mask(Es[0], xn, norm_thresh)[0]
        if details is not None:
            details["E"] = Es[0]
    ret, best_n = None, 0
    for E in Es:                                  # the reference's loop: every call updates the mask in place
        cnt, R, t, mask = recover_pose(E, xn, mask)
        if cnt > best_n:
            best_n, ret = cnt, (R, t, mask.copy())
    return ret
