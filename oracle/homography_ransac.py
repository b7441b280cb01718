"""numpy / Python float64 restatement of `roma_b200.find_homography` (roma_b200/csrc/homography.cu), for the tests only.

Steps, as in include/romab200.h:
  1. the points are rounded to float32;
  2. hypothesis h of pair b, attempt a: 4 distinct indices from Philox4x32-10, key (seed lo, seed hi), counter (h, b, a, s),
     words in order, index (w * n) >> 32, repeats skipped; OpenCV's checkSubset (haveCollinearPoints on either image with float
     differences and a double test, then the orientation signs over the triples 012, 123, 023, 130); after 10 000 rejected
     attempts the hypothesis is "not found";
  3. the minimal solver: OpenCV's normalisation, the null vector of the 8x9 system by Gauss-Jordan with partial pivoting (first
     largest |pivot|; no model on a pivot that is not finite or below 1e-12 of the first), de-normalised, times 1 / H[2][2].  Every
     operation is a Python float operation, i.e. rounded separately, as on the device;
  4. OpenCV's computeError in float32, <= float32(thresh^2);
  5. OpenCV's sequential loop: count > max(best, 3) replaces the best model, niters = RANSACUpdateNumIters(conf, (n - count) / n,
     4, niters) with (1 - ep)^4 as products from the left; a "not found" hypothesis ends the loop;
  6. the refinement: the normalised DLT on the inliers (smallest eigenvector of L^T L) and at most 10 Levenberg-Marquardt steps
     with the damping rule of `lm_refine`, on OpenCV's HomographyRefineCallback residual;
  7. the returned mask: the inliers of the refined model by the test of step 4, as cv2 4.13 returns it (n == 4: all ones).

`stream="opencv"` replaces step 2 by OpenCV's own sampling (cv::RNG seeded with (uint64)-1, getSubset's redraw on a repeated
index and full redraw on a failed checkSubset) and step 3 by OpenCV's eigenvector solver, so that the loop can be pinned against
cv2.findHomography itself.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.ransac import draw_distinct, ransac_update_num_iters

FLT_EPS = float(np.finfo(np.float32).eps)
DBL_EPS = float(np.finfo(np.float64).eps)
MAX_ATTEMPTS = 10000
RANSAC = 8


# ---- subsets -------------------------------------------------------------------------------------------------------------
def _collinear_last(p):
    """haveCollinearPoints(p, 4): p float32 [4, 2]; differences in float32, the test in double."""
    for j in range(3):
        dx1, dy1 = float(p[j, 0] - p[3, 0]), float(p[j, 1] - p[3, 1])
        for k in range(j):
            dx2, dy2 = float(p[k, 0] - p[3, 0]), float(p[k, 1] - p[3, 1])
            if abs(dx2 * dy1 - dy2 * dx1) <= FLT_EPS * (((abs(dx1) + abs(dy1)) + abs(dx2)) + abs(dy2)):
                return True
    return False


def _det3(a, b, c):
    x0, y0, x1, y1, x2, y2 = float(a[0]), float(a[1]), float(b[0]), float(b[1]), float(c[0]), float(c[1])
    return (x0 * (y1 * 1.0 - y2 * 1.0) - y0 * (x1 * 1.0 - x2 * 1.0)) + 1.0 * (x1 * y2 - x2 * y1)


def check_subset(s4, d4):
    """OpenCV's HomographyEstimatorCallback::checkSubset of 4 correspondences (float32 [4, 2] each)."""
    if _collinear_last(s4) or _collinear_last(d4):
        return False
    neg = 0
    for i, j, k in ((0, 1, 2), (1, 2, 3), (0, 2, 3), (1, 3, 0)):
        neg += _det3(s4[i], s4[j], s4[k]) * _det3(d4[i], d4[j], d4[k]) < 0
    return neg in (0, 4)


def draw_subset(h, b, n, seed, src, dst):
    """Hypothesis h of pair b (n > 4): returns (indices, rejected attempts, found)."""
    for att in range(MAX_ATTEMPTS):
        idx = draw_distinct(4, n, seed, lambda sub: (h, b, att, sub))
        if check_subset(src[idx], dst[idx]):
            return idx, att, True
    return idx, MAX_ATTEMPTS, False


class CvRNG:
    """cv::RNG: multiply-with-carry, state (uint64)-1 by default; uniform(0, n) = next() % n."""

    def __init__(self, state=(1 << 64) - 1):
        self.state = state

    def next(self):
        self.state = ((self.state & 0xFFFFFFFF) * 4164903690 + (self.state >> 32)) & ((1 << 64) - 1)
        return self.state & 0xFFFFFFFF

    def uniform(self, a, b):
        return a if a == b else self.next() % (b - a) + a


def cv_subset(rng, src, dst):
    """OpenCV's getSubset (checkPartialSubsets off): redraw an index that repeats an earlier one; redraw all 4 when checkSubset
    fails, at most 10 000 times.  Returns (indices, found)."""
    n = len(src)
    for _ in range(MAX_ATTEMPTS):
        idx = []
        for _i in range(4):
            v = rng.uniform(0, n)
            while v in idx:
                v = rng.uniform(0, n)
            idx.append(v)
        if check_subset(src[idx], dst[idx]):
            return idx, True
    return idx, False


# ---- solvers -------------------------------------------------------------------------------------------------------------
def _normalisation(src, dst):
    """OpenCV's: centroids and scale = count / sum |x - c| per axis (sequential sums); None when a sum is below DBL_EPSILON."""
    count = len(src)
    cm = [0.0, 0.0]
    cM = [0.0, 0.0]
    for i in range(count):
        cm[0] += float(dst[i, 0]); cm[1] += float(dst[i, 1])
        cM[0] += float(src[i, 0]); cM[1] += float(src[i, 1])
    cm = [c / count for c in cm]
    cM = [c / count for c in cM]
    sm = [0.0, 0.0]
    sM = [0.0, 0.0]
    for i in range(count):
        sm[0] += abs(float(dst[i, 0]) - cm[0]); sm[1] += abs(float(dst[i, 1]) - cm[1])
        sM[0] += abs(float(src[i, 0]) - cM[0]); sM[1] += abs(float(src[i, 1]) - cM[1])
    if not all(abs(s) >= DBL_EPS for s in sm + sM):
        return None
    return cm, [count / s for s in sm], cM, [count / s for s in sM]


def _denormalise(h0, cm, sm, cM, sM):
    inv = [1.0 / sm[0], 0.0, cm[0], 0.0, 1.0 / sm[1], cm[1], 0.0, 0.0, 1.0]
    nrm = [sM[0], 0.0, -(cM[0] * sM[0]), 0.0, sM[1], -(cM[1] * sM[1]), 0.0, 0.0, 1.0]
    t = [(inv[3 * i] * h0[j] + inv[3 * i + 1] * h0[3 + j]) + inv[3 * i + 2] * h0[6 + j] for i in range(3) for j in range(3)]
    H = [(t[3 * i] * nrm[j] + t[3 * i + 1] * nrm[3 + j]) + t[3 * i + 2] * nrm[6 + j] for i in range(3) for j in range(3)]
    s = 1.0 / H[8]
    return np.array([v * s for v in H]).reshape(3, 3)


def solve_four(s4, d4):
    """The device's minimal solver (Gauss-Jordan on the normalised 8x9 system).  Returns H [3, 3] or None."""
    nz = _normalisation(s4, d4)
    if nz is None:
        return None
    cm, sm, cM, sM = nz
    a = []
    for i in range(4):
        x, y = (float(d4[i, 0]) - cm[0]) * sm[0], (float(d4[i, 1]) - cm[1]) * sm[1]
        X, Y = (float(s4[i, 0]) - cM[0]) * sM[0], (float(s4[i, 1]) - cM[1]) * sM[1]
        a.append([X, Y, 1.0, 0.0, 0.0, 0.0, -(x * X), -(x * Y), -x])
        a.append([0.0, 0.0, 0.0, X, Y, 1.0, -(y * X), -(y * Y), -y])
    p0 = 0.0
    for k in range(8):
        piv, best = k, -1.0
        for r in range(k, 8):
            if abs(a[r][k]) > best:
                best, piv = abs(a[r][k]), r
        a[k], a[piv] = a[piv], a[k]
        p = a[k][k]
        if k == 0:
            p0 = abs(p)
        if not (abs(p) > 1e-12 * p0) or not math.isfinite(p):
            return None
        a[k] = [a[k][c] / p if c >= k else a[k][c] for c in range(9)]
        for r in range(8):
            if r != k:
                f = a[r][k]
                a[r] = [a[r][c] - f * a[k][c] if c >= k else a[r][c] for c in range(9)]
    H = _denormalise([-a[r][8] for r in range(8)] + [1.0], cm, sm, cM, sM)
    return H if np.all(np.isfinite(H)) else None


def dlt(src, dst):
    """OpenCV's runKernel: the normalised DLT over all given points, the smallest eigenvector of the 9x9 L^T L.  Returns H or None."""
    src = np.asarray(src, dtype=np.float32)
    dst = np.asarray(dst, dtype=np.float32)
    n = len(src)
    cm = dst.astype(np.float64).sum(axis=0) / n
    cM = src.astype(np.float64).sum(axis=0) / n
    s_m = np.abs(dst - cm).sum(axis=0)
    s_M = np.abs(src - cM).sum(axis=0)
    if not (np.all(np.abs(s_m) >= DBL_EPS) and np.all(np.abs(s_M) >= DBL_EPS)):
        return None
    sm, sM = n / s_m, n / s_M
    x, y = ((dst - cm) * sm).T
    X, Y = ((src - cM) * sM).T
    o, z = np.ones(n), np.zeros(n)
    Lx = np.stack([X, Y, o, z, z, z, -x * X, -x * Y, -x], axis=1)
    Ly = np.stack([z, z, z, X, Y, o, -y * X, -y * Y, -y], axis=1)
    LtL = Lx.T @ Lx + Ly.T @ Ly
    if not np.all(np.isfinite(LtL)):
        return None
    _w, V = np.linalg.eigh(LtL)
    H = _denormalise(list(V[:, 0]), list(cm), list(sm), list(cM), list(sM))
    return H if np.all(np.isfinite(H)) else None


# ---- scoring and selection -----------------------------------------------------------------------------------------------
def inlier_mask(H, src, dst, thresh):
    """OpenCV's computeError in float32 (every operation rounded) <= float32(thresh^2); bool [N]."""
    f = np.asarray(H, dtype=np.float64).ravel()[:8].astype(np.float32)
    x, y = src[:, 0], src[:, 1]
    one = np.float32(1.0)
    with np.errstate(all="ignore"):
        ww = one / ((f[6] * x + f[7] * y) + one)
        ex = ((f[0] * x + f[1] * y) + f[2]) * ww - dst[:, 0]
        ey = ((f[3] * x + f[4] * y) + f[5]) * ww - dst[:, 1]
        err = ex * ex + ey * ey
    return err <= np.float32(thresh * thresh)


def select(hypothesis, n, conf, max_iters):
    """OpenCV's loop: hypothesis(h) -> (status, count) with status 1 (model), 0 (no model) or -1 (not found).
    Returns (best hypothesis, best count, final niters, iterations run, ended on a not-found hypothesis)."""
    best, hyp, niters, it, nf = 0, -1, max_iters, 0, False
    while it < niters:
        status, c = hypothesis(it)
        if status < 0:
            nf = True
            break
        if status == 1 and c > max(best, 3):
            best, hyp = c, it
            niters = ransac_update_num_iters(conf, (n - c) / n, niters, 4)
        it += 1
    return hyp, best, niters, it, nf


# ---- refinement ----------------------------------------------------------------------------------------------------------
def _residual(x, src, dst, jac=True):
    """HomographyRefineCallback: r [2N] (x, y interleaved) and J [2N, 8] at the 8 parameters x (H[2][2] = 1)."""
    Mx, My = src[:, 0].astype(np.float64), src[:, 1].astype(np.float64)
    w = x[6] * Mx + x[7] * My + 1.0
    with np.errstate(all="ignore"):
        ww = np.where(np.abs(w) > DBL_EPS, 1.0 / w, 0.0)
    xi = (x[0] * Mx + x[1] * My + x[2]) * ww
    yi = (x[3] * Mx + x[4] * My + x[5]) * ww
    r = np.stack([xi - dst[:, 0], yi - dst[:, 1]], axis=1).ravel()
    if not jac:
        return r, None
    n = len(src)
    J = np.zeros((n, 2, 8))
    J[:, 0, 0], J[:, 0, 1], J[:, 0, 2] = Mx * ww, My * ww, ww
    J[:, 0, 6], J[:, 0, 7] = -Mx * ww * xi, -My * ww * xi
    J[:, 1, 3], J[:, 1, 4], J[:, 1, 5] = Mx * ww, My * ww, ww
    J[:, 1, 6], J[:, 1, 7] = -Mx * ww * yi, -My * ww * yi
    return r, J.reshape(2 * n, 8)


def lm_refine(H, src, dst, max_iters=10):
    """Levenberg-Marquardt on the 8 parameters of H (H[2][2] kept), the device's damping rule (OpenCV's LMSolver):
    d = (A + lambda diag(D))^-1 J^T r with A = J^T J and D = diag(A) at the start; the step is taken iff it lowers |r|^2; the gain
    ratio R = (S - Sd) / d.(2 J^T r - A d) halves lambda above 0.75 (to 0 below lc = 0.75) and multiplies it by
    nu = clip((Sd - S) / d.J^T r + 2, 2, 10) below 0.25 (from 0: lambda = lc = 1 / max |diag(inv(A))|, nu halved); stops after
    max_iters steps or when |d|_inf or |r|_inf (at the current parameters) falls below FLT_EPSILON."""
    x = np.asarray(H, dtype=np.float64).ravel()[:8].copy()
    h22 = float(np.asarray(H).ravel()[8])
    r, J = _residual(x, src, dst)
    S = float(r @ r)
    A, v = J.T @ J, J.T @ r
    D = np.diag(A).copy()
    lam, lc = 1.0, 0.75
    for _ in range(max_iters):
        try:
            d = np.linalg.solve(A + lam * np.diag(D), v)
        except np.linalg.LinAlgError:
            break
        xd = x - d
        rd, Jd = _residual(xd, src, dst)
        Sd = float(rd @ rd)
        dS = float(d @ (2.0 * v - A @ d))
        R = (S - Sd) / (dS if abs(dS) > DBL_EPS else 1.0)
        if R > 0.75:
            lam *= 0.5
            if lam < lc:
                lam = 0.0
        elif R < 0.25:
            t = float(d @ v)
            nu = (Sd - S) / (t if abs(t) > DBL_EPS else 1.0) + 2.0
            nu = min(max(nu, 2.0), 10.0)
            if lam == 0.0:
                maxval = DBL_EPS
                try:
                    maxval = max(maxval, float(np.abs(np.diag(np.linalg.inv(A))).max()))
                except np.linalg.LinAlgError:
                    pass
                lam = lc = 1.0 / maxval
                nu *= 0.5
            lam *= nu
        if Sd < S:
            S, x, r = Sd, xd, rd
            A, v = Jd.T @ Jd, Jd.T @ rd
        if not (np.abs(d).max() >= FLT_EPS and np.abs(r).max() >= FLT_EPS):
            break
    return np.r_[x, h22].reshape(3, 3)


def refine(H, src, dst):
    """findHomography after RANSAC (or for method 0): DLT on the given points (kept H when it is degenerate), then LM when
    there are more than 4 points."""
    Hd = dlt(src, dst)
    H = H if Hd is None else Hd
    return lm_refine(H, src, dst) if len(src) > 4 else H


# ---- the whole estimate --------------------------------------------------------------------------------------------------
def find_homography(src, dst, method=RANSAC, thresh=3.0, conf=0.995, max_iters=2000, seed=0, b=0, stream="philox", details=None):
    """The device estimator restated (stream="philox") or OpenCV's loop (stream="opencv").  Returns (H or None, mask bool [N]).
    `details` (a dict) receives the best hypothesis, count, final niters, iterations run, the best model and its inlier mask."""
    src = np.asarray(src, dtype=np.float32).reshape(-1, 2)
    dst = np.asarray(dst, dtype=np.float32).reshape(-1, 2)
    n = len(src)
    if n < 4:
        raise ValueError("fewer than 4 points")
    zeros = np.zeros(n, bool)
    thresh = 3.0 if thresh <= 0 else thresh
    if method == 0:
        H = dlt(src, dst)
        if H is None:
            return None, zeros
        if n == 4:
            return H, np.ones(n, bool)
        H = lm_refine(H, src, dst)
        return H, inlier_mask(H, src, dst, thresh)
    max_iters = max(int(max_iters), 1)
    if n == 4:
        H = solve_four(src, dst) if stream == "philox" else dlt(src, dst)
        return (None, zeros) if H is None else (H, np.ones(n, bool))
    models = {}
    rng = CvRNG() if stream == "opencv" else None

    def hypothesis(h):
        if stream == "philox":
            idx, _att, found = draw_subset(h, b, n, seed, src, dst)
        else:
            idx, found = cv_subset(rng, src, dst)
        if not found:
            return -1, 0
        H = solve_four(src[idx], dst[idx]) if stream == "philox" else dlt(src[idx], dst[idx])
        if H is None:
            return 0, 0
        models[h] = H
        return 1, int(inlier_mask(H, src, dst, thresh).sum())

    hyp, best, niters, it, nf = select(hypothesis, n, conf, max_iters)
    if details is not None:
        details.update(hyp=hyp, best=best, niters=niters, iters=it, not_found=nf)
    if hyp < 0:
        return None, zeros
    Hb = models[hyp]
    mask = inlier_mask(Hb, src, dst, thresh)
    if details is not None:
        details.update(H_best=Hb, ransac_mask=mask)
    H = refine(Hb, src[mask], dst[mask])
    return H, inlier_mask(H, src, dst, thresh)           # OpenCV 4.13 returns the inliers of the refined model


def corners(H, w, h):
    """The four image corners (0, 0), (0, h - 1), (w - 1, 0), (w - 1, h - 1) mapped by H."""
    c = np.array([[0, 0, 1], [0, h - 1, 1], [w - 1, 0, 1], [w - 1, h - 1, 1]], dtype=np.float64) @ np.asarray(H, dtype=np.float64).T
    return c[:, :2] / c[:, 2:]
