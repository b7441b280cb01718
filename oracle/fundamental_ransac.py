"""numpy / float64 restatement of `roma_b200.find_fundamental` (roma_b200/csrc/fundamental.cu), for the tests only.

Steps, as in include/romab200.h:
  1. normalisation of the pair: centroid and mean distance over the rows with four finite coordinates, summed in the device's
     fixed order (`cta_sum`), scale = sqrt(2) / mean distance;
  2. hypothesis h: 7 distinct indices from Philox4x32-10, key (seed lo, seed hi), counter (h, s, 0, RB_FUND_CTR); the
     seven-point solver (Gauss-Jordan on the normalised 7x9 system, the cubic's real roots by bracketing and bisection, the oriented
     epipolar constraint), de-normalised and scaled to unit Frobenius norm.  Every operation is a separately rounded float64
     operation, vectorised over hypotheses, so the models equal the device's bit for bit;
  3. per slice of SLICE points: the sequential sum of the MAGSAC++ losses (sigma_max = thr, table interpolation up to k^2 thr^2)
     and the count of points with squared Sampson distance below thr^2;
  4. the sequential loop: a model replaces the best iff its loss is lower, niters = RANSACUpdateNumIters(conf, (n - count) / n, 7,
     niters);
  5. sigma-consensus++: weighted normalised eight-point fits while the loss decreases (at most 10), numpy's eigh and svd in place
     of the device's Jacobi (agreement to about 1e-12); the mask is r2 < thresh^2 under the returned F.
"""
from __future__ import annotations

import numpy as np

from oracle.ransac import draw_distinct, ransac_update_num_iters

ROUND, MODELS, SLICE, TABLE, REFINE_ITERS = 1024, 3, 512, 1024, 10
CTR = 0x46370000
SQRT2 = 1.4142135623730951
K2 = 13.276704135987622         # the 0.99 quantile of chi^2 with 4 degrees of freedom


# ---- fixed-order sums ----------------------------------------------------------------------------------------------------
def cta_sum(vals, threads=256):
    """The device's `cta_sum` of per-row values vals [n, K] (zero rows for skipped points): thread t adds rows t, t + threads, ...
    in order, a butterfly within each warp, then the warp partials in warp order.  Returns [K]."""
    vals = np.asarray(vals, dtype=np.float64)
    n, K = vals.shape
    R = max(1, -(-n // threads))
    P = np.zeros((R * threads, K))
    P[:n] = vals
    part = np.add.accumulate(P.reshape(R, threads, K), axis=0)[-1]
    w = part.reshape(threads // 32, 32, K)
    lanes = np.arange(32)
    for d in (16, 8, 4, 2, 1):
        w = w + w[:, lanes ^ d]
    tot = np.zeros(K)
    for q in range(threads // 32):
        tot = tot + w[q, 0]
    return tot


def normalise(x0, x1):
    """Step 1: returns (nr = (cx0, cy0, s0, cx1, cy1, s1), xn [n, 4])."""
    X = np.c_[x0, x1].astype(np.float64)
    fin = np.isfinite(X).all(axis=1)
    Z = np.where(fin[:, None], X, 0.0)
    s = cta_sum(np.c_[Z, fin.astype(np.float64)])
    cnt = s[4]
    with np.errstate(all="ignore"):
        c = s[:4] / cnt
        D = Z - c
        d = np.c_[np.sqrt(D[:, 0] * D[:, 0] + D[:, 1] * D[:, 1]), np.sqrt(D[:, 2] * D[:, 2] + D[:, 3] * D[:, 3])]
        t = cta_sum(np.where(fin[:, None], d, 0.0))
        s0, s1 = SQRT2 / (t[0] / cnt), SQRT2 / (t[1] / cnt)
        xn = np.c_[(X[:, 0] - c[0]) * s0, (X[:, 1] - c[1]) * s0, (X[:, 2] - c[2]) * s1, (X[:, 3] - c[3]) * s1]
    return np.array([c[0], c[1], s0, c[2], c[3], s1]), xn


# ---- the seven-point solver, vectorised over hypotheses --------------------------------------------------------------------
def _cofactors(A):
    return [A[4] * A[8] - A[5] * A[7], A[5] * A[6] - A[3] * A[8], A[3] * A[7] - A[4] * A[6],
            A[2] * A[7] - A[1] * A[8], A[0] * A[8] - A[2] * A[6], A[1] * A[6] - A[0] * A[7],
            A[1] * A[5] - A[2] * A[4], A[2] * A[3] - A[0] * A[5], A[0] * A[4] - A[1] * A[3]]


def _dot9(B, c):
    s = B[0] * c[0]
    for i in range(1, 9):
        s = s + B[i] * c[i]
    return s


def _cubic(c, x):
    return ((c[3] * x + c[2]) * x + c[1]) * x + c[0]


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _norm2(c):
    return (c[0] * c[0] + c[1] * c[1]) + c[2] * c[2]


def oriented(F, p):
    """The oriented epipolar constraint: F [H, 9] (normalised), p [H, 7, 4].  Returns bool [H]."""
    f = [F[:, i] for i in range(9)]
    e = _cross([f[0], f[3], f[6]], [f[2], f[5], f[8]])
    ne = _norm2(e)
    for a, b in (([f[1], f[4], f[7]], [f[2], f[5], f[8]]), ([f[0], f[3], f[6]], [f[1], f[4], f[7]])):
        t = _cross(a, b)
        nt = _norm2(t)
        take = nt > ne
        e = [np.where(take, t[i], e[i]) for i in range(3)]
        ne = np.where(take, nt, ne)
    pos = np.zeros(len(F), int)
    neg = np.zeros(len(F), int)
    for i in range(7):
        x, y, u, v = (p[:, i, j] for j in range(4))
        f0 = (f[0] * x + f[1] * y) + f[2]
        f1 = (f[3] * x + f[4] * y) + f[5]
        f2 = (f[6] * x + f[7] * y) + f[8]
        l0, l1, l2 = e[1] - e[2] * v, e[2] * u - e[0], e[0] * v - e[1] * u
        s = (l0 * f0 + l1 * f1) + l2 * f2
        pos += s > 0
        neg += s < 0
    return (pos == 7) | (neg == 7)


def seven_point(p, orient=True):
    """The device's seven-point solver on normalised points p [H, 7, 4] = (x, y, x', y').  Returns (nmod [H], F [H, 3, 9]): the
    models of each hypothesis in ascending root order (those that pass `oriented` when orient is set), row-major, x'^T F x = 0."""
    p = np.asarray(p, dtype=np.float64)
    H = len(p)
    x, y, u, v = (p[:, :, j] for j in range(4))
    a = np.stack([u * x, u * y, u, v * x, v * y, v, x, y, np.ones_like(x)], axis=2)
    ok = np.ones(H, bool)
    p0 = np.zeros(H)
    ar = np.arange(H)
    with np.errstate(all="ignore"):
        for k in range(7):
            col = np.abs(a[:, k:, k])
            piv = k + np.argmax(np.where(np.isnan(col), -1.0, col), axis=1)
            rk = a[ar, piv].copy()
            a[ar, piv] = a[:, k]
            a[:, k] = rk
            pk = a[:, k, k].copy()
            if k == 0:
                p0 = np.abs(pk)
            ok &= (np.abs(pk) > 1e-12 * p0) & np.isfinite(pk)
            a[:, k, k:] = a[:, k, k:] / pk[:, None]
            others = np.arange(7) != k
            a[:, others, k:] = a[:, others, k:] - a[:, others, k][:, :, None] * a[:, k, None, k:]
        F2 = [-a[:, i, 8] for i in range(7)] + [np.zeros(H), np.ones(H)]
        D = [-a[:, i, 7] - F2[i] for i in range(7)] + [np.ones(H), -np.ones(H)]
        cf = _cofactors(F2)
        c0 = (F2[0] * cf[0] + F2[1] * cf[1]) + F2[2] * cf[2]
        c1 = _dot9(D, cf)
        cf = _cofactors(D)
        c3 = (D[0] * cf[0] + D[1] * cf[1]) + D[2] * cf[2]
        c2 = _dot9(F2, cf)
        c = (c0, c1, c2, c3)
        B = 1.0 + np.fmax(np.fmax(np.abs(c2), np.abs(c1)), np.abs(c0)) / np.abs(c3)
        ok &= np.isfinite(B)
        c33 = 3.0 * c3
        disc = c2 * c2 - c33 * c1
        has = disc > 0
        q = np.sqrt(np.where(has, disc, 0.0))
        t0, t1 = (-c2 - q) / c33, (-c2 + q) / c33
        lo_c = np.fmin(np.fmax(np.fmin(t0, t1), -B), B)
        hi_c = np.fmin(np.fmax(np.fmax(t0, t1), -B), B)
        edge = [-B, np.where(has, lo_c, B), np.where(has, hi_c, B), B]
        ne = np.where(has, 4, 2)
        nm = np.zeros(H, int)
        out = np.zeros((H, MODELS, 9))
        for k in range(3):
            na, nb = _cubic(c, edge[k]) < 0, _cubic(c, edge[k + 1]) < 0
            act = ok & (k + 1 < ne) & (na != nb)
            lo, hi, live = edge[k].copy(), edge[k + 1].copy(), act.copy()
            for _ in range(128):
                mid = (lo + hi) * 0.5
                live = live & (mid > lo) & (mid < hi)
                if not live.any():
                    break
                same = (_cubic(c, mid) < 0) == na
                lo = np.where(live & same, mid, lo)
                hi = np.where(live & ~same, mid, hi)
            F = np.stack([F2[i] + lo * D[i] for i in range(9)], axis=1)
            keep = act & np.isfinite(F).all(axis=1)
            if orient:
                keep &= oriented(F, p)
            idx = np.nonzero(keep)[0]
            out[idx, nm[idx]] = F[idx]
            nm += keep
    return nm, out


def denormalise(Fn, nr):
    """T1^T Fn T0, scaled to unit Frobenius norm (squares summed in index order).  Fn [..., 9].  Returns (F [..., 9], finite)."""
    Fn = np.asarray(Fn, dtype=np.float64)
    T0 = [nr[2], 0.0, -(nr[2] * nr[0]), 0.0, nr[2], -(nr[2] * nr[1]), 0.0, 0.0, 1.0]
    T1 = [nr[5], 0.0, -(nr[5] * nr[3]), 0.0, nr[5], -(nr[5] * nr[4]), 0.0, 0.0, 1.0]
    f = [Fn[..., i] for i in range(9)]
    with np.errstate(all="ignore"):
        A = [(f[3 * i] * T0[j] + f[3 * i + 1] * T0[3 + j]) + f[3 * i + 2] * T0[6 + j] for i in range(3) for j in range(3)]
        F = [(T1[i] * A[j] + T1[3 + i] * A[3 + j]) + T1[6 + i] * A[6 + j] for i in range(3) for j in range(3)]
        s = np.zeros_like(F[0])
        for i in range(9):
            s = s + F[i] * F[i]
        s = np.sqrt(s)
        F = np.stack([F[i] / s for i in range(9)], axis=-1)
    return F, np.isfinite(F).all(axis=-1)


def draw(h, n, seed):
    return draw_distinct(7, n, seed, lambda sub: (h, sub, 0, CTR))


def hypotheses(xn, nr, n, seed, rnd, max_iters):
    """Round `rnd`: (sample [ROUND, 7], nmod [ROUND], F [ROUND, 3, 9]) as the device writes them for drawn hypotheses
    (nmod 0 for the rest)."""
    hs = [h for h in range(rnd * ROUND, (rnd + 1) * ROUND) if h < max_iters and (n > 7 or h == 0)]
    sample = np.zeros((ROUND, 7), int)
    nmod = np.zeros(ROUND, int)
    F = np.zeros((ROUND, MODELS, 9))
    if not hs:
        return sample, nmod, F
    for h in hs:
        sample[h - rnd * ROUND] = draw(h, n, seed) if n > 7 else list(range(7))
    loc = np.array(hs) - rnd * ROUND
    nm, Fn = seven_point(xn[sample[loc]])
    for j, hl in enumerate(loc):
        for m in range(nm[j]):
            Fd, fin = denormalise(Fn[j, m], nr)
            if fin:
                F[hl, nmod[hl]] = Fd
                nmod[hl] += 1
    return sample, nmod, F


# ---- loss, score, select -------------------------------------------------------------------------------------------------
def sampson2(F, x0, x1):
    """Squared Sampson distances, every operation rounded: F [M, 9] (or [9]), x0, x1 [N, 2].  Returns [M, N] (or [N])."""
    F = np.asarray(F, dtype=np.float64)
    one = F.ndim == 1
    F = F.reshape(-1, 9)
    f = [F[:, i, None] for i in range(9)]
    x, y, u, v = x0[:, 0], x0[:, 1], x1[:, 0], x1[:, 1]
    with np.errstate(all="ignore"):
        a0 = (f[0] * x + f[1] * y) + f[2]
        a1 = (f[3] * x + f[4] * y) + f[5]
        a2 = (f[6] * x + f[7] * y) + f[8]
        b0 = (f[0] * u + f[3] * v) + f[6]
        b1 = (f[1] * u + f[4] * v) + f[7]
        e = (u * a0 + v * a1) + a2
        r2 = (e * e) / (((a0 * a0 + a1 * a1) + b0 * b0) + b1 * b1)
    return r2[0] if one else r2


def loss_range(thr):
    """k^2 thr^2: the squared residual where the loss reaches 1 (sigma_max = thr)."""
    return K2 * (thr * thr)


def table_at(t, r2, thr):
    """Table t [TABLE + 1] at r2 (< loss_range(thr) where it matters): linear interpolation at p = r2 (TABLE / loss_range(thr))."""
    l2 = loss_range(thr)
    p = np.where(r2 < l2, r2, 0.0) * (float(TABLE) / l2)
    i = np.minimum(p.astype(np.int64), TABLE - 1)
    return t[i] + (p - i) * (t[i + 1] - t[i])


def point_losses(r2, thr, tables):
    return np.where(r2 < loss_range(thr), table_at(tables[0], r2, thr), 1.0)


def score(F, x0, x1, thr, tables):
    """Per slice of SLICE points: (losses [S, M], counts [S, M]) of the models F [M, 9], each loss the sequential sum."""
    n = len(x0)
    S = max(1, -(-n // SLICE))
    L, C = np.zeros((S, len(F))), np.zeros((S, len(F)), int)
    r2 = sampson2(F, x0, x1)
    loss = point_losses(r2, thr, tables)
    for y in range(S):
        j0, j1 = y * SLICE, min(n, (y + 1) * SLICE)
        if j1 > j0:
            L[y] = np.add.accumulate(loss[:, j0:j1], axis=1)[:, -1]
            C[y] = (r2[:, j0:j1] < thr * thr).sum(axis=1)
    return L, C


def model_loss(parts):
    """A model's loss from its slice losses, added in slice order."""
    s = 0.0
    for v in parts:
        s = s + float(v)
    return s


def select(models, n, conf, max_iters):
    """The sequential loop.  models(h) -> list of (loss, count) of hypothesis h.  Returns (hypothesis, slot, loss, niters, iters)."""
    best, hyp, slot, it = np.inf, -1, 0, 0
    niters = 1 if n == 7 else max_iters
    while it < niters:
        for m, (loss, cnt) in enumerate(models(it)):
            if loss < best:
                best, hyp, slot = loss, it, m
                niters = ransac_update_num_iters(conf, (n - cnt) / n, niters, 7)
        it += 1
    return hyp, slot, best, niters, it


# ---- refinement ----------------------------------------------------------------------------------------------------------
def weighted_eight_point(xn, w, nr):
    """The weighted normalised eight-point fit: the smallest eigenvector of sum w a a^T, a = (x'x, x'y, x', y'x, y'y, y', x, y, 1)
    of the normalised points, rank 2 by SVD, de-normalised.  Returns (F [9], finite)."""
    x, y, u, v = xn[:, 0], xn[:, 1], xn[:, 2], xn[:, 3]
    A = np.stack([u * x, u * y, u, v * x, v * y, v, x, y, np.ones_like(x)], axis=1)
    M = (A * w[:, None]).T @ A
    if not np.isfinite(M).all():
        return np.zeros(9), False
    _e, V = np.linalg.eigh(M)
    U, S, Vt = np.linalg.svd(V[:, 0].reshape(3, 3))
    Fn = (U[:, :2] * S[:2]) @ Vt[:2]
    return denormalise(Fn.ravel(), nr)


def total_loss(F, x0, x1, thr, tables):
    return float(point_losses(sampson2(F, x0, x1), thr, tables).sum())


def refine(F, x0, x1, xn, nr, thr, tables):
    """sigma-consensus++ from F [9]: returns the refined F (unit Frobenius norm, largest-magnitude entry positive)."""
    cur = total_loss(F, x0, x1, thr, tables)
    for _ in range(REFINE_ITERS if len(x0) >= 8 else 0):
        r2 = sampson2(F, x0, x1)
        w = np.where(r2 < loss_range(thr), table_at(tables[1], r2, thr), 0.0)
        sel = w > 0
        Fr, fin = weighted_eight_point(xn[sel], w[sel], nr)
        if not fin:
            break
        nl = total_loss(Fr, x0, x1, thr, tables)
        if not nl < cur:
            break
        F, cur = Fr, nl
    F = np.asarray(F, dtype=np.float64)
    m = F[np.argmax(np.abs(F))]
    return F * (-1.0 if m < 0 else 1.0)


# ---- the whole estimate --------------------------------------------------------------------------------------------------
def find_fundamental(x0, x1, thr, conf, max_iters, tables, seed=0, details=None):
    """The device estimator restated.  Returns (F [3, 3] or None, mask bool [N]).  `details` (a dict) receives the
    normalisation, the best hypothesis, slot and loss, final niters, iterations run and the best model."""
    x0 = np.asarray(x0, dtype=np.float64).reshape(-1, 2)
    x1 = np.asarray(x1, dtype=np.float64).reshape(-1, 2)
    n = len(x0)
    if n < 7:
        raise ValueError("fewer than 7 points")
    nr, xn = normalise(x0, x1)
    rounds = {}

    def models(h):
        r = h // ROUND
        if r not in rounds:
            _s, nm, F = hypotheses(xn, nr, n, seed, r, max_iters)
            L, C = score(F.reshape(-1, 9), x0, x1, thr, tables)
            rounds[r] = (nm, F, L, C)
        nm, F, L, C = rounds[r]
        hl = h - r * ROUND
        return [(model_loss(L[:, hl * MODELS + m]), int(C[:, hl * MODELS + m].sum())) for m in range(nm[hl])]

    hyp, slot, best, niters, it = select(models, n, conf, max_iters)
    if details is not None:
        details.update(nr=nr, xn=xn, hyp=hyp, slot=slot, loss=best, niters=niters, iters=it)
    if hyp < 0:
        return None, np.zeros(n, bool)
    Fb = rounds[hyp // ROUND][1][hyp % ROUND, slot]
    if details is not None:
        details.update(F_best=Fb)
    F = refine(Fb, x0, x1, xn, nr, thr, tables)
    return F.reshape(3, 3), sampson2(F, x0, x1) < thr * thr
