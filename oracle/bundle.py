"""numpy statement of `roma_b200.bundle_adjust` (include/romab200.h, INTEGRATION.md), rules 1-7 in float64 for small scenes: the
Jacobian blocks of every used observation, the blocks of H = J^T W J, the Schur complement on the free cameras as a dense matrix,
`np.linalg.cholesky` and triangular solves.  The device sums in other orders, so the two agree to a tolerance, and their kept and
rejected trials agree wherever rho is not within rounding of 1e-3: every trial reports F, pred, rho and that margin."""
from __future__ import annotations

import math

import numpy as np

LAMBDA0, NU0, MIN_RELATIVE_DECREASE, MAX_LAMBDA = 1e-4, 2.0, 1e-3, 1e32


def _arr(v, dtype):
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype)


def rodrigues(w):
    """Rule 3's Exp of w [..., 3]: Rodrigues, or I + [w]x where |w|^2 <= 2^-52."""
    w = np.asarray(w, np.float64)
    t2 = (w * w).sum(-1)
    big = t2 > 2.0 ** -52
    th = np.sqrt(np.where(big, t2, 1.0))
    k = np.where(big[..., None], w / th[..., None], w)
    Kx = np.zeros(w.shape[:-1] + (3, 3))
    Kx[..., 0, 1], Kx[..., 0, 2], Kx[..., 1, 2] = -k[..., 2], k[..., 1], -k[..., 0]
    Kx -= np.swapaxes(Kx, -1, -2)
    c, s = np.cos(th)[..., None, None], np.sin(th)[..., None, None]
    kk = k[..., :, None] * k[..., None, :]
    full = c * np.eye(3) + (1 - c) * kk + s * Kx
    return np.where(big[..., None, None], full, np.eye(3) + Kx)


def camera_major(track_offsets, elements, ok, inlier, num_images):
    """Rule 1's used observations in camera-major order, ascending element order within an image: (obs_offsets [N + 1], obs)."""
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    used = np.repeat(_arr(ok, bool), np.diff(off)) & _arr(inlier, bool)
    e = np.flatnonzero(used)
    obs = e[np.argsort(el[e, 0], kind="stable")]
    return np.searchsorted(el[obs, 0], np.arange(num_images + 1), "left").astype(np.int64), obs


def _rho(s, c2):
    if c2 == 0.0:
        return s, np.ones_like(s)
    return c2 * np.log1p(s / c2), 1.0 / (1.0 + s / c2)


def bundle_adjust(kp_offsets, keypoints, track_offsets, elements, X, ok, inlier, K, R, t, *, fixed_poses=(0,), fixed_tx=(1,),
                  loss_scale=None, max_iterations=50, function_tolerance=1e-6):
    """Rules 1-7.  Returns dict(R, t, X, cost [n + 1], accepted [n], termination, trials: per trial F, F_new, pred, rho, margin
    (rho - 1e-3), step (the largest |d| entry))."""
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    X, okb, inl = _arr(X, np.float64).copy(), _arr(ok, bool), _arr(inlier, bool)
    K, R, t = _arr(K, np.float64), _arr(R, np.float64).copy(), _arr(t, np.float64).copy()
    N, T = K.shape[0], off.size - 1
    if N == 1 and tuple(fixed_tx) == (1,):
        fixed_tx = ()
    c2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(okb, np.diff(off)) & inl)
    img, trk = el[e, 0], track[e]
    obs = xy[kpo[img] + el[e, 1]]
    free = [i for i in range(N) if i not in set(fixed_poses)]
    F_ = len(free)
    fidx = np.full(N, -1)
    fidx[free] = np.arange(F_)
    tx = [fidx[i] for i in set(fixed_tx) if fidx[i] >= 0]
    out = dict(R=R, t=t, X=X, cost=np.zeros(1), accepted=np.zeros(0, bool), termination="nothing_to_adjust", trials=[])
    if e.size == 0:
        return out

    def evaluate(R, t, X, jac):
        A = np.einsum("mij,mj->mi", R[img], X[trk])
        p = A + t[img]
        q = np.einsum("mij,mj->mi", K[img], p)
        u = q[:, :2] / q[:, 2:3]
        r = u - obs
        s = (r * r).sum(1)
        rho, w = _rho(s, c2)
        F = 0.5 * rho.sum()
        if not jac:
            return F, p[:, 2]
        iz = 1.0 / q[:, 2]
        Jq = np.zeros((e.size, 2, 3))
        Jq[:, 0, 0] = Jq[:, 1, 1] = iz
        Jq[:, 0, 2], Jq[:, 1, 2] = -u[:, 0] * iz, -u[:, 1] * iz
        Jp = Jq @ K[img]
        Jc = np.concatenate((np.cross(A[:, None, :], Jp), Jp), 2)          # d_omega: (R X) x Jp, then d_t
        JX = Jp @ R[img]
        return F, r, w, Jc, JX

    F, _ = evaluate(R, t, X, False)
    cost, accepted, trials, lam, nu, term = [F], [], [], LAMBDA0, NU0, "max_iterations"
    for _ in range(max_iterations):
        F, r, w, Jc, JX = evaluate(R, t, X, True)
        U = np.zeros((N, 6, 6))
        gc = np.zeros((N, 6))
        V = np.zeros((T, 3, 3))
        gp = np.zeros((T, 3))
        np.add.at(U, img, np.einsum("m,mai,maj->mij", w, Jc, Jc))
        np.add.at(gc, img, np.einsum("m,mai,ma->mi", w, Jc, r))
        np.add.at(V, trk, np.einsum("m,mai,maj->mij", w, JX, JX))
        np.add.at(gp, trk, np.einsum("m,mai,ma->mi", w, JX, r))
        Wm = np.einsum("m,mai,maj->mij", w, Jc, JX)                        # [M, 6, 3]
        Dc = np.clip(np.diagonal(U, 0, 1, 2), 1e-6, 1e32)
        Dp = np.clip(np.diagonal(V, 0, 1, 2), 1e-6, 1e32)
        Vinv = np.linalg.inv(V + lam * Dp[:, :, None] * np.eye(3))
        n = 6 * F_
        S = np.zeros((n, n))
        b = np.zeros(n)
        for fi, i in enumerate(free):
            S[6 * fi:6 * fi + 6, 6 * fi:6 * fi + 6] = U[i] + lam * np.diag(Dc[i])
            b[6 * fi:6 * fi + 6] = -gc[i]
        order = np.argsort(trk, kind="stable")
        bounds = np.searchsorted(trk[order], np.arange(T + 1))
        for k in range(T):
            m = order[bounds[k]:bounds[k + 1]]
            m = m[fidx[img[m]] >= 0]
            if m.size == 0:
                continue
            Ak = Wm[m] @ Vinv[k]                                           # [L, 6, 3]
            blocks = np.einsum("arm,bcm->abrc", Ak, Wm[m])
            f = fidx[img[m]]
            S4 = S.reshape(F_, 6, F_, 6)
            for a_ in range(m.size):                                       # a track's images are distinct
                b[6 * f[a_]:6 * f[a_] + 6] += Ak[a_] @ gp[k]
                S4[f[a_], :, f, :] -= blocks[a_]
        for fi in tx:
            j = 6 * fi + 3
            S[j, :] = 0.0
            S[:, j] = 0.0
            S[j, j] = 1.0
            b[j] = 0.0
        dc = np.zeros(n)
        pivot_ok = True
        if n:
            try:
                L = np.linalg.cholesky(S)
                dc = np.linalg.solve(L.T, np.linalg.solve(L, b))
            except np.linalg.LinAlgError:
                pivot_ok = False
        dC = np.zeros((N, 6))
        dC[free] = dc.reshape(F_, 6)
        bX = np.zeros((T, 3))
        np.add.at(bX, trk, np.einsum("mij,mi->mj", Wm, dC[img]))
        dX = np.einsum("kij,kj->ki", Vinv, -gp - bX)
        dX[~okb] = 0.0
        pred = 0.5 * (np.einsum("ni,ni->", dC[free], lam * Dc[free] * dC[free] - gc[free])
                      + np.einsum("ki,ki->", dX[okb], lam * Dp[okb] * dX[okb] - gp[okb]))
        R1 = rodrigues(dC[:, :3]) @ R
        t1, X1 = t + dC[:, 3:], X + dX
        F1, depth = evaluate(R1, t1, X1, False)
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = float(np.float64(F - F1) / np.float64(pred))
        keep = pivot_ok and math.isfinite(F1) and (depth > 0).all() and rho > MIN_RELATIVE_DECREASE
        trials.append(dict(F=F, F_new=F1, pred=pred, rho=rho, margin=rho - MIN_RELATIVE_DECREASE,
                           step=float(max(np.abs(dc).max(initial=0.0), np.abs(dX).max(initial=0.0)))))
        accepted.append(bool(keep))
        if keep:
            R, t, X = R1, t1, X1
            cost.append(F1)
            lam *= max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3)
            nu = NU0
            if F - F1 <= function_tolerance * F:
                term = "function_tolerance"
                break
        else:
            cost.append(F)
            lam *= nu
            nu *= 2.0
            if lam > MAX_LAMBDA:
                term = "no_progress"
                break
    return dict(R=R, t=t, X=X, cost=np.asarray(cost), accepted=np.asarray(accepted, bool), termination=term, trials=trials)


def track_costs(kp_offsets, keypoints, track_offsets, elements, X, ok, inlier, K, R, t, loss_scale=None):
    """Rule 2's cost of every track [T] at the given cameras and points (0 for a track that is not ok)."""
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    X, okb, inl = _arr(X, np.float64), _arr(ok, bool), _arr(inlier, bool)
    K, R, t = _arr(K, np.float64), _arr(R, np.float64), _arr(t, np.float64)
    T = off.size - 1
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(okb, np.diff(off)) & inl)
    img = el[e, 0]
    q = np.einsum("mij,mj->mi", K[img], np.einsum("mij,mj->mi", R[img], X[track[e]]) + t[img])
    r = q[:, :2] / q[:, 2:3] - xy[kpo[img] + el[e, 1]]
    rho, _ = _rho((r * r).sum(1), 0.0 if loss_scale is None else float(loss_scale) ** 2)
    out = np.zeros(T)
    np.add.at(out, track[e], 0.5 * rho)
    return out
