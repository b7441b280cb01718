"""numpy statement of `roma_b200.bundle_adjust(..., camera_model="SIMPLE_RADIAL")` (include/romab200.h rules 1-8 with 2', 3',
4' and 6'), in float64 for small scenes.  It is `oracle/bundle.py` with 8 parameters per camera (the pose, f and k) and the gauge
as pinned rows; the pinhole oracle stays the statement of camera_model="PINHOLE".  The LM loop, the Schur reduction and the
`systems` capture restate oracle/bundle.py's rather than share them, so that file stays the unchanged reference of the pinhole
path; a change to the rules of one must be made in both by hand."""
from __future__ import annotations

import math

import numpy as np

from .bundle import LAMBDA0, MAX_LAMBDA, MIN_RELATIVE_DECREASE, NU0, _arr, _rho, rodrigues

NC = 8


def pins(N, fixed_poses=(0,), fixed_tx=(1,), refine_focal_length=True, refine_extra_params=True, fixed_intrinsics=()):
    """Rule 4': the pinned rows [N, 8] bool of every camera; a camera is free when any of its rows is not pinned."""
    if N == 1 and tuple(fixed_tx) == (1,):
        fixed_tx = ()
    p = np.zeros((N, NC), bool)
    p[list(fixed_poses), :6] = True
    p[list(fixed_tx), 3] = True
    p[:, 6] = not refine_focal_length
    p[:, 7] = not refine_extra_params
    p[list(fixed_intrinsics), 6:] = True
    return p


def project(intr, R, t, X, jac):
    """Rule 2' per observation (rows of intr [M, 4], R [M, 3, 3], t [M, 3], X [M, 3]): pixels u [M, 2] and depth; with jac also
    Jc [M, 2, 8] (d_omega, d_t, d_f, d_k) and JX [M, 2, 3] (rule 3')."""
    f, cx, cy, k = (intr[:, j] for j in range(4))
    A = np.einsum("mij,mj->mi", R, X)
    p = A + t
    x, y = p[:, 0] / p[:, 2], p[:, 1] / p[:, 2]
    r2 = x * x + y * y
    d = 1.0 + k * r2
    u = np.stack((f * d * x + cx, f * d * y + cy), 1)
    if not jac:
        return u, p[:, 2]
    iz = 1.0 / p[:, 2]
    Juv = np.empty((p.shape[0], 2, 2))
    Juv[:, 0, 0], Juv[:, 1, 1] = f * (d + 2 * k * x * x), f * (d + 2 * k * y * y)
    Juv[:, 0, 1] = Juv[:, 1, 0] = 2 * f * k * x * y
    Jxy = np.zeros((p.shape[0], 2, 3))
    Jxy[:, 0, 0] = Jxy[:, 1, 1] = iz
    Jxy[:, 0, 2], Jxy[:, 1, 2] = -x * iz, -y * iz
    Jp = Juv @ Jxy
    xy = np.stack((x, y), 1)
    Jc = np.concatenate((np.cross(A[:, None, :], Jp), Jp, (d[:, None] * xy)[:, :, None], (f * r2)[:, None, None] * xy[:, :, None]), 2)
    return u, p[:, 2], Jc, Jp @ R


def bundle_adjust(kp_offsets, keypoints, track_offsets, elements, X, ok, inlier, intrinsics, R, t, *, fixed_poses=(0,), fixed_tx=(1,),
                  refine_focal_length=True, refine_extra_params=True, fixed_intrinsics=(), loss_scale=None, max_iterations=50,
                  function_tolerance=1e-6, systems=None):
    """Returns dict(R, t, intrinsics, X, cost, accepted, termination, trials) as `oracle.bundle.bundle_adjust` does.  A list
    `systems` receives one dict per trial: lam, S [8F, 8F] and b [8F] after rule 4', dc, Dc [F, 8], S_abs, b_abs, and H, g: the
    damped Hessian [8N + 3T, 8N + 3T] and gradient of the whole problem before reduction when `systems` is given with a first
    element "dense" (small scenes only)."""
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    X, okb, inl = _arr(X, np.float64).copy(), _arr(ok, bool), _arr(inlier, bool)
    intr, R, t = _arr(intrinsics, np.float64).copy(), _arr(R, np.float64).copy(), _arr(t, np.float64).copy()
    N, T = intr.shape[0], off.size - 1
    c2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    pin = pins(N, fixed_poses, fixed_tx, refine_focal_length, refine_extra_params, fixed_intrinsics)
    free = [i for i in range(N) if not pin[i].all()]
    F_ = len(free)
    fidx = np.full(N, -1)
    fidx[free] = np.arange(F_)
    pinned = pin[free].reshape(-1)
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(okb, np.diff(off)) & inl)
    img, trk = el[e, 0], track[e]
    obs = xy[kpo[img] + el[e, 1]]
    out = dict(R=R, t=t, intrinsics=intr, X=X, cost=np.zeros(1), accepted=np.zeros(0, bool), termination="nothing_to_adjust", trials=[])
    if e.size == 0:
        return out
    dense = systems is not None and len(systems) > 0 and systems[0] == "dense"
    if dense:
        systems.pop(0)

    def evaluate(intr, R, t, X, jac):
        res = project(intr[img], R[img], t[img], X[trk], jac)
        r = res[0] - obs
        rho, w = _rho((r * r).sum(1), c2)
        F = 0.5 * rho.sum()
        if not jac:
            return F, res[1], intr[img, 0]
        return F, r, w, res[2], res[3]

    F = evaluate(intr, R, t, X, False)[0]
    cost, accepted, trials, lam, nu, term = [F], [], [], LAMBDA0, NU0, "max_iterations"
    for _ in range(max_iterations):
        F, r, w, Jc, JX = evaluate(intr, R, t, X, True)
        U, gc = np.zeros((N, NC, NC)), np.zeros((N, NC))
        V, gp = np.zeros((T, 3, 3)), np.zeros((T, 3))
        np.add.at(U, img, np.einsum("m,mai,maj->mij", w, Jc, Jc))
        np.add.at(gc, img, np.einsum("m,mai,ma->mi", w, Jc, r))
        np.add.at(V, trk, np.einsum("m,mai,maj->mij", w, JX, JX))
        np.add.at(gp, trk, np.einsum("m,mai,ma->mi", w, JX, r))
        Wm = np.einsum("m,mai,maj->mij", w, Jc, JX)
        Dc = np.clip(np.diagonal(U, 0, 1, 2), 1e-6, 1e32)
        Dp = np.clip(np.diagonal(V, 0, 1, 2), 1e-6, 1e32)
        Vinv = np.linalg.inv(V + lam * Dp[:, :, None] * np.eye(3))
        n = NC * F_
        S, b = np.zeros((n, n)), np.zeros(n)
        for fi, i in enumerate(free):
            S[NC * fi:NC * fi + NC, NC * fi:NC * fi + NC] = U[i] + lam * np.diag(Dc[i])
            b[NC * fi:NC * fi + NC] = -gc[i]
        if systems is not None:
            aJc, aJX, ar = np.abs(Jc), np.abs(JX), np.abs(r)
            Uabs, gcabs, gpabs = np.zeros((N, NC, NC)), np.zeros((N, NC)), np.zeros((T, 3))
            np.add.at(Uabs, img, np.einsum("m,mai,maj->mij", w, aJc, aJc))
            np.add.at(gcabs, img, np.einsum("m,mai,ma->mi", w, aJc, ar))
            np.add.at(gpabs, trk, np.einsum("m,mai,ma->mi", w, aJX, ar))
            Wabs, Vabs = np.einsum("m,mai,maj->mij", w, aJc, aJX), np.abs(Vinv)
            S_abs, b_abs = np.zeros((n, n)), np.zeros(n)
            for fi, i in enumerate(free):
                S_abs[NC * fi:NC * fi + NC, NC * fi:NC * fi + NC] = Uabs[i] + lam * np.diag(Dc[i])
                b_abs[NC * fi:NC * fi + NC] = gcabs[i]
        order = np.argsort(trk, kind="stable")
        bounds = np.searchsorted(trk[order], np.arange(T + 1))
        S4 = S.reshape(F_, NC, F_, NC)
        for k in range(T):
            m = order[bounds[k]:bounds[k + 1]]
            m = m[fidx[img[m]] >= 0]
            if m.size == 0:
                continue
            Ak = Wm[m] @ Vinv[k]
            blocks = np.einsum("arm,bcm->abrc", Ak, Wm[m])
            f = fidx[img[m]]
            for a_ in range(m.size):
                b[NC * f[a_]:NC * f[a_] + NC] += Ak[a_] @ gp[k]
                S4[f[a_], :, f, :] -= blocks[a_]
            if systems is not None:
                Aabs = Wabs[m] @ Vabs[k]
                S4abs = S_abs.reshape(F_, NC, F_, NC)
                blocks_abs = np.einsum("arm,bcm->abrc", Aabs, Wabs[m])
                for a_ in range(m.size):
                    b_abs[NC * f[a_]:NC * f[a_] + NC] += Aabs[a_] @ gpabs[k]
                    S4abs[f[a_], :, f, :] += blocks_abs[a_]
        for j in np.flatnonzero(pinned):
            S[j, :] = S[:, j] = 0.0
            S[j, j] = 1.0
            b[j] = 0.0
            if systems is not None:
                S_abs[j, :] = S_abs[:, j] = b_abs[j] = 0.0
        dc, pivot_ok = np.zeros(n), True
        if n:
            try:
                L = np.linalg.cholesky(S)
                dc = np.linalg.solve(L.T, np.linalg.solve(L, b))
            except np.linalg.LinAlgError:
                pivot_ok = False
        if systems is not None:
            rec = dict(lam=lam, S=S, b=b, dc=dc, Dc=Dc[free], S_abs=S_abs, b_abs=b_abs, free=free)
            if dense:
                H = np.zeros((NC * N + 3 * T,) * 2)
                g = np.zeros(NC * N + 3 * T)
                for q, (i, kk) in enumerate(zip(img, trk)):
                    J = np.zeros((2, NC * N + 3 * T))
                    J[:, NC * i:NC * i + NC] = Jc[q]
                    J[:, NC * N + 3 * kk:NC * N + 3 * kk + 3] = JX[q]
                    H += w[q] * J.T @ J
                    g += w[q] * J.T @ r[q]
                D = np.clip(np.diag(H), 1e-6, 1e32)
                rec.update(H=H + lam * np.diag(D), g=g)
            systems.append(rec)
        dC = np.zeros((N, NC))
        dC[free] = dc.reshape(F_, NC)
        bX = np.zeros((T, 3))
        np.add.at(bX, trk, np.einsum("mij,mi->mj", Wm, dC[img]))
        dX = np.einsum("kij,kj->ki", Vinv, -gp - bX)
        dX[~okb] = 0.0
        pred = 0.5 * (np.einsum("ni,ni->", dC[free], lam * Dc[free] * dC[free] - gc[free])
                      + np.einsum("ki,ki->", dX[okb], lam * Dp[okb] * dX[okb] - gp[okb]))
        R1 = np.where(pin[:, :3].all(1)[:, None, None], R, rodrigues(dC[:, :3]) @ R)
        t1 = np.where(pin[:, 3:6], t, t + dC[:, 3:6])
        intr1 = intr.copy()
        intr1[:, 0] = np.where(pin[:, 6], intr[:, 0], intr[:, 0] + dC[:, 6])
        intr1[:, 3] = np.where(pin[:, 7], intr[:, 3], intr[:, 3] + dC[:, 7])
        X1 = X + dX
        F1, depth, f1 = evaluate(intr1, R1, t1, X1, False)
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = float(np.float64(F - F1) / np.float64(pred))
        keep = pivot_ok and math.isfinite(F1) and (depth > 0).all() and (f1 > 0).all() and rho > MIN_RELATIVE_DECREASE
        trials.append(dict(F=F, F_new=F1, pred=pred, rho=rho, margin=rho - MIN_RELATIVE_DECREASE,
                           step=float(max(np.abs(dc).max(initial=0.0), np.abs(dX).max(initial=0.0)))))
        accepted.append(bool(keep))
        if keep:
            intr, R, t, X = intr1, R1, t1, X1
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
    return dict(R=R, t=t, intrinsics=intr, X=X, cost=np.asarray(cost), accepted=np.asarray(accepted, bool), termination=term,
                trials=trials)


def track_costs(kp_offsets, keypoints, track_offsets, elements, X, ok, inlier, intrinsics, R, t, loss_scale=None):
    """Rule 2's cost of every track [T] under SIMPLE_RADIAL cameras (0 for a track that is not ok)."""
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    X, okb, inl = _arr(X, np.float64), _arr(ok, bool), _arr(inlier, bool)
    intr, R, t = _arr(intrinsics, np.float64), _arr(R, np.float64), _arr(t, np.float64)
    T = off.size - 1
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(okb, np.diff(off)) & inl)
    img = el[e, 0]
    r = project(intr[img], R[img], t[img], X[track[e]], False)[0] - xy[kpo[img] + el[e, 1]]
    rho, _ = _rho((r * r).sum(1), 0.0 if loss_scale is None else float(loss_scale) ** 2)
    out = np.zeros(T)
    np.add.at(out, track[e], 0.5 * rho)
    return out
