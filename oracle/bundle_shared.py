"""numpy statement of `roma_b200.bundle_adjust(..., camera_model="SIMPLE_RADIAL", camera_ids=ids)` (include/romab200.h rules 1-8
with 2'-6' and the shared-intrinsics rules 4''-5''), in float64 for small scenes.  It builds every observation's Jacobian in the
shared parameters directly: the pose of each free camera, then (f, k) of each group that has a free camera.  It then assembles
and Schur-reduces that system and solves it by dense Cholesky.  It never forms the per-image system and never folds it, so the
device's fold is checked against an independent statement.  Per-image intrinsics (oracle/bundle_radial.py) are the special case
camera_ids = arange(N) up to rounding.  The LM loop restates oracle/bundle_radial.py's; a change to the rules of one must be made
in both by hand."""
from __future__ import annotations

import math

import numpy as np

from .bundle import LAMBDA0, MAX_LAMBDA, MIN_RELATIVE_DECREASE, NU0, _arr, _rho, rodrigues
from .bundle_radial import project


def layout(camera_ids, fixed_poses=(0,), fixed_tx=(1,), refine_focal_length=True, refine_extra_params=True, fixed_intrinsics=()):
    """Rule 4'': the pinned pose rows [N, 6] bool, the pinned (f, k) of every camera id [C, 2] bool (fixed_intrinsics lists camera
    ids), the free cameras (pose free or group intrinsics free) ascending, and the groups with a free camera ascending."""
    ids = np.asarray(camera_ids, np.int64)
    N, C = ids.size, int(ids.max()) + 1
    if N == 1 and tuple(fixed_tx) == (1,):
        fixed_tx = ()
    pose_pin = np.zeros((N, 6), bool)
    pose_pin[list(fixed_poses)] = True
    pose_pin[list(fixed_tx), 3] = True
    group_pin = np.zeros((C, 2), bool)
    group_pin[:, 0] = not refine_focal_length
    group_pin[:, 1] = not refine_extra_params
    group_pin[list(fixed_intrinsics)] = True
    free = [i for i in range(N) if not (pose_pin[i].all() and group_pin[ids[i]].all())]
    groups = sorted(set(ids[free].tolist()))
    return pose_pin, group_pin, free, groups


def bundle_adjust(kp_offsets, keypoints, track_offsets, elements, X, ok, inlier, intrinsics, R, t, camera_ids, *, fixed_poses=(0,),
                  fixed_tx=(1,), refine_focal_length=True, refine_extra_params=True, fixed_intrinsics=(), loss_scale=None,
                  max_iterations=50, function_tolerance=1e-6, systems=None):
    """Returns dict(R, t, intrinsics, X, cost, accepted, termination, trials) as `oracle.bundle_radial.bundle_adjust` does; the
    rows of intrinsics within a group stay equal.  A list `systems` receives one dict per trial: lam, S [n', n'] and b [n'] after
    the pins, d [n'], D [n'] (the damping diagonal: each free camera's clamped pose diagonal, and per group the sum of its free
    members' clamped f and k diagonals), gc [n'] (the gradient J'^T W r in the shared parameters), and S_abs, b_abs: the assembly
    of S and b repeated over the absolute value of every term (0 in pinned rows and columns), the summation scale of their rounding
    error; with n' = 6F + 2G."""
    kpo, xy = _arr(kp_offsets, np.int64), _arr(keypoints, np.float64)
    off, el = _arr(track_offsets, np.int64), _arr(elements, np.int64).reshape(-1, 2)
    X, okb, inl = _arr(X, np.float64).copy(), _arr(ok, bool), _arr(inlier, bool)
    intr, R, t = _arr(intrinsics, np.float64).copy(), _arr(R, np.float64).copy(), _arr(t, np.float64).copy()
    ids = np.asarray(camera_ids, np.int64)
    N, T = intr.shape[0], off.size - 1
    c2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    pose_pin, group_pin, free, groups = layout(ids, fixed_poses, fixed_tx, refine_focal_length, refine_extra_params, fixed_intrinsics)
    F_, G = len(free), len(groups)
    n = 6 * F_ + 2 * G
    # the shared parameter of each camera's 8 local ones, or -1
    col = np.full((N, 8), -1, np.int64)
    for fi, i in enumerate(free):
        col[i, :6] = 6 * fi + np.arange(6)
    for gl, g in enumerate(groups):
        col[ids == g, 6:] = 6 * F_ + 2 * gl + np.arange(2)
    is_free = np.zeros(N, bool)
    is_free[free] = True
    col[~is_free] = -1              # a camera that is not free is pinned in all 8, so it adds nothing
    pinned = np.zeros(n, bool)
    for fi, i in enumerate(free):
        pinned[6 * fi:6 * fi + 6] = pose_pin[i]
    for gl, g in enumerate(groups):
        pinned[6 * F_ + 2 * gl:6 * F_ + 2 * gl + 2] = group_pin[g]
    track = np.repeat(np.arange(T), np.diff(off))
    e = np.flatnonzero(np.repeat(okb, np.diff(off)) & inl)
    img, trk = el[e, 0], track[e]
    obs = xy[kpo[img] + el[e, 1]]
    out = dict(R=R, t=t, intrinsics=intr, X=X, cost=np.zeros(1), accepted=np.zeros(0, bool), termination="nothing_to_adjust", trials=[])
    if e.size == 0:
        return out

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
        M = img.size
        # the Jacobian of every observation in the shared parameters [M, 2, n'], built directly
        J = np.zeros((M, 2, n))
        c = col[img]
        for p in range(8):
            on = c[:, p] >= 0
            J[np.flatnonzero(on), :, c[on, p]] += Jc[on, :, p]
        U = np.einsum("m,mai,maj->ij", w, J, J)
        gc = np.einsum("m,mai,ma->i", w, J, r)
        V, gp = np.zeros((T, 3, 3)), np.zeros((T, 3))
        np.add.at(V, trk, np.einsum("m,mai,maj->mij", w, JX, JX))
        np.add.at(gp, trk, np.einsum("m,mai,ma->mi", w, JX, r))
        Wk = np.zeros((T, n, 3))
        np.add.at(Wk, trk, np.einsum("m,mai,maj->mij", w, J, JX))
        # damping: the clamped diagonal of each free camera's own 8 x 8 block, summed into its shared parameters
        Ui = np.zeros((N, 8))
        np.add.at(Ui, img, np.einsum("m,map,map->mp", w, Jc, Jc))
        D = np.zeros(n)
        for i in free:
            np.add.at(D, col[i], np.clip(Ui[i], 1e-6, 1e32))
        Dp = np.clip(np.diagonal(V, 0, 1, 2), 1e-6, 1e32)
        Vinv = np.linalg.inv(V + lam * Dp[:, :, None] * np.eye(3))
        A = Wk @ Vinv                                   # W_k V_k^-1 [T, n', 3]
        S = U + lam * np.diag(D) - np.tensordot(A, Wk, axes=([0, 2], [0, 2]))
        b = -gc + np.einsum("kai,ki->a", A, gp)
        if systems is not None:
            # the same assembly over |term|: folding only adds entries, so this is P^T S_abs P of the per-image system
            # (in matrix products: this is a scale, so its summation order does not matter)
            aJ, ar, aJX = np.abs(J), np.abs(r), np.abs(JX)
            wJ = (w[:, None, None] * aJ).reshape(-1, n)
            Wabs = np.zeros((T, n, 3))
            np.add.at(Wabs, trk, wJ.reshape(M, 2, n).transpose(0, 2, 1) @ aJX)
            gpabs = np.zeros((T, 3))
            np.add.at(gpabs, trk, np.einsum("m,mai,ma->mi", w, aJX, ar))
            Aabs = Wabs @ np.abs(Vinv)
            S_abs = wJ.T @ aJ.reshape(-1, n) + lam * np.diag(D) + np.tensordot(Aabs, Wabs, axes=([0, 2], [0, 2]))
            b_abs = wJ.T @ ar.reshape(-1) + np.einsum("kai,ki->a", Aabs, gpabs)
        for j in np.flatnonzero(pinned):
            S[j, :] = S[:, j] = 0.0
            S[j, j] = 1.0
            b[j] = 0.0
            if systems is not None:
                S_abs[j, :] = S_abs[:, j] = b_abs[j] = 0.0
        d, pivot_ok = np.zeros(n), True
        if n:
            try:
                L = np.linalg.cholesky(S)
                d = np.linalg.solve(L.T, np.linalg.solve(L, b))
            except np.linalg.LinAlgError:
                pivot_ok = False
        if systems is not None:
            systems.append(dict(lam=lam, S=S, b=b, d=d, D=D, gc=gc, free=free, groups=groups, S_abs=S_abs, b_abs=b_abs))
        dX = np.einsum("kij,kj->ki", Vinv, -gp - np.einsum("kai,a->ki", Wk, d))
        dX[~okb] = 0.0
        pred = 0.5 * (d @ (lam * D * d - gc) + np.einsum("ki,ki->", dX[okb], lam * Dp[okb] * dX[okb] - gp[okb]))
        # every camera's local step: its pose rows, and its group's (f, k)
        dC = np.where(col >= 0, np.concatenate((d, [0.0]))[col], 0.0)
        R1 = np.where(pose_pin[:, :3].all(1)[:, None, None] | ~is_free[:, None, None], R, rodrigues(dC[:, :3]) @ R)
        t1 = np.where(pose_pin[:, 3:6] | ~is_free[:, None], t, t + dC[:, 3:6])
        intr1 = intr.copy()
        fpin, kpin = group_pin[ids, 0] | ~is_free, group_pin[ids, 1] | ~is_free
        intr1[:, 0] = np.where(fpin, intr[:, 0], intr[:, 0] + dC[:, 6])
        intr1[:, 3] = np.where(kpin, intr[:, 3], intr[:, 3] + dC[:, 7])
        X1 = X + dX
        F1, depth, f1 = evaluate(intr1, R1, t1, X1, False)
        with np.errstate(divide="ignore", invalid="ignore"):
            rho = float(np.float64(F - F1) / np.float64(pred))
        keep = pivot_ok and math.isfinite(F1) and (depth > 0).all() and (f1 > 0).all() and rho > MIN_RELATIVE_DECREASE
        trials.append(dict(F=F, F_new=F1, pred=pred, rho=rho, margin=rho - MIN_RELATIVE_DECREASE,
                           step=float(max(np.abs(d).max(initial=0.0), np.abs(dX).max(initial=0.0)))))
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
