"""numpy float64 statement of the dense reconstruction rules (include/romab200.h): `triangulate_warps` (per element: position,
rejection reason, depth, and the cell winner), `fuse_depth_maps` (multi-view agreement and the emission rule) and the camera table
they share (`roma_b200.dense.camera_table`).  The device may contract a multiply and an add into one FMA and solves the DLT by
Jacobi rather than LAPACK, so its float64 values differ from these in the last bits: depths agree to float32 rounding, and a
decision agrees wherever the tested quantity is clear of its threshold.  `margins` returns the relative distance of every tested
quantity to its threshold, so tests can tell the two apart."""
from __future__ import annotations

import numpy as np

from oracle.camera import ITERS

CERT, RANGE, UNREG, CLAMP, BEHIND, REPROJ, ANGLE = 1, 2, 3, 4, 5, 6, 7


def _normalise(cam, radial, x, y):
    """Rule 4: (a, b, clamped) of pixels (x, y) [M] under camera rows cam [M, 36]."""
    if not radial:
        Ki = cam[:, 9:18].reshape(-1, 3, 3)
        h = Ki @ np.stack((x, y, np.ones_like(x)), 1)[..., None]
        return h[:, 0, 0] / h[:, 2, 0], h[:, 1, 0] / h[:, 2, 0], np.zeros(x.shape, bool)
    f, cx, cy, k = cam[:, 30], cam[:, 31], cam[:, 32], cam[:, 33]
    dx, dy = x - cx, y - cy
    rd = np.sqrt(dx * dx + dy * dy) / f
    plain = (k == 0.0) | (rd == 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        clamp = ~plain & (k < 0.0) & (rd >= 2.0 / (3.0 * np.sqrt(-3.0 * k)))
        rho = rd.copy()
        live = ~plain & ~clamp
        for _ in range(ITERS):
            step = (rho * (1.0 + k * rho * rho) - rd) / (1.0 + 3.0 * k * rho * rho)
            rho = np.where(live, rho - step, rho)
            live &= step != 0.0
        s = np.where(plain | clamp, 1.0, rho / rd)
    return dx * s / f, dy * s / f, clamp


def _project(cam, radial, X):
    """Pixels [M, 2] of camera-frame points X [M, 3]."""
    if not radial:
        p = (cam[:, 0:9].reshape(-1, 3, 3) @ X[..., None])[..., 0]
        return p[:, :2] / p[:, 2:]
    f, cx, cy, k = cam[:, 30], cam[:, 31], cam[:, 32], cam[:, 33]
    x, y = X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    d = 1.0 + k * (x * x + y * y)
    return np.stack((f * d * x + cx, f * d * y + cy), 1)


def _dlt(R, t, x0, y0, x1, y1):
    """dlt_two_view for M elements: the eigenvector of the smallest eigenvalue of A^T A, as homogeneous Q [M, 4]."""
    z, o = np.zeros_like(x0), np.ones_like(x0)
    A = np.stack([np.stack((-o, z, x0, z), 1), np.stack((z, -o, y0, z), 1),
                  np.stack((x1 * R[6] - R[0], x1 * R[7] - R[1], x1 * R[8] - R[2], x1 * t[2] - t[0]), 1),
                  np.stack((y1 * R[6] - R[3], y1 * R[7] - R[4], y1 * R[8] - R[5], y1 * t[2] - t[1]), 1)], 1)
    _, V = np.linalg.eigh(np.einsum("mki,mkj->mij", A, A))
    return V[:, :, 0]


def pair_elements(pair, half, warp, certainty, image_sizes, cameras, registered, radial, min_certainty, max_error, min_angle):
    """Rules 1-5 for every element of one pair-half: warp [H, 2W, 4] and certainty [H, 2W] of the pair (i, j) = pair.  Returns a
    dict of [H, W] arrays: reason int, depth float64 (NaN unless accepted), cert float32, and the margins of every tested quantity
    (error2 of each side, the angle, the two depths) for the accepted and later-rejected elements."""
    H, W = certainty.shape[0], certainty.shape[1] // 2
    g, m = int(pair[half]), int(pair[1 - half])
    cert = certainty[:, half * W:(half + 1) * W].reshape(-1).astype(np.float32)
    uv = warp[:, half * W:(half + 1) * W, 2 * (1 - half):2 * (1 - half) + 2].reshape(-1, 2).astype(np.float32)
    r, c = np.divmod(np.arange(H * W), W)
    Hg, Wg = float(image_sizes[g][0]), float(image_sizes[g][1])
    Hm, Wm = image_sizes[m]
    xg, yg = Wg * (c + 0.5) / W, Hg * (r + 0.5) / H
    xm = (np.float32(Wm) * np.float32(0.5) * (uv[:, 0] + np.float32(1))).astype(np.float64)
    ym = (np.float32(Hm) * np.float32(0.5) * (uv[:, 1] + np.float32(1))).astype(np.float64)
    reason = np.zeros(H * W, np.int64)
    bad = ~(cert > np.float32(min_certainty)) | ~np.isfinite(cert) | ~np.isfinite(uv).all(1)
    reason[bad] = CERT
    with np.errstate(invalid="ignore"):
        out = ~((np.abs(uv) <= 1).all(1))
    reason[(reason == 0) & out] = RANGE
    if not (registered[g] and registered[m]):
        reason[reason == 0] = UNREG
    M = H * W
    cg, cm = np.repeat(cameras[g][None], M, 0), np.repeat(cameras[m][None], M, 0)
    with np.errstate(all="ignore"):
        ag, bg, clg = _normalise(cg, radial, xg, yg)
        am, bm, clm = _normalise(cm, radial, xm, ym)
        reason[(reason == 0) & (clg | clm)] = CLAMP
        Rg, Rm = cameras[g][18:27].reshape(3, 3), cameras[m][18:27].reshape(3, 3)
        Rr = Rm @ Rg.T
        tr = cameras[m][27:30] - Rr @ cameras[g][27:30]
        live = reason == 0
        Q = np.full((M, 4), np.nan)
        if live.any():
            Q[live] = _dlt(Rr.reshape(9), tr, ag[live], bg[live], am[live], bm[live])
        X = Q[:, :3] / Q[:, 3:]
        Xm = X @ Rr.T + tr
        behind = (Q[:, 3] == 0) | ~(X[:, 2] > 0) | ~(Xm[:, 2] > 0)
        reason[(reason == 0) & behind] = BEHIND
        pg, pm = _project(cg, radial, X), _project(cm, radial, Xm)
        eg = (pg[:, 0] - xg) ** 2 + (pg[:, 1] - yg) ** 2
        em = (pm[:, 0] - xm) ** 2 + (pm[:, 1] - ym) ** 2
        reason[(reason == 0) & ~((eg <= max_error ** 2) & (em <= max_error ** 2))] = REPROJ
        C = -Rr.T @ tr
        b = X - C
        ang = np.arctan2(np.linalg.norm(np.cross(X, b), axis=1), (X * b).sum(1))
        reason[(reason == 0) & ~(ang >= np.deg2rad(min_angle))] = ANGLE
    depth = np.where(reason == 0, X[:, 2], np.nan)
    sh = (H, W)
    return {"reason": reason.reshape(sh), "depth": depth.reshape(sh), "cert": cert.reshape(sh), "eg": eg.reshape(sh), "em": em.reshape(sh),
            "angle": ang.reshape(sh), "z": X[:, 2].reshape(sh), "zm": Xm[:, 2].reshape(sh), "image": g}


def triangulate_warps(pairs, warps, certainties, image_sizes, cameras, registered, radial=0, min_certainty=0.05, max_error=4.0,
                      min_angle=1.5, first_pair=0, maps=None):
    """The whole call: returns maps dict(depth [N, H, W] float32, score, source int64, pair_counts [P, 8]) and the per pair-half
    element dicts.  `maps` accumulates as depth_maps does."""
    pairs = np.asarray(pairs, np.int64)
    N, (H, W) = len(image_sizes), (certainties.shape[1], certainties.shape[2] // 2)
    if maps is None:
        maps = {"depth": np.zeros((N, H, W), np.float32), "score": np.zeros((N, H, W), np.float32),
                "source": np.full((N, H, W), -1, np.int64), "pair_counts": np.zeros((len(pairs), 8), np.int64)}
    elems = {}
    for row in range(warps.shape[0]):
        k = first_pair + row
        for half in (0, 1):
            e = pair_elements(pairs[k], half, warps[row], certainties[row], image_sizes, cameras, registered, radial, min_certainty,
                              max_error, min_angle)
            elems[(k, half)] = e
            maps["pair_counts"][k] += np.bincount(e["reason"].reshape(-1), minlength=8)
            g, ok = e["image"], e["reason"] == 0
            src = 2 * k + half
            sc, so = maps["score"][g], maps["source"][g]
            better = ok & ((e["cert"] > sc) | ((e["cert"] == sc) & ((so < 0) | (src < so))))
            maps["depth"][g][better] = e["depth"][better].astype(np.float32)
            sc[better], so[better] = e["cert"][better], src
    return maps, elems


def neighbours(pairs, registered):
    nb = [set() for _ in registered]
    for i, j in np.asarray(pairs).tolist():
        if i != j and registered[i] and registered[j]:
            nb[i].add(j)
            nb[j].add(i)
    return [sorted(s) for s in nb]


def _backproject(cam, radial, img_size, H, W, r, c, d):
    """F1: (position [M, 2], world points [M, 3], clamped [M]) of grid pixels (r, c) at depths d."""
    x, y = float(img_size[1]) * (c + 0.5) / W, float(img_size[0]) * (r + 0.5) / H
    cams = np.repeat(cam[None], len(r), 0)
    a, b, cl = _normalise(cams, radial, x, y)
    q = np.stack((d * a, d * b, d), 1) - cam[27:30]
    return np.stack((x, y), 1), q @ cam[18:27].reshape(3, 3), cl


def fuse_depth_maps(depth, score, pairs, image_sizes, cameras, registered, radial=0, colors=None, max_reproj_error=2.0,
                    max_depth_error=0.01, min_num_views=3, margins=None):
    """Rules F1-F3.  Returns dict(points, colors, image, pixel, num_views, score) in emission order.  A list `margins` receives, per
    image, the per-pixel minimum relative distance of its depth and reprojection tests to their thresholds (inf without a test)."""
    N, H, W = depth.shape
    nb = neighbours(pairs, registered)
    out = {k: [] for k in ("points", "colors", "image", "pixel", "num_views", "score")}
    for i in range(N):
        if not registered[i]:
            continue
        pix = np.flatnonzero(depth[i].reshape(-1) > 0)
        r, c = np.divmod(pix, W)
        d = depth[i].reshape(-1)[pix].astype(np.float64)
        pos, X, cl = _backproject(cameras[i], radial, image_sizes[i], H, W, r, c, d)
        S, agree, lower = X.copy(), np.zeros(len(pix), np.int64), np.zeros(len(pix), bool)
        marg = np.full(len(pix), np.inf)
        ci = np.repeat(cameras[i][None], len(pix), 0)
        for j in nb[i]:
            cj = np.repeat(cameras[j][None], len(pix), 0)
            with np.errstate(all="ignore"):
                Xj = X @ cameras[j][18:27].reshape(3, 3).T + cameras[j][27:30]
                front = Xj[:, 2] > 0
                uv = _project(cj, radial, Xj)
                gc = np.floor(uv[:, 0] * W / image_sizes[j][1])
                gr = np.floor(uv[:, 1] * H / image_sizes[j][0])
                inside = front & (gc >= 0) & (gc < W) & (gr >= 0) & (gr < H)
                qr, qc = np.where(inside, gr, 0).astype(np.int64), np.where(inside, gc, 0).astype(np.int64)
                dq = depth[j][qr, qc].astype(np.float64)
                derr = np.abs(dq - Xj[:, 2])
                ok = inside & (dq > 0) & (derr <= max_depth_error * Xj[:, 2])
                marg = np.where(inside & (dq > 0), np.minimum(marg, np.abs(derr - max_depth_error * Xj[:, 2]) / Xj[:, 2]), marg)
                _, Y, clq = _backproject(cameras[j], radial, image_sizes[j], H, W, qr, qc, dq)
                Yi = Y @ cameras[i][18:27].reshape(3, 3).T + cameras[i][27:30]
                pi = _project(ci, radial, Yi)
                e2 = ((pi - pos) ** 2).sum(1)
                ok &= ~clq & (Yi[:, 2] > 0)
                marg = np.where(ok, np.minimum(marg, np.abs(e2 - max_reproj_error ** 2) / max_reproj_error ** 2), marg)
                ok &= e2 <= max_reproj_error ** 2
            ok &= ~cl
            agree += ok
            lower |= ok & (j < i)
            S[ok] += Y[ok]
        emit = ~cl & (agree >= min_num_views - 1) & ~lower
        if margins is not None:
            full = np.full(H * W, np.inf)
            full[pix] = marg
            margins.append(full.reshape(H, W))
        nv = 1 + agree[emit]
        out["points"].append(S[emit] / nv[:, None])
        out["image"].append(np.full(emit.sum(), i, np.int32))
        out["pixel"].append(pix[emit])
        out["num_views"].append(nv.astype(np.int32))
        out["score"].append(score[i].reshape(-1)[pix[emit]])
        if colors is None:
            out["colors"].append(np.full((emit.sum(), 3), 128, np.uint8))
        else:
            Hc, Wc = colors[i].shape[:2]
            out["colors"].append(colors[i][(2 * r[emit] + 1) * Hc // (2 * H), (2 * c[emit] + 1) * Wc // (2 * W)])
    cat = {"points": (np.float64, (0, 3)), "colors": (np.uint8, (0, 3)), "image": (np.int32, (0,)), "pixel": (np.int64, (0,)),
           "num_views": (np.int32, (0,)), "score": (np.float32, (0,))}
    return {k: np.concatenate(out[k]).astype(dt) if out[k] else np.zeros(sh, dt) for k, (dt, sh) in cat.items()}
