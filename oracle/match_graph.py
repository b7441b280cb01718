"""numpy statement of `roma_b200.consolidate_matches` (include/romab200.h, INTEGRATION.md): sampled dense matches of many pairs ->
per-image keypoints (one per occupied pixel cell, raster-order ids) and one-to-one mutual-best matches per pair.  Plain sorts and
unique runs, no device code; the device result is pinned to this bit for bit."""
from __future__ import annotations

import numpy as np


def consolidate(pairs, matches, certainty, image_sizes, cell_size=1, min_certainty=0.0):
    """pairs [P, 2], matches [P, n, 4] (or [P, ..., 4]) and certainty [P, n] (or [P, ...]) fp32, image_sizes [N, 2] (H, W).  Returns a
    dict of numpy arrays: kp_offsets [N + 1], keypoints [K, 2], kp_scores [K], match_offsets [P + 1], matches [M, 2] int32 (local ids),
    match_scores [M], and sid [P, n, 2] int32 (the keypoint id of every sample side, -1 when ignored)."""
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    P = pairs.shape[0]
    c = np.asarray(certainty, np.float32)
    c = c.reshape(P, -1) if P else c.reshape(0, 0)
    m = np.asarray(matches, np.float32).reshape(P, c.shape[1], 4)
    n = c.shape[1]
    sizes = np.asarray(image_sizes, np.int64).reshape(-1, 2)
    N = sizes.shape[0]
    cs = int(cell_size)

    img = np.broadcast_to(pairs[:, None, :], (P, n, 2))                    # side 0 in image i, side 1 in image j
    H, W = sizes[img, 0], sizes[img, 1]
    u, v = m[..., 0::2], m[..., 1::2]
    cc = np.broadcast_to(c[..., None], (P, n, 2))
    with np.errstate(all="ignore"):
        x = (W / 2).astype(np.float32) * (u + np.float32(1))               # fp32, as matcher.py:_to_pixel_coordinates
        y = (H / 2).astype(np.float32) * (v + np.float32(1))
        valid = (cc > np.float32(min_certainty)) & np.isfinite(cc) & np.isfinite(u) & np.isfinite(v)
        cx = np.clip(np.floor(x), 0, W - 1)
        cy = np.clip(np.floor(y), 0, H - 1)
    cx = np.where(valid, cx, 0).astype(np.int64) // cs
    cy = np.where(valid, cy, 0).astype(np.int64) // cs
    cell = cy * (-(-W // cs)) + cx
    g = np.arange(P * n * 2, dtype=np.int64).reshape(P, n, 2)              # (k * n + s) * 2 + side

    vi, vc, vg, vcert = img[valid], cell[valid], g[valid], cc[valid]
    vx, vy = x[valid], y[valid]
    order = np.lexsort((vg, -vcert, vc, vi))                               # by image, cell, certainty descending, g ascending
    si, sc = vi[order], vc[order]
    head = np.ones(order.size, bool)
    head[1:] = (si[1:] != si[:-1]) | (sc[1:] != sc[:-1])
    win = order[head]                                                      # winners in (image, cell) order = raster order per image
    counts = np.bincount(vi[win], minlength=N)
    kp_offsets = np.zeros(N + 1, np.int64)
    kp_offsets[1:] = np.cumsum(counts)
    run = np.cumsum(head) - 1                                              # global keypoint of every sorted side
    gid = np.empty(order.size, np.int64)
    gid[order] = run
    sid = np.full((P, n, 2), -1, np.int32)
    sid[valid] = (gid - kp_offsets[vi]).astype(np.int32)

    match_offsets = np.zeros(P + 1, np.int64)
    out_m, out_s = [], []
    for k in range(P):
        a, b = sid[k, :, 0].astype(np.int64), sid[k, :, 1].astype(np.int64)
        ok = (a >= 0) & (b >= 0)
        s = np.nonzero(ok)[0]
        a, b, w = a[ok], b[ok], c[k, ok]
        best_a = _best(a, w, s)                                            # per distinct a (ascending): the sample of its best b
        best_b = _best(b, w, s)
        ub, ab = b[best_b], a[best_b]                                      # b ascending -> best_a(b)
        bb = b[best_a]
        keep = ab[np.searchsorted(ub, bb)] == a[best_a]
        sel = best_a[keep]
        out_m.append(np.stack((a[sel], b[sel]), 1).astype(np.int32))
        out_s.append(w[sel])
        match_offsets[k + 1] = match_offsets[k] + sel.size
    return dict(kp_offsets=kp_offsets, keypoints=np.stack((vx[win], vy[win]), 1).reshape(-1, 2).astype(np.float32),
                kp_scores=vcert[win].astype(np.float32), match_offsets=match_offsets,
                matches=np.concatenate(out_m).reshape(-1, 2) if out_m else np.zeros((0, 2), np.int32),
                match_scores=np.concatenate(out_s).astype(np.float32) if out_s else np.zeros(0, np.float32), sid=sid)


def _best(key, w, s):
    """Index (into key) of the largest certainty w of each distinct key, ties to the smallest sample s; in ascending key order."""
    order = np.lexsort((s, -w, key))
    sk = key[order]
    head = np.ones(order.size, bool)
    head[1:] = sk[1:] != sk[:-1]
    return order[head]
