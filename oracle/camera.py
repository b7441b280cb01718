"""numpy statement of the SIMPLE_RADIAL camera and `roma_b200.camera.undistort_keypoints` (include/romab200.h): the same float64
operations in the same order.  The device may contract a multiply and an add into one FMA (nvcc's default), so its float64 values
can differ in the last bits and its fp32 outputs by up to 1 ulp from these; the device tests hold it to that bar."""
from __future__ import annotations

import numpy as np

ITERS = 20


def distort(xy, intrinsics):
    """Pixels of undistorted points xy [M, 2] (of the pinhole camera f, cx, cy) under SIMPLE_RADIAL intrinsics [M, 4]: the model
    applied to the normalised coordinates."""
    xy, c = np.asarray(xy, np.float64), np.asarray(intrinsics, np.float64)
    f, cx, cy, k = c[:, 0], c[:, 1], c[:, 2], c[:, 3]
    x, y = (xy[:, 0] - cx) / f, (xy[:, 1] - cy) / f
    d = 1.0 + k * (x * x + y * y)
    return np.stack((f * d * x + cx, f * d * y + cy), 1)


def undistort(keypoints, intrinsics, history=None):
    """Rules 1-4 for keypoints [M, 2] (fp32) with per-keypoint intrinsics [M, 4]: (undistorted fp32 [M, 2], clamped bool [M]).  A
    list `history` receives the Newton iterates rho [ITERS + 1, M] (NaN after a keypoint has stopped)."""
    kp, c = np.asarray(keypoints, np.float32), np.asarray(intrinsics, np.float64)
    f, cx, cy, k = c[:, 0], c[:, 1], c[:, 2], c[:, 3]
    dx, dy = kp[:, 0].astype(np.float64) - cx, kp[:, 1].astype(np.float64) - cy
    rd = np.sqrt(dx * dx + dy * dy) / f
    copy = (k == 0.0) | (rd == 0.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        clamp = ~copy & (k < 0.0) & (rd >= 2.0 / (3.0 * np.sqrt(-k * 3.0)))
        rho = np.where(clamp, 1.0 / np.sqrt(-3.0 * k), rd)
    live = ~copy & ~clamp
    hist = [np.where(live, rho, np.nan)]
    for _ in range(ITERS):
        with np.errstate(divide="ignore", invalid="ignore"):
            step = (rho * (1.0 + k * rho * rho) - rd) / (1.0 + 3.0 * k * rho * rho)
        rho = np.where(live, rho - step, rho)
        live &= step != 0.0
        hist.append(np.where(live | (step != 0.0) & ~copy & ~clamp, rho, np.nan))
    if history is not None:
        history.append(np.stack(hist))
    with np.errstate(divide="ignore", invalid="ignore"):
        s = rho / rd
    out = np.stack((cx + dx * s, cy + dy * s), 1).astype(np.float32)
    out[copy] = kp[copy]
    return out, clamp


def undistort_graph_keypoints(kp_offsets, keypoints, intrinsics):
    """`undistort_keypoints` on a match graph's keypoints: (fp32 [K, 2], number clamped)."""
    off = np.asarray(kp_offsets, np.int64)
    img = np.repeat(np.arange(off.size - 1), np.diff(off))
    out, clamp = undistort(np.asarray(keypoints, np.float32).reshape(-1, 2), np.asarray(intrinsics, np.float64)[img])
    return out, int(clamp.sum())
