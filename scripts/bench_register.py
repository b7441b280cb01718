#!/usr/bin/env python
"""Absolute-pose estimation on the device (`estimate_absolute_pose_batched`, the estimator of `register_images`) against
cv2.solvePnPRansac on the host and the numpy restatement.

    python scripts/bench_register.py [--m 50 200] [--n 20000] [--outliers 0.2] [--host-images 4] [--reps 3]

Each of M cameras (intrinsics of a 768 x 1024 image, 8-10 units from a cloud in a 8 x 6 x 6 box) sees --n world points, projected
with 0.5 px noise; a fraction --outliers of the pixels is replaced by uniform ones.  The device call (max_error 12 px, confidence
0.9999, max_iters 10 000) is timed with CUDA events around the whole call and a synchronise (median of --reps after a warm-up).
cv2.solvePnPRansac (SOLVEPNP_P3P, the same threshold, confidence and iteration cap, one host thread as OpenCV schedules it) and
`oracle/absolute_pose.py` run on the first --host-images cameras; their time per camera is scaled to M.  Prints the card, a markdown
table and one JSON line; writes nothing.
"""
import argparse
import json
import math
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_triangulate import card, device_ms  # noqa: E402
from oracle import absolute_pose as oracle  # noqa: E402
from roma_b200 import estimate_absolute_pose_batched, synthetic  # noqa: E402


def scene(seed, M, n, outliers):
    rng = np.random.default_rng(seed)
    H, W = 768, 1024
    xs, Xs, Ks, Rs, ts = [], [], [], [], []
    for _ in range(M):
        K = synthetic._scene_intrinsics(rng, W, H)
        az, r, h = np.deg2rad(rng.uniform(-40, 40)), rng.uniform(8, 10), rng.uniform(-1, 1)
        C = np.array([r * math.sin(az), h, -r * math.cos(az)])
        z = -C / np.linalg.norm(C)
        x_ = np.cross([0.0, 1.0, 0.0], z)
        x_ /= np.linalg.norm(x_)
        R = np.stack((x_, np.cross(z, x_), z))
        t = -R @ C
        X = rng.uniform(-1, 1, (n, 3)) * [4.0, 3.0, 3.0]
        p = (X @ R.T + t) @ K.T
        x = p[:, :2] / p[:, 2:] + rng.normal(scale=0.5, size=(n, 2))
        out = rng.random(n) < outliers
        x[out] = rng.uniform([0, 0], [W, H], (int(out.sum()), 2))
        xs.append(x), Xs.append(X), Ks.append(K), Rs.append(R), ts.append(t)
    return xs, Xs, np.stack(Ks), Rs, ts


def rot_deg(Ra, Rb):
    return math.degrees(math.acos(min(1.0, max(-1.0, (np.trace(Ra.T @ Rb) - 1) / 2))))


def row(M, n, outliers, host_images, reps):
    xs, Xs, K, Rs, ts = scene(M, M, n, outliers)
    dx = [torch.from_numpy(v).cuda() for v in xs]
    dX = [torch.from_numpy(v).cuda() for v in Xs]
    dK = torch.from_numpy(K).cuda()
    ms, (R, t, ok, ninl, _) = device_ms(lambda: estimate_absolute_pose_batched(dx, dX, dK), reps)
    R = R.cpu().numpy()
    err = [rot_deg(R[m], Rs[m]) for m in range(M)]
    hi = min(host_images, M)
    t0 = time.perf_counter()
    cv_err = []
    for m in range(hi):
        _, rv, _, _ = cv2.solvePnPRansac(Xs[m], xs[m], K[m], None, iterationsCount=10000, reprojectionError=12.0, confidence=0.9999,
                                        flags=cv2.SOLVEPNP_P3P)
        cv_err.append(rot_deg(cv2.Rodrigues(rv)[0], Rs[m]))
    cv_s = (time.perf_counter() - t0) / hi * M
    t0 = time.perf_counter()
    for m in range(hi):
        oracle.estimate(xs[m], Xs[m], K[m], max_error=12.0, confidence=0.9999, max_iters=10000)
    or_s = (time.perf_counter() - t0) / hi * M
    return dict(M=M, n=n, outliers=outliers, device_ms=round(ms, 2), ok=int(ok.sum()), median_rot_err_deg=float(np.median(err)),
                cv2_median_rot_err_deg=float(np.median(cv_err)), cv2_host_s_scaled=round(cv_s, 2), oracle_host_s_scaled=round(or_s, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--m", type=int, nargs="+", default=[50, 200])
    ap.add_argument("--n", type=int, default=20000)
    ap.add_argument("--outliers", type=float, default=0.2)
    ap.add_argument("--host-images", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['max_sm_clock']}")
    rows = [row(M, args.n, args.outliers, args.host_images, args.reps) for M in args.m]
    print("| M | points / image | device ms | ok | median rot err (deg) | cv2 (host, s, scaled) | numpy (s, scaled) |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['M']} | {r['n']} | {r['device_ms']} | {r['ok']} | {r['median_rot_err_deg']:.4f} (cv2 {r['cv2_median_rot_err_deg']:.4f}) "
              f"| {r['cv2_host_s_scaled']} | {r['oracle_host_s_scaled']} |")
    print(json.dumps(dict(card=dev, rows=rows)))


if __name__ == "__main__":
    main()
