#!/usr/bin/env python
"""Bundle adjustment on the device (`bundle_adjust`) against the same rules on the host.

    python scripts/bench_bundle.py [--n 50 200] [--points 40000] [--host-tracks 300] [--reps 3]

Scenes: the triangulation benchmark's (scripts/bench_triangulate.py): exhaustive graphs of N images at 768 x 1024 from
`synthetic.planted_cameras` with 40 000 scene points, consolidated and joined into tracks on the device; the cameras are perturbed
by 0.3 degrees and 0.05 units (`perturb_cameras`) and the tracks triangulated with them (`triangulate_tracks`, max_error 20 px).
The whole call is timed with CUDA events (median of --reps after a warm-up).  The per-trial split comes from a separate run that
synchronises after every C-ABI call: linearize + cameras, cholesky, and step.  Camera errors are medians after a 7-DoF alignment of
the centres to the truth.  The host restatement (`oracle/bundle.py`) runs the same problem restricted to the first --host-tracks
tracks; its time per trial is scaled to all tracks.  `scipy.optimize.least_squares` is not run at these sizes.  Prints the
card, a markdown table and one JSON line; writes nothing else.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_triangulate import card, device_ms  # noqa: E402
from oracle.bundle import bundle_adjust as oracle_ba  # noqa: E402
from roma_b200 import build_tracks, bundle_adjust, cabi, consolidate_matches, synthetic, triangulate_tracks  # noqa: E402

H, W = 768, 1024
PHASE = {"romab200_ba_linearize": "linearize + cameras", "romab200_ba_cameras": "linearize + cameras", "romab200_ba_cholesky": "cholesky",
         "romab200_ba_step": "step"}


def camera_errors(R, t, Rt, tt):
    R, t, Rt, tt = (np.asarray(v.cpu() if hasattr(v, "cpu") else v) for v in (R, t, Rt, tt))
    C, Ct = -np.einsum("nji,nj->ni", R, t), -np.einsum("nji,nj->ni", Rt, tt)
    mc, mt = C.mean(0), Ct.mean(0)
    U, S, Vt = np.linalg.svd((Ct - mt).T @ (C - mc) / len(C))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / ((C - mc) ** 2).sum(1).mean()
    dR = np.einsum("nij,kj,nlk->nil", R, Q, Rt)
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    return float(np.median(ang)), float(np.median(np.linalg.norm(s * C @ Q.T + mt - s * Q @ mc - Ct, axis=1)))


def phase_split(args):
    """ms per phase summed over one call, each C-ABI call followed by a synchronise."""
    acc = {}
    orig = cabi.call

    def timed(fn, *a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        orig(fn, *a, **k)
        torch.cuda.synchronize()
        if fn in PHASE:
            acc[PHASE[fn]] = acc.get(PHASE[fn], 0.0) + 1e3 * (time.perf_counter() - t0)

    cabi.call = timed
    try:
        res = bundle_adjust(*args)
    finally:
        cabi.call = orig
    return acc, res


def host_subset(g, tr, pts, K, R, t, n_tracks):
    off = tr.track_offsets.cpu().numpy()
    T = min(n_tracks, off.size - 1)
    E = off[T]
    t0 = time.perf_counter()
    ref = oracle_ba(g.kp_offsets, g.keypoints, off[:T + 1], tr.elements[:E], pts.X[:T], pts.ok[:T], pts.inlier[:E], K, R, t, max_iterations=3)
    per_trial = (time.perf_counter() - t0) / max(ref["accepted"].size, 1)
    return per_trial * (off.size - 1) / T


def row(n, points, host_tracks, reps):
    pairs, m, c, sizes, views, K, Rt, tt, X = synthetic.planted_cameras(n, n, points, size=(H, W), device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    R, t = synthetic.perturb_cameras(n, Rt, tt, 0.3, 0.05)
    pts = triangulate_tracks(g, tr, K, R, t, max_error=20.0)
    args = (g, tr, pts, K, R, t)
    ms, res = device_ms(lambda: bundle_adjust(*args), reps)
    split, _ = phase_split(args)
    trials = int(res.accepted.size)
    r0, c0 = camera_errors(R, t, Rt, tt)
    r1, c1 = camera_errors(res.R, res.t, Rt, tt)
    host_s = host_subset(g, tr, pts, K.cpu().numpy(), R.cpu().numpy(), t.cpu().numpy(), host_tracks)
    out = {"N": n, "tracks": len(tr), "observations": int(pts.inlier.sum()), "trials": trials, "kept": int(res.accepted.sum()),
           "termination": res.termination, "total_ms": ms, "ms_per_trial": {k: v / max(trials, 1) for k, v in split.items()},
           "F_before": float(res.cost[0]), "F_after": float(res.cost[-1]), "rot_err_deg": [r0, r1], "centre_err": [c0, c1],
           "host_s_per_trial_scaled": host_s}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[50, 200])
    ap.add_argument("--points", type=int, default=40000)
    ap.add_argument("--host-tracks", type=int, default=300)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['max_sm_clock']}")
    rows = [row(n, a.points, a.host_tracks, a.reps) for n in a.n]
    print("| N | tracks | observations | trials (kept) | total ms | ms/trial: linearize + cameras, cholesky, step | F before -> after | "
          "rotation error deg | centre error | host s/trial (scaled) |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        sp = r["ms_per_trial"]
        print(f"| {r['N']} | {r['tracks']} | {r['observations']} | {r['trials']} ({r['kept']}) | {r['total_ms']:.1f} | "
              f"{sp.get('linearize + cameras', 0):.2f}, {sp.get('cholesky', 0):.2f}, {sp.get('step', 0):.2f} | "
              f"{r['F_before']:.4g} -> {r['F_after']:.4g} | {r['rot_err_deg'][0]:.3f} -> {r['rot_err_deg'][1]:.4f} | "
              f"{r['centre_err'][0]:.4f} -> {r['centre_err'][1]:.5f} | {r['host_s_per_trial_scaled']:.1f} |")
    print(json.dumps({"card": dev, "rows": rows}))


if __name__ == "__main__":
    main()
