"""Shared cameras on the device: what folding the camera system costs in bundle adjustment, and what one shared (f, k) buys in
`reconstruct` over per-image self-calibration.

    python scripts/bench_shared_intrinsics.py [--n 50 200] [--points 40000] [--reps 3] [--recon-n 30] [--recon-points 1500]

Table 1, `bundle_adjust(camera_model="SIMPLE_RADIAL")` per trial, per-image intrinsics against one camera group
(camera_ids = zeros).  Scenes: those of scripts/bench_bundle.py (exhaustive graphs of N images at 768 x 1024 from
`synthetic.planted_cameras` with 40 000 points, perturbed cameras, tracks triangulated with them), drawn with camera_ids = zeros so
that every image has the same intrinsics and both runs start from the same (f, cx, cy, 0).  Both run max_iterations = 10 trials
with function_tolerance = 0.  The per-trial split (camera blocks = linearize + cameras, fold = fold + unfold, Cholesky, step)
comes from a run that synchronises after every C-ABI call; the whole call is timed with CUDA events (median of --reps after a
warm-up).  The shared run's Cholesky has order 6N + 2 instead of 8N.

Table 2, `reconstruct(..., intrinsics=prior, refine_intrinsics=True)` on a single-camera `planted_cameras(..., radial=(-0.05, 0.05),
spread=True, camera_ids=zeros)` scene of --recon-n images at 384 x 512, from a prior whose f is off by the given fraction with
k = 0, per-image against camera_ids = zeros: registered images, the median and worst focal error of the registered images, the k
error, camera errors after a 7-DoF alignment of the centres, and the time of one call (host clock around a synchronised call,
after a warm-up call).  Prints the card, markdown tables and one JSON line; writes nothing else.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_bundle import H, W  # noqa: E402
from bench_self_calibration import worst_camera_errors  # noqa: E402
from bench_triangulate import card, device_ms  # noqa: E402

from roma_b200 import build_tracks, bundle_adjust, cabi, consolidate_matches, reconstruct, synthetic, triangulate_tracks  # noqa: E402

PHASE = {"romab200_ba_linearize": "camera blocks", "romab200_ba_cameras": "camera blocks", "romab200_ba_fold": "fold",
         "romab200_ba_unfold": "fold", "romab200_ba_cholesky": "cholesky", "romab200_ba_groups_cholesky": "cholesky",
         "romab200_ba_step": "step"}


def phase_split(args, kw):
    """ms per phase over one call, each C-ABI call followed by a synchronise."""
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
        res = bundle_adjust(*args, **kw)
    finally:
        cabi.call = orig
    return acc, res


def rows(n, points, reps):
    ids = np.zeros(n, np.int64)
    pairs, m, c, sizes, views, K, Rt, tt, X = synthetic.planted_cameras(n, n, points, size=(H, W), camera_ids=ids, device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    R, t = synthetic.perturb_cameras(n, Rt, tt, 0.3, 0.05)
    pts = triangulate_tracks(g, tr, K, R, t, max_error=20.0)
    intr = torch.stack((K[:, 0, 0], K[:, 0, 2], K[:, 1, 2], torch.zeros_like(K[:, 0, 0])), 1)
    out = []
    for name, extra in (("per-image", {}), ("one group", dict(camera_ids=ids))):
        kw = dict(max_iterations=10, function_tolerance=0.0, camera_model="SIMPLE_RADIAL", **extra)
        ms, res = device_ms(lambda: bundle_adjust(g, tr, pts, intr, R, t, **kw), reps)
        split, _ = phase_split((g, tr, pts, intr, R, t), kw)
        trials = int(res.accepted.size)
        out.append({"N": n, "intrinsics": name, "observations": int(pts.inlier.sum()), "trials": trials, "kept": int(res.accepted.sum()),
                    "total_ms": ms, "ms_per_trial": {k: v / max(trials, 1) for k, v in split.items()},
                    "F_before": float(res.cost[0]), "F_after": float(res.cost[-1])})
    return out


def recon_rows(n, points, errors=(0.0, 0.03, 0.10, 0.20), seed=7):
    ids = np.zeros(n, np.int64)
    pairs, m, c, sizes, views, intr, Rt, tt, X = synthetic.planted_cameras(seed, n, points, size=(384, 512), radial=(-0.05, 0.05),
                                                                           spread=True, camera_ids=ids, device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    truth = intr.cpu().numpy()
    out = []
    for e in errors:
        prior = truth.copy()
        prior[:, 0] *= 1 + e
        prior[:, 3] = 0.0
        for name, extra in (("per-image", {}), ("shared", dict(camera_ids=ids))):
            reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True, **extra)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rec = reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True, **extra)
            torch.cuda.synchronize()
            ms = 1e3 * (time.perf_counter() - t0)
            reg = rec.registered.cpu().numpy()
            row = {"prior_f_error": e, "intrinsics": name, "registered": int(reg.sum()), "N": n, "termination": rec.termination, "ms": ms}
            if reg.sum() >= 3:
                fin = rec.intrinsics.cpu().numpy()[reg]
                ferr = np.abs(fin[:, 0] / truth[reg, 0] - 1)
                R, t = rec.R.cpu().numpy()[reg], rec.t.cpu().numpy()[reg]
                row.update(f_err_median=float(np.median(ferr)), f_err_max=float(ferr.max()),
                           k_err_max=float(np.abs(fin[:, 3] - truth[reg, 3]).max()),
                           cam_err=worst_camera_errors(R, t, Rt.cpu().numpy()[reg], tt.cpu().numpy()[reg]))
            out.append(row)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[50, 200])
    ap.add_argument("--points", type=int, default=40000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--recon-n", type=int, default=30)
    ap.add_argument("--recon-points", type=int, default=1500)
    a = ap.parse_args()
    dev = card()
    print(f"card: {dev['name']}, power limit {dev['power_limit']}, max SM clock {dev['max_sm_clock']}")
    out = [r for n in a.n for r in rows(n, a.points, a.reps)]
    print("| N | intrinsics | observations | trials (kept) | total ms | ms/trial: camera blocks, fold, cholesky, step | F before -> after |")
    print("|---|---|---|---|---|---|---|")
    for r in out:
        sp = r["ms_per_trial"]
        print(f"| {r['N']} | {r['intrinsics']} | {r['observations']} | {r['trials']} ({r['kept']}) | {r['total_ms']:.1f} | "
              f"{sp.get('camera blocks', 0):.2f}, {sp.get('fold', 0):.2f}, {sp.get('cholesky', 0):.2f}, {sp.get('step', 0):.2f} | "
              f"{r['F_before']:.4g} -> {r['F_after']:.4g} |")
    rec = recon_rows(a.recon_n, a.recon_points)
    print("| prior f error | intrinsics | registered | f error median / max | k error max | worst rotation error deg | worst centre error | ms |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rec:
        if "cam_err" in r:
            print(f"| {r['prior_f_error']:.0%} | {r['intrinsics']} | {r['registered']} / {r['N']} | {r['f_err_median']:.2e} / "
                  f"{r['f_err_max']:.2e} | {r['k_err_max']:.2e} | {r['cam_err'][0]:.4f} | {r['cam_err'][1]:.5f} | {r['ms']:.0f} |")
        else:
            print(f"| {r['prior_f_error']:.0%} | {r['intrinsics']} | {r['registered']} / {r['N']} ({r['termination']}) | - | - | - | - | "
                  f"{r['ms']:.0f} |")
    print(json.dumps({"card": dev, "rows": out, "reconstruct": rec}))


if __name__ == "__main__":
    main()
