"""Self-calibration on the device: what it costs in bundle adjustment, and how far from the truth a focal prior may be.

    python scripts/bench_self_calibration.py [--n 50 200] [--points 40000] [--reps 3] [--recon-n 30] [--recon-points 1500]

Table 1, `bundle_adjust` per trial with camera_model="PINHOLE" against "SIMPLE_RADIAL".

Scenes: those of scripts/bench_bundle.py (exhaustive graphs of N images at 768 x 1024 from `synthetic.planted_cameras` with 40 000
scene points, perturbed cameras, tracks triangulated with them).  SIMPLE_RADIAL starts from (f, cx, cy, k) = (K_00, K_02, K_12, 0)
with every focal length and k free; PINHOLE is the unchanged call.  Both run to max_iterations = 10 trials with
function_tolerance = 0, so they do the same number of trials.  The per-trial split comes from a run that synchronises after
every C-ABI call, split into bench_bundle.py's phases; the whole call is timed with CUDA events (median of --reps after a warm-up).  The
reduced system grows from 6N to 8N rows, and the camera-block kernel's work per observation from 36 to 64 S entries.  Prints the
card, a markdown table and one JSON line; writes nothing else.

Table 2, `reconstruct(..., intrinsics=prior, refine_intrinsics=True)` on a `planted_cameras(..., radial=(-0.05, 0.05))` scene of
--recon-n images at 384 x 512 (--recon-points points, no outliers), from a prior whose every f is off by the given fraction
(alternating signs) with k = 0: registered images, the median and worst focal error and worst k error of the registered images,
camera errors after a 7-DoF alignment of the centres (worst rotation and centre), and the time of one call (host clock around a
synchronised call, after a warm-up call on the same scene).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import torch  # noqa: E402

from bench_bundle import H, PHASE, W  # noqa: E402
from bench_triangulate import card, device_ms  # noqa: E402
import numpy as np  # noqa: E402

from roma_b200 import build_tracks, bundle_adjust, cabi, consolidate_matches, reconstruct, synthetic, triangulate_tracks  # noqa: E402


def rows(n, points, reps):
    pairs, m, c, sizes, views, K, Rt, tt, X = synthetic.planted_cameras(n, n, points, size=(H, W), device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    R, t = synthetic.perturb_cameras(n, Rt, tt, 0.3, 0.05)
    pts = triangulate_tracks(g, tr, K, R, t, max_error=20.0)
    intr = torch.stack((K[:, 0, 0], K[:, 0, 2], K[:, 1, 2], torch.zeros_like(K[:, 0, 0])), 1)
    out = []
    for model, cams in (("PINHOLE", K), ("SIMPLE_RADIAL", intr)):
        kw = dict(max_iterations=10, function_tolerance=0.0, camera_model=model)
        ms, res = device_ms(lambda: bundle_adjust(g, tr, pts, cams, R, t, **kw), reps)
        split, _ = phase_split_kw((g, tr, pts, cams, R, t), kw)
        trials = int(res.accepted.size)
        out.append({"N": n, "model": model, "tracks": len(tr), "observations": int(pts.inlier.sum()), "trials": trials,
                    "kept": int(res.accepted.sum()), "total_ms": ms, "ms_per_trial": {k: v / max(trials, 1) for k, v in split.items()},
                    "F_before": float(res.cost[0]), "F_after": float(res.cost[-1])})
    return out


def phase_split_kw(args, kw):
    """bench_bundle.phase_split with keyword arguments: ms per phase over one call, each C-ABI call followed by a synchronise."""
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


def recon_rows(n, points, errors=(0.0, 0.03, 0.10, 0.20)):
    pairs, m, c, sizes, views, intr, Rt, tt, X = synthetic.planted_cameras(7, n, points, size=(384, 512), radial=(-0.05, 0.05), device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    tr = build_tracks(pairs, g)
    truth = intr.cpu().numpy()
    out = []
    for e in errors:
        prior = truth.copy()
        prior[:, 0] *= 1 + e * np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
        prior[:, 3] = 0.0
        reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rec = reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True)
        torch.cuda.synchronize()
        ms = 1e3 * (time.perf_counter() - t0)
        reg = rec.registered.cpu().numpy()
        row = {"prior_f_error": e, "registered": int(reg.sum()), "N": n, "termination": rec.termination, "ms": ms,
               "rounds": len(rec.rounds)}
        if reg.sum() >= 3:
            fin = rec.intrinsics.cpu().numpy()[reg]
            ferr = np.abs(fin[:, 0] / truth[reg, 0] - 1)
            R, t = rec.R.cpu().numpy()[reg], rec.t.cpu().numpy()[reg]
            row.update(f_err_median=float(np.median(ferr)), f_err_max=float(ferr.max()), k_err_max=float(np.abs(fin[:, 3] - truth[reg, 3]).max()),
                       cam_err=worst_camera_errors(R, t, Rt.cpu().numpy()[reg], tt.cpu().numpy()[reg]))
        out.append(row)
    return out


def worst_camera_errors(R, t, Rt, tt):
    """Worst rotation error (degrees) and centre error after a 7-DoF alignment of the centres to the truth."""
    C, Ct = -np.einsum("nji,nj->ni", R, t), -np.einsum("nji,nj->ni", Rt, tt)
    mc, mt = C.mean(0), Ct.mean(0)
    U, S, Vt = np.linalg.svd((Ct - mt).T @ (C - mc) / len(C))
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / ((C - mc) ** 2).sum(1).mean()
    dR = np.einsum("nij,kj,nlk->nil", R, Q, Rt)
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    return [float(ang.max()), float(np.linalg.norm(s * C @ Q.T + mt - s * Q @ mc - Ct, axis=1).max())]


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
    print("| N | model | observations | trials (kept) | total ms | ms/trial: linearize + cameras, cholesky, step | F before -> after |")
    print("|---|---|---|---|---|---|---|")
    for r in out:
        sp = r["ms_per_trial"]
        print(f"| {r['N']} | {r['model']} | {r['observations']} | {r['trials']} ({r['kept']}) | {r['total_ms']:.1f} | "
              f"{sp.get('linearize + cameras', 0):.2f}, {sp.get('cholesky', 0):.2f}, {sp.get('step', 0):.2f} | "
              f"{r['F_before']:.4g} -> {r['F_after']:.4g} |")
    rec = recon_rows(a.recon_n, a.recon_points)
    print("| prior f error | registered | f error median / max | k error max | worst rotation error deg | worst centre error | ms |")
    print("|---|---|---|---|---|---|---|")
    for r in rec:
        if "cam_err" in r:
            print(f"| {r['prior_f_error']:.0%} | {r['registered']} / {r['N']} | {r['f_err_median']:.2e} / {r['f_err_max']:.2e} | "
                  f"{r['k_err_max']:.2e} | {r['cam_err'][0]:.4f} | {r['cam_err'][1]:.5f} | {r['ms']:.0f} |")
        else:
            print(f"| {r['prior_f_error']:.0%} | {r['registered']} / {r['N']} ({r['termination']}) | - | - | - | - | {r['ms']:.0f} |")
    print(json.dumps({"card": dev, "rows": out, "reconstruct": rec}))


if __name__ == "__main__":
    main()
