#!/usr/bin/env python
"""Track triangulation on the device (`triangulate_tracks`) against the same rules on the host.

    python scripts/bench_triangulate.py [--n 50 200] [--points 40000] [--host-tracks 300] [--reps 5]

Scenes: exhaustive graphs of N images at 768 x 1024 from `synthetic.planted_cameras` (the sizes of scripts/bench_tracks.py: 40 000
scene points, each seen by an image with probability 1/2), consolidated and joined into tracks on the device, and triangulated with
the true cameras and the default options.  Device times are medians of CUDA events around whole calls (each ends in its host read
of the status word).  The host restatement (`oracle/triangulate.py`, numpy, one track at a time) runs on the first --host-tracks
tracks; its time is scaled to all tracks, and the device's ok, num_inliers and inlier must equal it on those tracks.  The 3-D
error is against the planted points.  Prints the card, a markdown table and one JSON line; writes nothing else.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle.triangulate import triangulate  # noqa: E402
from roma_b200 import Tracks, build_tracks, consolidate_matches, synthetic, triangulate_tracks  # noqa: E402

H, W = 768, 1024


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:              # nvidia-smi missing: the numbers still carry the device name
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def device_ms(fn, reps):
    """Median ms of CUDA events around fn() after one warm-up call, and the last result."""
    out = fn()
    times = []
    for _ in range(reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        out = fn()
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    return statistics.median(times), out


def row(n, points, host_tracks, reps):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(n, n, points, size=(H, W), device="cuda")
    g = consolidate_matches(pairs, m, c, sizes)
    del m, c
    tr = build_tracks(pairs, g)
    dev_ms, res = device_ms(lambda: triangulate_tracks(g, tr, K, R, t), reps)
    T, E = len(tr), int(tr.elements.shape[0])
    off = tr.track_offsets.cpu().numpy()
    lengths = np.diff(off)
    # the host restatement on the first host_tracks tracks
    S = min(host_tracks, T)
    sub = Tracks(tr.track_offsets[:S + 1], tr.elements[:off[S]], tr.kp_track, tr.num_conflicting)
    t0 = time.perf_counter()
    ref = triangulate(g.kp_offsets, g.keypoints, sub.track_offsets, sub.elements, K, R, t)
    host_ms = 1e3 * (time.perf_counter() - t0) * T / max(S, 1)
    equal = (np.array_equal(res.ok[:S].cpu().numpy(), ref["ok"]) and np.array_equal(res.num_inliers[:S].cpu().numpy(), ref["num_inliers"])
             and np.array_equal(res.inlier[:off[S]].cpu().numpy(), ref["inlier"]))
    ok = res.ok.cpu().numpy()
    pts = synthetic.track_points(tr.track_offsets, tr.elements, g.kp_offsets, g.keypoints, views, W)
    sel = ok & (pts >= 0)
    err = np.linalg.norm(res.X.cpu().numpy()[sel] - X.cpu().numpy()[pts[sel]], axis=1)
    return dict(N=n, tracks=T, elements=E, median_length=float(np.median(lengths)), max_length=int(lengths.max()),
                drawn=int((lengths * (lengths - 1) // 2 > 256).sum()), device_ms=dev_ms, host_ms=host_ms, host_tracks=S,
                speedup=host_ms / dev_ms, ok=float(ok.mean()), inliers=float(res.inlier.float().mean().item()),
                err_median=float(np.median(err)), err_p95=float(np.percentile(err, 95)), equal=bool(equal))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[50, 200])
    ap.add_argument("--points", type=int, default=40000)
    ap.add_argument("--host-tracks", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    info = card()
    rows = []
    for n in args.n:
        rows.append(row(n, args.points, args.host_tracks, args.reps))
        torch.cuda.empty_cache()
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    print("| N | tracks | elements | median / max length | tracks on drawn pairs | device ms | host (numpy) ms, scaled | speed-up | ok "
          "| inlier observations | 3-D error median / p95 | equal on host tracks |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['N']} | {r['tracks']:,} | {r['elements']:,} | {r['median_length']:g} / {r['max_length']} | {r['drawn']:,} | "
              f"{r['device_ms']:.2f} | {r['host_ms']:,.0f} | {r['speedup']:,.0f}x | {r['ok']:.4f} | {r['inliers']:.4f} | "
              f"{r['err_median']:.4f} / {r['err_p95']:.3f} | {r['equal']} ({r['host_tracks']}) |")
    print(json.dumps({"card": info, "rows": rows}))


if __name__ == "__main__":
    main()
