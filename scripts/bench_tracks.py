#!/usr/bin/env python
"""Feature tracks on the device (`build_tracks`) against the same rules on the host.

    python scripts/bench_tracks.py [--n 16 50 200] [--uniform-n 16 50] [--reps 5]

(1) Planted scenes: exhaustive graphs of N images at 768 x 1024 from `synthetic.planted_views` (40 000 scene points, each seen by an
image with probability 1/2, so about 10 000 inlier samples per pair), with outlier_frac 0 and 0.2, consolidated on the device by
`consolidate_matches`.  (2) Uniform random samples: the generator of scripts/bench_match_graph.py (10 000 samples per pair), whose
graph holds one giant conflicting component.  On each graph, `build_tracks` against `oracle/tracks.py` (numpy and scipy) on the
host's cores, whose result the device must equal bit for bit.  Device times are medians of CUDA events around whole calls (each ends
in its host read); host times are one wall-clock run on arrays already on the host; peak device memory is measured per call above
what was allocated before it.  Recall is the fraction of planted tracks with two or more views returned exactly.  Prints a markdown
table and one JSON line; writes nothing else.
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

from oracle.tracks import tracks  # noqa: E402
from roma_b200 import build_tracks, consolidate_matches, synthetic  # noqa: E402

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
    """Median ms of CUDA events around fn() (after one warm-up call) and the peak device memory of one call above what was
    allocated before it."""
    fn()
    times = []
    for _ in range(reps):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        out = fn()
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
        del out
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return statistics.median(times), torch.cuda.max_memory_allocated() - base, out


def same(res, ref):
    for name in ("track_offsets", "elements", "kp_track"):
        got, want = getattr(res, name).cpu().numpy(), ref[name]
        if got.shape != want.shape or got.tobytes() != np.ascontiguousarray(want).astype(got.dtype).tobytes():
            return False
    return res.num_conflicting == ref["num_conflicting"]


def histogram(res):
    """Track lengths in the bins 2, 3, 4-7, 8-15, 16-31, 32-63, 64+."""
    lengths = torch.diff(res.track_offsets).cpu().numpy()
    edges = [2, 3, 4, 8, 16, 32, 64, np.iinfo(np.int64).max]
    counts = np.histogram(lengths, bins=edges)[0]
    names = ["2", "3", "4-7", "8-15", "16-31", "32-63", "64+"]
    return {n: int(c) for n, c in zip(names, counts)}


def row(kind, n_images, pairs, g, reps, views=None, outlier_frac=None):
    dev_ms, peak, res = device_ms(lambda: build_tracks(pairs, g), reps)
    host = {k: getattr(g, k).cpu().numpy() for k in ("kp_offsets", "match_offsets", "matches", "match_scores")}
    t0 = time.perf_counter()
    ref = tracks(pairs.cpu().numpy(), host)
    host_ms = 1e3 * (time.perf_counter() - t0)
    recall = None
    if views is not None:
        planted = synthetic.planted_tracks(views)
        found = synthetic.track_cells(res.track_offsets, res.elements, g.kp_offsets, g.keypoints, W)
        recall = len(planted & found) / len(planted)
    K, M = int(g.kp_offsets[-1]), int(g.match_offsets[-1])
    return dict(kind=kind, N=n_images, outlier_frac=outlier_frac, pairs=int(pairs.shape[0]), keypoints=K, matches=M, device_ms=dev_ms,
                host_ms=host_ms, speedup=host_ms / dev_ms, peak_mb=peak / 2 ** 20, tracks=len(res), elements=int(res.elements.shape[0]),
                lengths=histogram(res), num_conflicting=res.num_conflicting, largest_component=int(np.bincount(ref["root"]).max()),
                recall=recall, equal=same(res, ref))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[16, 50, 200])
    ap.add_argument("--uniform-n", type=int, nargs="+", default=[16, 50])
    ap.add_argument("--points", type=int, default=40000)
    ap.add_argument("--num", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    info = card()
    rows = []
    for n in args.n:
        for f in (0.0, 0.2):
            pairs, m, c, sizes, views = synthetic.planted_views(n, n, args.points, size=(H, W), outlier_frac=f, device="cuda")
            g = consolidate_matches(pairs, m, c, sizes)
            del m, c
            rows.append(row("planted", n, pairs, g, args.reps, views, f))
            del g
            torch.cuda.empty_cache()
    for n in args.uniform_n:
        pairs = torch.triu_indices(n, n, 1).T.contiguous()
        gen = torch.Generator(device="cuda").manual_seed(n)
        m = torch.rand(pairs.shape[0], args.num, 4, device="cuda", generator=gen) * 2 - 1
        c = torch.rand(pairs.shape[0], args.num, device="cuda", generator=gen)
        g = consolidate_matches(pairs, m, c, torch.tensor([[H, W]] * n))
        del m, c
        rows.append(row("uniform", n, pairs, g, args.reps))
        del g
        torch.cuda.empty_cache()
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    print("| samples | N | outliers | keypoints | matches | device ms | host (numpy + scipy) ms | speed-up | device peak MB | tracks | elements "
          "| lengths 2 / 3 / 4-7 / 8-15 / 16-31 / 32-63 / 64+ | conflicting | largest component | recall | equal |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        rec = "–" if r["recall"] is None else f"{r['recall']:.3f}"
        out = "–" if r["outlier_frac"] is None else f"{r['outlier_frac']:g}"
        print(f"| {r['kind']} | {r['N']} | {out} | {r['keypoints']:,} | {r['matches']:,} | {r['device_ms']:.2f} | {r['host_ms']:.0f} | "
              f"{r['speedup']:.0f}x | {r['peak_mb']:.0f} | {r['tracks']:,} | {r['elements']:,} | {' / '.join(str(v) for v in r['lengths'].values())} | "
              f"{r['num_conflicting']:,} | {r['largest_component']:,} | {rec} | {r['equal']} |")
    print(json.dumps({"card": info, "rows": rows}))


if __name__ == "__main__":
    main()
