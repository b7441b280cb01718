#!/usr/bin/env python
"""Geometric verification of a match graph on the device (`verify_matches`) against the same work written out by hand and against
cv2 on the host.

    python scripts/bench_verify.py [--n 16 50 200] [--outliers 0 0.2] [--points 20000] [--reps 5] [--cv2-n 16 50]

Scenes: exhaustive graphs of N images at 768 x 1024 from `synthetic.planted_cameras` (`--points` scene points, each seen by an image
with probability 1/2 where it projects into it, 0.5 px noise), with outlier_frac 0 and 0.2, consolidated on the device by
`consolidate_matches` at cell_size 1.
- Device: `verify_matches` with its defaults, the median of `--reps` calls from CUDA events, with the number of estimator chunks and
  the peak device memory of one call above what was allocated before it.
- By hand: the five steps a user writes without it (the offsets to the host, two lists of P point tensors, one
  `find_fundamental_batched` call, torch compaction of the masks into match offsets, a new MatchGraph), timed the same way,
  alternated with the device call in this process; "did not fit" when it runs out of device memory.  Both give the same graph.
- cv2: a `cv2.findFundamentalMat(..., cv2.USAC_MAGSAC, 2.0, 0.999, 10000)` loop over the pairs on the host, one wall-clock run, at
  the N of `--cv2-n` ("not run" elsewhere).
- Quality: the share of planted inlier matches kept and of outlier matches removed, and `build_tracks` before and after verification:
  recall (the share of planted tracks with two or more views returned exactly), conflicting components and the largest component
  (the longest track with drop_conflicts=False).
Prints progress to stderr, one JSON line per scene, then the card, a markdown table and one JSON line; writes nothing else.
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

from roma_b200 import MatchGraph, USAC_MAGSAC, build_tracks, consolidate_matches, find_fundamental_batched, synthetic, verify_matches  # noqa: E402
from roma_b200.match_graph import WORKSPACE_BYTES  # noqa: E402
from roma_b200.verify import plan_chunks  # noqa: E402

H, W = 768, 1024


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:              # nvidia-smi missing: the numbers still carry the device name
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), out


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base, out


def by_hand(pairs, g, threshold=2.0, confidence=0.999, max_iters=10000):
    """The verification a user writes without `verify_matches`."""
    kp_off, m_off = g.kp_offsets.tolist(), g.match_offsets.tolist()                      # 1. the offsets to the host
    x0, x1 = [], []                                                                      # 2. two lists of P point tensors
    for k, (i, j) in enumerate(pairs.tolist()):
        m = g.matches[m_off[k]:m_off[k + 1]].long()
        x0.append(g.keypoints[kp_off[i] + m[:, 0]].double())
        x1.append(g.keypoints[kp_off[j] + m[:, 1]].double())
    F, ok, masks = find_fundamental_batched(x0, x1, USAC_MAGSAC, threshold, confidence, max_iters)   # 3. one batched estimate
    mask = torch.cat([mk.view(-1) for mk in masks]).bool()                               # 4. compaction into match offsets
    counts = torch.tensor([mk.shape[0] for mk in masks], device=mask.device)
    pair_of = torch.repeat_interleave(torch.arange(len(masks), device=mask.device), counts)
    inliers = torch.zeros(len(masks), dtype=torch.int64, device=mask.device).index_add_(0, pair_of, mask.long())
    accepted = ok & (inliers >= 15)
    keep = mask & accepted[pair_of]
    offsets = torch.zeros(len(masks) + 1, dtype=torch.int64, device=mask.device)
    offsets[1:] = torch.where(accepted, inliers, 0).cumsum(0)
    return MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, offsets, g.matches[keep], g.match_scores[keep])   # 5. a new graph


def cv2_loop(pairs, g):
    import cv2

    kp, xy = g.kp_offsets.cpu().numpy(), g.keypoints.cpu().numpy().astype(np.float64)
    mo, m = g.match_offsets.cpu().numpy(), g.matches.cpu().numpy().astype(np.int64)
    pts = [(xy[kp[i] + m[mo[k]:mo[k + 1], 0]], xy[kp[j] + m[mo[k]:mo[k + 1], 1]]) for k, (i, j) in enumerate(pairs.cpu().numpy())]
    t0 = time.perf_counter()
    for a, b in pts:
        if len(a) >= 7:
            cv2.findFundamentalMat(a, b, cv2.USAC_MAGSAC, 2.0, 0.999, 10000)
    return 1e3 * (time.perf_counter() - t0)


def labels(pairs, g, views):
    """Per match of g: True when its two keypoints are one planted point's views (cell_size 1)."""
    kp, xy = g.kp_offsets.cpu().numpy(), g.keypoints.cpu().numpy()
    mo, m = g.match_offsets.cpu().numpy(), g.matches.cpu().numpy().astype(np.int64)
    v = views.cpu().numpy()
    cell = np.floor(xy[:, 1]).astype(np.int64) * W + np.floor(xy[:, 0]).astype(np.int64)
    p_idx, img = np.nonzero(v >= 0)
    keys = img * (H * W) + v[p_idx, img]
    order = np.argsort(keys)
    keys, point = keys[order], p_idx[order]

    def point_of(i, c):
        q = i * (H * W) + c
        at = np.minimum(np.searchsorted(keys, q), keys.size - 1)
        return np.where(keys[at] == q, point[at], -1)

    pr = pairs.cpu().numpy()
    pair_of = np.repeat(np.arange(pr.shape[0]), np.diff(mo))
    i, j = pr[pair_of, 0], pr[pair_of, 1]
    pa, pb = point_of(i, cell[kp[i] + m[:, 0]]), point_of(j, cell[kp[j] + m[:, 1]])
    return (pa >= 0) & (pa == pb)


def kept_mask(g, out):
    """Per match of g: whether the verified graph `out` keeps it (ids < 2^20 per image, matches one-to-one per pair)."""
    def keys(h):
        mo, m = h.match_offsets.cpu().numpy(), h.matches.cpu().numpy().astype(np.int64)
        assert m.size == 0 or m.max() < 1 << 20
        return np.repeat(np.arange(mo.size - 1), np.diff(mo)) << 40 | m[:, 0] << 20 | m[:, 1]
    return np.isin(keys(g), keys(out))


def track_stats(pairs, g, views):
    t = build_tracks(pairs, g)
    planted = synthetic.planted_tracks(views)
    found = synthetic.track_cells(t.track_offsets, t.elements, g.kp_offsets, g.keypoints, W)
    loose = build_tracks(pairs, g, drop_conflicts=False)
    largest = int(torch.diff(loose.track_offsets).max()) if len(loose) else 0
    return dict(recall=len(planted & found) / len(planted), conflicting=t.num_conflicting, largest=largest)


def same(a, b):
    return all(torch.equal(getattr(a, n), getattr(b, n)) for n in ("match_offsets", "matches", "match_scores"))


def stage(what, t0):
    print(f"  N={what}: {time.perf_counter() - t0:.1f} s", file=sys.stderr, flush=True)


def row(n, f, args):
    t0 = time.perf_counter()
    pairs, m, c, sizes, views = synthetic.planted_cameras(n, n, args.points, size=(H, W), outlier_frac=f, device="cuda")[:5]
    g = consolidate_matches(pairs, m, c, sizes)
    del m, c
    torch.cuda.empty_cache()
    P, M = int(pairs.shape[0]), int(g._m_off[-1])
    ns = [e - b for b, e in zip(g._m_off, g._m_off[1:])]
    stage(f"{n} outliers={f} scene", t0)
    dev_peak, (out, geom) = peak(lambda: verify_matches(pairs, g))
    hand_ok, hand_peak, equal = True, None, None
    try:
        hand_peak, hand = peak(lambda: by_hand(pairs, g))
        equal = same(out, hand)
        del hand
    except torch.OutOfMemoryError:
        hand_ok = False
    torch.cuda.empty_cache()
    dev_t, hand_t = [], []
    for _ in range(args.reps):                                        # alternated in one process
        dev_t.append(timed(lambda: verify_matches(pairs, g))[0])
        if hand_ok:
            hand_t.append(timed(lambda: by_hand(pairs, g))[0])
    stage(f"{n} outliers={f} timings", t0)
    cv2_ms = None
    if n in args.cv2_n:
        try:
            cv2_ms = cv2_loop(pairs, g)
        except ImportError:
            cv2_ms = "cv2 missing"
    stage(f"{n} outliers={f} cv2", t0)
    inl = labels(pairs, g, views)
    kept = kept_mask(g, out)
    before, after = track_stats(pairs, g, views), track_stats(pairs, out, views)
    return dict(N=n, outlier_frac=f, pairs=P, keypoints=int(g._kp_off[-1]), matches=M, kept=int(out._m_off[-1]),
                accepted=int(geom.accepted.sum()), chunks=len(plan_chunks(ns, WORKSPACE_BYTES)), device_ms=statistics.median(dev_t),
                device_peak_mb=dev_peak / 2 ** 20, hand_ms=statistics.median(hand_t) if hand_ok else None,
                hand_peak_mb=hand_peak / 2 ** 20 if hand_ok else None, hand_equal=equal, cv2_ms=cv2_ms,
                inlier_kept=float(kept[inl].mean()), outlier_removed=float((~kept[~inl]).mean()) if (~inl).any() else None,
                before=before, after=after)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[16, 50, 200])
    ap.add_argument("--points", type=int, default=20000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--outliers", type=float, nargs="+", default=[0.0, 0.2])
    ap.add_argument("--cv2-n", type=int, nargs="*", default=[16, 50])
    args = ap.parse_args()
    info = card()
    rows = []
    for n in args.n:
        for f in args.outliers:
            rows.append(row(n, f, args))
            print(json.dumps(rows[-1]), flush=True)
            torch.cuda.empty_cache()
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    print("| N | outliers | pairs | matches | kept | accepted | chunks | device ms | device peak MB | by hand ms | by hand peak MB | cv2 ms "
          "| inliers kept | outliers removed | recall before / after | conflicting before / after | largest component before / after |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        hand = "did not fit" if r["hand_ms"] is None else f"{r['hand_ms']:.0f}"
        hand_mb = "–" if r["hand_peak_mb"] is None else f"{r['hand_peak_mb']:,.0f}"
        cv = "not run" if r["cv2_ms"] is None else (r["cv2_ms"] if isinstance(r["cv2_ms"], str) else f"{r['cv2_ms']:,.0f}")
        out = "–" if r["outlier_removed"] is None else f"{r['outlier_removed']:.4f}"
        b, a = r["before"], r["after"]
        print(f"| {r['N']} | {r['outlier_frac']:g} | {r['pairs']:,} | {r['matches']:,} | {r['kept']:,} | {r['accepted']:,} | {r['chunks']} | "
              f"{r['device_ms']:.0f} | {r['device_peak_mb']:,.0f} | {hand} | {hand_mb} | {cv} | {r['inlier_kept']:.4f} | {out} | "
              f"{b['recall']:.3f} / {a['recall']:.3f} | {b['conflicting']:,} / {a['conflicting']:,} | {b['largest']:,} / {a['largest']:,} |")
    print(json.dumps({"card": info, "rows": rows}))


if __name__ == "__main__":
    main()
