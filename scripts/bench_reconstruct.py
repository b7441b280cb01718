#!/usr/bin/env python
"""Reconstruction without known cameras on the device (`reconstruct`): the two-view initialisation and the register -> triangulate
-> adjust loop, against the same loop with the numpy oracles on the host.

    python scripts/bench_reconstruct.py [--n 50 200] [--points 40000] [--host-n 10] [--host-points 1500]

Scenes: exhaustive graphs of N images at 768 x 1024 from `synthetic.planted_cameras` with --points scene points, 0.5 px noise and
20 % outlier samples, through consolidate_matches -> verify_matches -> build_tracks on the device; no camera is given to
`reconstruct`.  Each scene runs once after a warm-up on a small scene.  The stages are timed with a host clock around each call and
a synchronise (each ends in host reads anyway): the initialisation's pose estimate (gather and five-point RANSAC) and its score
(romab200_twoview_score), then per round triangulation (both calls), bundle adjustment and registration.  Camera errors are the
median and max over the registered images after a 7-DoF alignment of their centres to the truth.  The host comparison runs
`oracle/mapper.py`'s loop at --host-n images only.  Prints the card, a markdown table and one JSON line; writes nothing.
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

from bench_triangulate import card  # noqa: E402
from oracle import mapper as oracle  # noqa: E402
from roma_b200 import build_tracks, consolidate_matches, geometry, mapper, synthetic, verify_matches  # noqa: E402

TIMES = []


def _timed(name, fn):
    """fn, recording (name, seconds) of every call with a synchronise on both sides."""
    def wrap(*a, **k):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a, **k)
        torch.cuda.synchronize()
        TIMES.append((name, time.perf_counter() - t0))
        return out
    return wrap


for _name, _mod, _attr in (("pose", geometry, "_launch"), ("gather", mapper, "_gather"), ("score", mapper, "_score"),
                           ("triangulate", mapper, "triangulate_tracks"), ("ba", mapper, "bundle_adjust"),
                           ("register", mapper, "register_images")):
    setattr(_mod, _attr, _timed(_name, getattr(_mod, _attr)))


def scene(n, points, H=768, W=1024):
    pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(n, n, points, size=(H, W), outlier_frac=0.2, device="cuda")
    g = verify_matches(pairs, consolidate_matches(pairs, m, c, sizes))[0]
    return pairs, g, build_tracks(pairs, g), K, R, t


def errors(Rr, tr, Rg, tg, reg):
    """(median, max) rotation error in degrees and (median, max) centre error after a 7-DoF alignment of the centres."""
    C, Ct = -np.einsum("nji,nj->ni", Rr[reg], tr[reg]), -np.einsum("nji,nj->ni", Rg[reg], tg[reg])
    mc, mt = C.mean(0), Ct.mean(0)
    A, B = C - mc, Ct - mt
    U, S, Vt = np.linalg.svd(B.T @ A / len(C))
    D = np.eye(3)
    D[2, 2] = np.sign(np.linalg.det(U @ Vt))
    Q = U @ D @ Vt
    s = np.trace(np.diag(S) @ D) / (A * A).sum(1).mean()
    dR = np.einsum("nij,kj,nlk->nil", Rr[reg], Q, Rg[reg])
    ang = np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))
    cen = np.linalg.norm(s * C @ Q.T + mt - s * Q @ mc - Ct, axis=1)
    return float(np.median(ang)), float(ang.max()), float(np.median(cen)), float(cen.max())


def run(n, points):
    pairs, g, tr, K, R, t = scene(n, points)
    TIMES.clear()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rec = mapper.reconstruct(pairs, g, tr, K)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    stages = list(TIMES)
    init = {k: sum(s for name, s in stages[:3] if name == k) for k in ("gather", "pose", "score")}
    groups = []
    for name, s in stages[3:]:                             # a round: triangulate, ba, triangulate, then register unless all are in
        if name == "triangulate" and (not groups or groups[-1][-1][0] == "register"):
            groups.append([])
        groups[-1].append((name, s))
    rounds = []
    for r, part in zip(rec.rounds, groups):
        rounds.append(dict(added=len(r["added"]), triangulate_s=sum(s for name, s in part if name == "triangulate"),
                           ba_s=sum(s for name, s in part if name == "ba"), register_s=sum(s for name, s in part if name == "register"),
                           ba_termination=r["ba_termination"]))
    reg = np.flatnonzero(rec.registered.cpu().numpy())
    med_r, max_r, med_c, max_c = errors(rec.R.cpu().numpy(), rec.t.cpu().numpy(), R.cpu().numpy(), t.cpu().numpy(), reg)
    return dict(n=n, points=points, pairs=len(pairs), tracks=len(tr), init_pose_s=init["gather"] + init["pose"], init_score_s=init["score"],
                candidates=len(rec.init.pair_index), rounds=rounds, total_s=total, registered=int(reg.size),
                termination=rec.termination, rot_err_deg=(med_r, max_r), centre_err=(med_c, max_c))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[50, 200])
    ap.add_argument("--points", type=int, default=40000)
    ap.add_argument("--host-n", type=int, default=10)
    ap.add_argument("--host-points", type=int, default=1500)
    args = ap.parse_args()
    info = card()
    print(f"card: {info}")
    run(10, 1500)                                          # warm-up: module loads and allocator
    rows = [run(n, args.points) for n in args.n]
    pairs, g, tr, K, R, t = scene(args.host_n, args.host_points)
    TIMES.clear()
    t0 = time.perf_counter()
    mapper.reconstruct(pairs, g, tr, K)
    torch.cuda.synchronize()
    dev_small = time.perf_counter() - t0
    t0 = time.perf_counter()
    ref = oracle.reconstruct(pairs.cpu().numpy(), g.kp_offsets, g.keypoints, g.match_offsets, g.matches, tr.track_offsets, tr.elements, K)
    host_small = time.perf_counter() - t0
    print("| N | tracks | init pose s | init score s | rounds (images added) | triangulate s / round | BA s / round | register s / round "
          "| total s | registered | rot err median / max deg | centre err median / max |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        rd = r["rounds"]
        print(f"| {r['n']} | {r['tracks']} | {r['init_pose_s']:.3f} | {r['init_score_s'] * 1e3:.2f} ms | {len(rd)} ({', '.join(str(x['added']) for x in rd)}) "
              f"| {', '.join(f'{x['triangulate_s']:.2f}' for x in rd)} | {', '.join(f'{x['ba_s']:.2f}' for x in rd)} "
              f"| {', '.join(f'{x['register_s']:.2f}' for x in rd)} | {r['total_s']:.2f} | {r['registered']} / {r['n']} "
              f"| {r['rot_err_deg'][0]:.3f} / {r['rot_err_deg'][1]:.3f} | {r['centre_err'][0]:.4f} / {r['centre_err'][1]:.4f} |")
    print(f"host oracle loop at N = {args.host_n}, {args.host_points} points: {host_small:.1f} s ({len(ref['registered'])} registered) "
          f"vs device {dev_small:.2f} s")
    print(json.dumps(dict(card=info, scenes=rows, host=dict(n=args.host_n, points=args.host_points, oracle_s=host_small, device_s=dev_small,
                                                            registered=len(ref["registered"])))))


if __name__ == "__main__":
    main()
