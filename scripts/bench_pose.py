"""Relative-pose throughput on one H100: `roma_b200.estimate_pose` (five-point RANSAC + recoverPose on the device) against the
reference's cv2 path on the host, on seeded synthetic two-view scenes (`synthetic.two_view_scene`) at the pose benchmarks'
threshold 0.5 px / (f0 + f1).

    python scripts/bench_pose.py [--steps 10] [--out FILE]

Prints one JSON line per configuration: device ms per pair (B = 1), batched pairs/s (B = 64), the per-kernel split of one B = 1
estimate (CUDA events), and the cv2 host time of the same inputs; then one MegaDepth-protocol step (TinyRoMa match of a
560x560 pair + 5 x (sample(5000) + estimate_pose)).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from roma_b200 import cabi, geometry, synthetic

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    lines = []

    def emit(d):
        d["gpu"] = smi
        print(json.dumps(d), flush=True)
        lines.append(d)

    def timed(fn, steps):
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps

    try:
        import cv2
    except ImportError:
        cv2 = None

    for n in (2000, 5000, 10000):
        for frac in (0.2, 0.5):
            scenes = [synthetic.two_view_scene(100 * n + b, n, frac) for b in range(64)]
            thr = 0.5 / 2400
            x0s = [torch.tensor(s["kpts0"], device=dev) for s in scenes]
            x1s = [torch.tensor(s["kpts1"], device=dev) for s in scenes]
            K0, K1 = np.stack([s["K0"] for s in scenes]), np.stack([s["K1"] for s in scenes])
            one = timed(lambda: geometry.estimate_pose(x0s[0], x1s[0], K0[0], K1[0], thr), args.steps)
            batch = timed(lambda: geometry.estimate_pose_batched(x0s, x1s, K0, K1, thr), max(1, args.steps // 2))
            # per-kernel split of one estimate
            x0, x1 = x0s[0], x1s[0]
            offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
            K = torch.tensor(np.stack([K0[0], K1[0]])[None], device=dev)
            split = {}
            orig = cabi.call

            def timed_call(fn_name, struct, **kw):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                orig(fn_name, struct, **kw)
                e1.record()
                e1.synchronize()
                split[fn_name] = split.get(fn_name, 0.0) + e0.elapsed_time(e1)
            cabi.call = timed_call
            try:
                for _ in range(3):
                    split.clear()
                    geometry._launch(x0, x1, offsets, K, n, thr, 0.99999, 1000, 0)
            finally:
                cabi.call = orig
            row = {"n": n, "outliers": frac, "device_ms_per_pair": round(one * 1e3, 3), "batched_pairs_per_s": round(64 / batch, 1),
                   "split_ms": {k.replace("romab200_pose_", ""): round(v, 3) for k, v in split.items()}}
            if cv2 is not None:
                s = scenes[0]
                K0i, K1i = np.linalg.inv(s["K0"][:2, :2]), np.linalg.inv(s["K1"][:2, :2])
                k0 = (K0i @ (s["kpts0"] - s["K0"][None, :2, 2]).T).T
                k1 = (K1i @ (s["kpts1"] - s["K1"][None, :2, 2]).T).T
                t0 = time.perf_counter()
                reps = 3
                for _ in range(reps):
                    E, m = cv2.findEssentialMat(k0, k1, np.eye(3), threshold=thr, prob=0.99999)
                    for _E in np.split(E, len(E) / 3):
                        cv2.recoverPose(_E, k0, k1, np.eye(3), 1e9, mask=m)
                row["cv2_ms_per_pair"] = round((time.perf_counter() - t0) / reps * 1e3, 1)
            emit(row)

    # MegaDepth protocol step: one match, then 5 x (sample(5000) + estimate_pose)
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    model = tiny_roma_v1_outdoor(dev, weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    g = torch.Generator().manual_seed(0)
    im_a, im_b = torch.rand(1, 3, 560, 560, generator=g).to(dev), torch.rand(1, 3, 560, 560, generator=g).to(dev)
    K = np.array([[600.0, 0, 280], [0, 600.0, 280], [0, 0, 1]])

    def protocol(pose=True):
        warp, cert = model.match(im_a, im_b)
        for _ in range(5):
            m, _c = model.sample(warp[0], cert[0], num=5000)
            if pose:
                kp = (m.double() + 1) * 280.0
                geometry.estimate_pose(kp[:, :2].contiguous(), kp[:, 2:].contiguous(), K, K, 0.5 / 1200)
    full = timed(protocol, args.steps)
    match_only = timed(lambda: protocol(False), args.steps)
    emit({"megadepth_step_ms": round(full * 1e3, 2), "match_and_sample_ms": round(match_only * 1e3, 2)})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
