"""Homography throughput on one H100: `roma_b200.find_homography` (four-point RANSAC + refinement on the device) against
cv2.findHomography(RANSAC) on the host, on seeded synthetic planar scenes (`synthetic.planar_scene`) at the HPatches harness's
settings (3 px threshold for 480 px images, confidence 0.99999).

    python scripts/bench_homography.py [--steps 10] [--out FILE]

Prints one JSON line per configuration: device ms per pair (B = 1), batched pairs/s (B = 64), the per-kernel split of one B = 1
estimate (CUDA events), and the cv2 host time of the same inputs; then one HPatches-protocol step (TinyRoMa match of a 560x560
pair + sample(5000) + find_homography) against the same step with cv2.
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

    conf = 0.99999
    for n in (2000, 5000, 10000):
        for frac in (0.2, 0.5, 0.7):
            scenes = [synthetic.planar_scene(100 * n + b, n, frac) for b in range(64)]
            srcs = [torch.tensor(s["src"], dtype=torch.float32, device=dev) for s in scenes]
            dsts = [torch.tensor(s["dst"], dtype=torch.float32, device=dev) for s in scenes]
            one = timed(lambda: geometry.find_homography(srcs[0], dsts[0], geometry.RANSAC, 3.0, confidence=conf), args.steps)
            batch = timed(lambda: geometry.find_homography_batched(srcs, dsts, geometry.RANSAC, 3.0, confidence=conf), max(1, args.steps // 2))
            offsets = torch.tensor([0, n], dtype=torch.int64, device=dev)
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
                    geometry._homog_launch(srcs[0], dsts[0], offsets, n, geometry.RANSAC, 3.0, conf, 2000, 0)
            finally:
                cabi.call = orig
            row = {"n": n, "outliers": frac, "device_ms_per_pair": round(one * 1e3, 3), "batched_pairs_per_s": round(64 / batch, 1),
                   "split_ms": {k.replace("romab200_homography_", ""): round(v, 3) for k, v in split.items()}}
            if cv2 is not None:
                s32, d32 = scenes[0]["src"].astype(np.float32), scenes[0]["dst"].astype(np.float32)
                reps = 3
                t0 = time.perf_counter()
                for _ in range(reps):
                    cv2.findHomography(s32, d32, cv2.RANSAC, 3.0, confidence=conf)
                row["cv2_ms_per_pair"] = round((time.perf_counter() - t0) / reps * 1e3, 2)
            emit(row)

    # HPatches protocol step (hpatches_sequences_homog_benchmark.py:72-91): one match, sample(5000), one homography
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    model = tiny_roma_v1_outdoor(dev, weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    g = torch.Generator().manual_seed(0)
    im_a, im_b = torch.rand(1, 3, 560, 560, generator=g).to(dev), torch.rand(1, 3, 560, 560, generator=g).to(dev)

    def protocol(mode):
        warp, cert = model.match(im_a, im_b)
        m, _c = model.sample(warp[0], cert[0], num=5000)
        kp = (m + 1) * 280.0
        if mode == "device":
            geometry.find_homography(kp[:, :2].contiguous(), kp[:, 2:].contiguous(), geometry.RANSAC, 3.0, confidence=conf)
        elif mode == "cv2":
            k = kp.cpu().numpy()
            cv2.findHomography(k[:, :2], k[:, 2:], cv2.RANSAC, 3.0, confidence=conf)
    row = {"hpatches_step_ms": round(timed(lambda: protocol("device"), args.steps) * 1e3, 2),
           "match_and_sample_ms": round(timed(lambda: protocol(None), args.steps) * 1e3, 2)}
    if cv2 is not None:
        row["hpatches_step_cv2_ms"] = round(timed(lambda: protocol("cv2"), args.steps) * 1e3, 2)
    emit(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
