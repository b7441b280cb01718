"""Fundamental-matrix throughput on one H100: `roma_b200.find_fundamental` (seven-point MAGSAC++ on the device) against
cv2.findFundamentalMat(USAC_MAGSAC) on the host, on seeded two-view scenes (`synthetic.two_view_scene`, 0.5 px noise) at the
arguments of the reference's usage example (README.md:62-78: threshold 0.2, confidence 0.999999, maxIters 10000).

    python scripts/bench_fundamental.py [--steps 10] [--out FILE]

Prints one JSON line per configuration: device ms per pair (B = 1), batched pairs/s (B = 64), the per-kernel split of one B = 1
estimate (CUDA events), and the cv2 host time of the same inputs; then one step of the usage example (TinyRoMa match of a 560x560
pair + sample(5000) + one F) with the device F and with cv2's.
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

    thr, conf, iters = 0.2, 0.999999, 10000
    for n in (2000, 5000, 10000):
        for frac in (0.2, 0.5, 0.7):
            scenes = [synthetic.two_view_scene(100 * n + b, n, frac) for b in range(64)]
            x0s = [torch.tensor(s["kpts0"], device=dev) for s in scenes]
            x1s = [torch.tensor(s["kpts1"], device=dev) for s in scenes]
            one = timed(lambda: geometry.find_fundamental(x0s[0], x1s[0], geometry.USAC_MAGSAC, thr, conf, iters), args.steps)
            batch = timed(lambda: geometry.find_fundamental_batched(x0s, x1s, geometry.USAC_MAGSAC, thr, conf, iters), max(1, args.steps // 2))
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
                    buf = geometry._fund_launch(x0s[0], x1s[0], offsets, n, thr, conf, iters, 0)
            finally:
                cabi.call = orig
            row = {"n": n, "outliers": frac, "device_ms_per_pair": round(one * 1e3, 3), "batched_pairs_per_s": round(64 / batch, 1),
                   "iterations": int(buf["state"][0, 0]), "split_ms": {k.replace("romab200_fund_", ""): round(v, 3) for k, v in split.items()}}
            if cv2 is not None:
                reps = 3
                t0 = time.perf_counter()
                for _ in range(reps):
                    cv2.findFundamentalMat(scenes[0]["kpts0"], scenes[0]["kpts1"], cv2.USAC_MAGSAC, thr, conf, iters)
                row["cv2_ms_per_pair"] = round((time.perf_counter() - t0) / reps * 1e3, 2)
            emit(row)

    # the usage example (README.md:62-78): one match, sample(5000), to pixel coordinates, one fundamental matrix
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
            F, mask = geometry.find_fundamental(kp[:, :2].contiguous(), kp[:, 2:].contiguous(), geometry.USAC_MAGSAC, thr, conf, iters)
        elif mode == "cv2":
            k = kp.cpu().numpy()
            F, mask = cv2.findFundamentalMat(k[:, :2], k[:, 2:], cv2.USAC_MAGSAC, thr, conf, iters)
        torch.cuda.synchronize()
    warp, cert = model.match(im_a, im_b)
    m, _c = model.sample(warp[0], cert[0], num=5000)
    kp = ((m + 1) * 280.0).contiguous()
    fund_alone = timed(lambda: geometry.find_fundamental(kp[:, :2].contiguous(), kp[:, 2:].contiguous(), geometry.USAC_MAGSAC, thr, conf, iters),
                       args.steps)
    row = {"gist_step_ms": round(timed(lambda: protocol("device"), args.steps) * 1e3, 2), "find_fundamental_alone_ms": round(fund_alone * 1e3, 2),
           "match_and_sample_ms": round(timed(lambda: protocol(None), args.steps) * 1e3, 2)}
    if cv2 is not None:
        row["gist_step_cv2_ms"] = round(timed(lambda: protocol("cv2"), args.steps) * 1e3, 2)
    emit(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
