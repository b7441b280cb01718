"""Batched match sampling on one H100: `sample_batched` against the `sample()` loop it replaces, and the MegaDepth-protocol step built
on it.

    python scripts/bench_sample.py [--reps 5] [--sizes tiny roma] [--batches 1 8 64] [--protocol-batches 1 8 32] [--out FILE]

(a) For TinyRoMa 560x560 warps with num 5000 and RoMa 864x1728 symmetric warps (864 x 3456 pixels) with num 10000, B pairs and R
    draws per pair: the loop `for b, r: sample(M[b], C[b], num)` and `sample_batched(M, C, num, repeats=R)` alternate in one process
    after warm-up; each call is timed with CUDA events (medians), with the peak device memory it allocates beyond its inputs and
    whether the two outputs are bit-equal after the same seed.
(b) The MegaDepth-1500 protocol step for B TinyRoMa 560x560 pairs: per pair `match`, 5 x `sample(5000)` and 5 x `estimate_pose`
    (as in bench_pose.py), against `match` of the batch -> `sample_batched(repeats=5)` -> `estimate_pose_batched` over 5B problems.
    Each phase is timed with CUDA events.
Prints one JSON line per configuration, with the card's name, power limit and maximum SM clock.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", nargs="+", default=["tiny", "roma"])
    ap.add_argument("--batches", nargs="+", type=int, default=[1, 8, 64])
    ap.add_argument("--repeats", nargs="+", type=int, default=[1, 5])
    ap.add_argument("--protocol-batches", nargs="+", type=int, default=[1, 8, 32])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from roma_b200 import geometry, roma_outdoor, synthetic, tiny_roma_v1_outdoor

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    lines = []

    def emit(d):
        d["gpu"] = smi
        print(json.dumps(d), flush=True)
        lines.append(d)

    def event_ms(fn):
        """(result, device ms, peak bytes allocated beyond what was allocated before the call)"""
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        e1.synchronize()
        return out, e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base

    xf = synthetic.xfeat_standin()
    tiny = tiny_roma_v1_outdoor(dev, weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    models = {"tiny": (tiny, 560, 560, 5000)}
    if "roma" in args.sizes:
        w = synthetic.make_weights(0)
        models["roma"] = (roma_outdoor(dev, weights=w[0], dinov2_weights=w[1], coarse_res=112, upsample_res=168, amp_dtype=torch.float32),
                          864, 1728 * 2, 10000)

    def warps(B, H, W, seed):
        """Smooth seeded warps with a certainty map that is high in some regions and low in others (generated on the device)."""
        g = torch.Generator(device=dev).manual_seed(seed)
        ys, xs = torch.linspace(-1 + 1 / H, 1 - 1 / H, H, device=dev), torch.linspace(-1 + 1 / W, 1 - 1 / W, W, device=dev)
        grid = torch.stack((xs[None].expand(H, W), ys[:, None].expand(H, W)), -1)
        M = torch.empty(B, H, W, 4, device=dev)
        C = torch.empty(B, H, W, device=dev)
        for b in range(B):
            phase = torch.rand(2, device=dev, generator=g) * 6
            M[b, ..., :2] = grid
            M[b, ..., 2:] = (grid + 0.1 * torch.sin(3 * grid + phase) + 0.01 * torch.randn(H, W, 2, device=dev, generator=g)).clamp(-1, 1)
            C[b] = torch.sigmoid(4 * torch.randn(H, W, device=dev, generator=g) + 3 * grid[..., 0])
        return M, C

    # (a) the sample() loop against sample_batched
    for name in args.sizes:
        model, H, W, num = models[name]
        M_all, C_all = warps(max(args.batches), H, W, 0)
        for B in args.batches:
            M, C = M_all[:B], C_all[:B]
            for R in args.repeats:
                def loop():
                    outs = [model.sample(M[b], C[b], num) for b in range(B) for _ in range(R)]
                    return torch.stack([m for m, _ in outs]), torch.stack([c for _, c in outs])

                def batched():
                    return model.sample_batched(M, C, num, repeats=R)
                for fn in (loop, batched, loop, batched, loop, batched):       # warm-up, CUDA-graph capture of the single-pair chain
                    fn()
                t_loop, t_batch, mem_loop, mem_batch = [], [], 0, 0
                for _ in range(args.reps):
                    _, t, mem = event_ms(loop)
                    t_loop.append(t)
                    mem_loop = max(mem_loop, mem)
                    _, t, mem = event_ms(batched)
                    t_batch.append(t)
                    mem_batch = max(mem_batch, mem)
                torch.manual_seed(99)
                ref = loop()
                torch.manual_seed(99)
                got = batched()
                equal = torch.equal(got[0].reshape(ref[0].shape), ref[0]) and torch.equal(got[1].reshape(ref[1].shape), ref[1])
                ml, mb = statistics.median(t_loop), statistics.median(t_batch)
                emit({"model": name, "warp": [H, W], "num": num, "B": B, "R": R, "loop_ms": round(ml, 3), "batched_ms": round(mb, 3),
                      "speedup": round(ml / mb, 3), "loop_ms_per_draw": round(ml / (B * R), 3), "batched_ms_per_draw": round(mb / (B * R), 3),
                      "loop_peak_mb": round(mem_loop / 2 ** 20, 1), "batched_peak_mb": round(mem_batch / 2 ** 20, 1), "bit_equal": equal})
        del M_all, C_all
        torch.cuda.empty_cache()

    # (b) the MegaDepth-protocol step: match, five samples of each pair, a pose per sample
    K = np.array([[600.0, 0, 280], [0, 600.0, 280], [0, 0, 1]])
    thr = 0.5 / 1200
    for B in args.protocol_batches:
        g = torch.Generator().manual_seed(B)
        im_a, im_b = torch.rand(B, 3, 560, 560, generator=g).to(dev), torch.rand(B, 3, 560, 560, generator=g).to(dev)

        def per_pair():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ph = [0.0, 0.0, 0.0]
            for b in range(B):
                ev[0].record()
                warp, cert = tiny.match(im_a[b:b + 1], im_b[b:b + 1])
                ev[1].record()
                ms = [tiny.sample(warp[0], cert[0], num=5000)[0] for _ in range(5)]
                ev[2].record()
                for m in ms:
                    kp = (m.double() + 1) * 280.0
                    geometry.estimate_pose(kp[:, :2].contiguous(), kp[:, 2:].contiguous(), K, K, thr)
                ev[3].record()
                ev[3].synchronize()
                for i in range(3):
                    ph[i] += ev[i].elapsed_time(ev[i + 1])
            return ph

        def batched():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            warp, cert = tiny.match(im_a, im_b)
            ev[1].record()
            m, _ = tiny.sample_batched(warp, cert, 5000, repeats=5)
            ev[2].record()
            kp = ((m.double() + 1) * 280.0).reshape(B * 5, -1, 4)
            geometry.estimate_pose_batched([k[:, :2].contiguous() for k in kp], [k[:, 2:].contiguous() for k in kp], K, K, thr)
            ev[3].record()
            ev[3].synchronize()
            return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]
        for fn in (per_pair, batched, per_pair, batched, per_pair, batched):
            fn()
        loop_ph, batch_ph = [], []
        for _ in range(args.reps):
            loop_ph.append(per_pair())
            batch_ph.append(batched())
        lm = [statistics.median(p[i] for p in loop_ph) for i in range(3)]
        bm = [statistics.median(p[i] for p in batch_ph) for i in range(3)]
        emit({"protocol": "megadepth_tiny_560", "B": B, "loop_step_ms": round(sum(lm), 2), "batched_step_ms": round(sum(bm), 2),
              "loop_ms_per_pair": round(sum(lm) / B, 3), "batched_ms_per_pair": round(sum(bm) / B, 3),
              "loop_phase_ms": {"match": round(lm[0], 2), "sample": round(lm[1], 2), "pose": round(lm[2], 2)},
              "batched_phase_ms": {"match": round(bm[0], 2), "sample": round(bm[1], 2), "pose": round(bm[2], 2)}})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(lines, f, indent=1)


if __name__ == "__main__":
    main()
