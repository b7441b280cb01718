#!/usr/bin/env python
"""The match graph for structure-from-motion on the device against the same consolidation on the host.

    python scripts/bench_match_graph.py [--n 16 50] [--num 10000] [--e2e-n 8] [--reps 5]

(1) `consolidate_matches` on exhaustive graphs of N images (N (N - 1) / 2 pairs, `num` seeded samples per pair, 768 x 1024 images)
against `oracle/match_graph.py`, the numpy statement of the same rules, on the host's cores.  The device result must equal the
oracle's bit for bit.  (2) `match_graph` end to end on an exhaustive graph of `--e2e-n` synthetic images at 560 -> 864 (synthetic
weights, fp16 fast mode) against `match_pairs` + `sample_batched` + the host consolidation.  Device times are medians of CUDA events
around whole calls (each ends in a host read); host times are wall-clock medians; peak device memory is measured per call.  Prints a
markdown table and one JSON line; writes nothing else.
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

from oracle.match_graph import consolidate  # noqa: E402
from roma_b200 import consolidate_matches, roma_outdoor, synthetic  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:              # nvidia-smi missing: the numbers still carry the device name
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def device_ms(fn, reps):
    """Median ms of CUDA events around fn() and the peak device memory of one call above what was allocated before it."""
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
    peak = torch.cuda.max_memory_allocated() - base
    return statistics.median(times), peak, out


def host_ms(fn, reps):
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append(1e3 * (time.perf_counter() - t0))
    return statistics.median(times), out


def exhaustive(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def same(res, ref):
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        got, want = getattr(res, name).cpu().numpy(), ref[name]
        if got.shape != want.shape or got.tobytes() != np.ascontiguousarray(want).astype(got.dtype).tobytes():
            return False
    return True


def consolidate_rows(n_images, num, reps, host_reps):
    pairs = torch.tensor(exhaustive(n_images))
    P = pairs.shape[0]
    g = torch.Generator(device="cuda").manual_seed(n_images)
    m = torch.rand(P, num, 4, device="cuda", generator=g) * 2 - 1
    c = torch.rand(P, num, device="cuda", generator=g)
    sizes = torch.tensor([[768, 1024]] * n_images)
    dev_ms, peak, res = device_ms(lambda: consolidate_matches(pairs, m, c, sizes), reps)
    m_h, c_h = m.cpu().numpy(), c.cpu().numpy()
    cpu_ms, ref = host_ms(lambda: consolidate(pairs.numpy(), m_h, c_h, sizes.numpy()), host_reps)
    return dict(stage="consolidate_matches", N=n_images, pairs=P, num=num, samples=P * num, device_ms=dev_ms, host_ms=cpu_ms,
                speedup=cpu_ms / dev_ms, peak_mb=peak / 2 ** 20, input_mb=(m.numel() + c.numel()) * 4 / 2 ** 20,
                keypoints=int(res.keypoints.shape[0]), matches=int(res.matches.shape[0]), equal=same(res, ref))


def e2e_rows(n_images, num, reps):
    mw, dw = synthetic.make_weights(0)
    model = roma_outdoor("cuda", weights=mw, dinov2_weights=dw, coarse_res=560, upsample_res=864, amp_dtype=torch.float16)
    A, B, Ah, Bh = synthetic.make_pair((n_images + 1) // 2, 560, 864, seed=3)
    ims, his = torch.cat((A, B))[:n_images].cuda(), torch.cat((Ah, Bh))[:n_images].cuda()
    pairs = exhaustive(n_images)
    sizes = [(864, 864)] * n_images

    def device_graph():
        torch.manual_seed(0)
        return model.match_graph(ims, pairs, his, num=num, image_sizes=sizes)

    def host_graph():
        torch.manual_seed(0)
        parts = []
        model.match_pairs(ims, pairs, his, on_batch=lambda k0, w, c: parts.append([t[:, 0].cpu() for t in model.sample_batched(w, c, num)]))
        m = torch.cat([p[0] for p in parts]).numpy()
        c = torch.cat([p[1] for p in parts]).numpy()
        return consolidate(pairs, m, c, sizes)

    def dense_only():
        return model.match_pairs(ims, pairs, his, on_batch=lambda k0, w, c: None)

    for fn in (device_graph, host_graph, dense_only):       # warm-up: CUDA graphs of match_pairs and the sampler record here
        fn()
        fn()
    dev_ms, dev_peak, res = device_ms(device_graph, reps)
    host_total, host_peak, ref = device_ms(host_graph, reps)
    dense_ms, _, _ = device_ms(dense_only, reps)
    return dict(stage="match_graph", N=n_images, pairs=len(pairs), num=num, device_ms=dev_ms, host_pipeline_ms=host_total,
                match_pairs_only_ms=dense_ms, device_peak_mb=dev_peak / 2 ** 20, host_pipeline_peak_mb=host_peak / 2 ** 20,
                keypoints=int(res.keypoints.shape[0]), matches=int(res.matches.shape[0]), equal=same(res, ref))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[16, 50])
    ap.add_argument("--num", type=int, default=10000)
    ap.add_argument("--e2e-n", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=1)
    args = ap.parse_args()
    info = card()
    rows = [consolidate_rows(n, args.num, args.reps, args.host_reps) for n in args.n]
    e2e = e2e_rows(args.e2e_n, args.num, args.reps) if args.e2e_n else None
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}")
    print("| N | pairs | samples | device ms | host (numpy) ms | speed-up | device peak MB (input MB) | keypoints | matches | equal |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['N']} | {r['pairs']} | {r['samples']:,} | {r['device_ms']:.1f} | {r['host_ms']:.0f} | {r['speedup']:.0f}x | "
              f"{r['peak_mb']:.0f} ({r['input_mb']:.0f}) | {r['keypoints']:,} | {r['matches']:,} | {r['equal']} |")
    if e2e:
        print()
        print("| N | pairs | match_graph ms | match_pairs + sample_batched + host ms | match_pairs alone ms | peak MB (device / host pipeline) "
              "| equal |")
        print("|---|---|---|---|---|---|---|")
        print(f"| {e2e['N']} | {e2e['pairs']} | {e2e['device_ms']:.0f} | {e2e['host_pipeline_ms']:.0f} | {e2e['match_pairs_only_ms']:.0f} | "
              f"{e2e['device_peak_mb']:.0f} / {e2e['host_pipeline_peak_mb']:.0f} | {e2e['equal']} |")
    print(json.dumps({"card": info, "consolidate": rows, "end_to_end": e2e}))


if __name__ == "__main__":
    main()
