"""Dense reconstruction benchmark: `triangulate_warps` and `fuse_depth_maps` on `synthetic.depth_views` scenes at RoMa's 864 x 864
output grid with exhaustive pairs, against the numpy oracle (oracle/dense.py) timed on a subset of pairs / images and scaled to the
whole set; then `dense_cloud` end to end against `match_pairs` alone, to show what the dense step adds to matching.

The ground-truth warps come from `get_gt_warp` chunk by chunk (not timed), so no more than one chunk of warps is held.  Device
times are CUDA events around each call; the oracle runs on the host between them.  Accuracy is the relative depth error of every
emitted point against the planted depth of its pixel.  Prints one JSON line per measurement.

    python scripts/bench_dense.py [--sizes 16 50] [--grid 864] [--chunk 8] [--e2e 8]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import dense as oracle  # noqa: E402
from roma_b200 import dense, roma_outdoor, synthetic  # noqa: E402


def _gpu():
    name = torch.cuda.get_device_name()
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
        pl = pl.strip().splitlines()[0]
    except Exception:            # noqa: BLE001 - the power limit is reported when nvidia-smi can read it
        pl = "unknown"
    return name, pl


def bench_scene(N, grid, chunk, oracle_pairs, oracle_images):
    t0 = time.time()
    views = synthetic.depth_views(0, N, (grid, grid))
    gen_s = time.time() - t0
    pairs = [(i, j) for i in range(N) for j in range(i + 1, N)]
    P = len(pairs)
    K, R, t, sizes = views["K"], views["R"], views["t"], views["image_sizes"]
    table = dense.camera_table(K.numpy(), R.numpy(), t.numpy())
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    dm, tri_ms, ora_tri_s, ora_done = None, 0.0, 0.0, 0
    sub = set(np.linspace(0, P - 1, oracle_pairs).round().astype(int).tolist())
    for k0 in range(0, P, chunk):
        warp, cert = synthetic.depth_view_warps(views, pairs[k0:k0 + chunk], "cuda")
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dm = dense.triangulate_warps(pairs, warp, cert, K, R, t, sizes, first_pair=k0, depth_maps=dm)
        b.record()
        b.synchronize()
        tri_ms += a.elapsed_time(b)
        for k in range(k0, min(P, k0 + chunk)):
            if k in sub:                         # the oracle alternates with the device on the same warps
                w, c = warp[k - k0:k - k0 + 1].cpu().numpy(), cert[k - k0:k - k0 + 1].cpu().numpy()
                s = time.perf_counter()
                oracle.triangulate_warps(np.array(pairs), w, c, sizes.numpy(), table, np.ones(N, bool), first_pair=k)
                ora_tri_s += time.perf_counter() - s
                ora_done += 1
        del warp, cert
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    colors = [views["colors"][i].cuda() for i in range(N)]
    dense.fuse_depth_maps(dm, pairs, K, R, t, sizes, colors=colors)           # warm-up
    torch.cuda.synchronize()
    fuse_ms = []
    for _ in range(3):
        a.record()
        cloud = dense.fuse_depth_maps(dm, pairs, K, R, t, sizes, colors=colors)
        b.record()
        b.synchronize()
        fuse_ms.append(a.elapsed_time(b))
    peak = torch.cuda.max_memory_allocated() - base
    # the fusion oracle on the first images, scaled by pixels with depth
    d_np, s_np = dm.depth.cpu().numpy(), dm.score.cpu().numpy()
    keep = np.zeros(N, bool)
    keep[:oracle_images] = True
    s = time.perf_counter()
    oracle.fuse_depth_maps(np.where(keep[:, None, None], d_np, 0), s_np, np.array(pairs), sizes.numpy(), table, np.ones(N, bool))
    ora_fuse_s = (time.perf_counter() - s) * (d_np > 0).sum() / max(1, (d_np[:oracle_images] > 0).sum())
    img, pix = cloud.image.long().cpu(), cloud.pixel.cpu()
    z = (torch.einsum("mij,mj->mi", R[img], cloud.points.cpu()) + t[img])[:, 2]
    gt = views["depth"].reshape(N, -1)[img, pix].double()
    rel = ((z - gt).abs() / gt).numpy()
    return {"images": N, "pairs": P, "grid": grid, "generate_s": round(gen_s, 1),
            "triangulate_ms_per_pair": round(tri_ms / P, 4), "triangulate_oracle_ms_per_pair": round(1e3 * ora_tri_s / ora_done, 1),
            "fuse_ms": round(float(np.median(fuse_ms)), 2), "fuse_oracle_ms_scaled": round(1e3 * ora_fuse_s, 0),
            "peak_MiB": round(peak / 2 ** 20, 1), "pixels_with_depth": int((d_np > 0).sum()), "points": int(cloud.points.shape[0]),
            "rel_depth_error_median": float(np.median(rel)), "rel_depth_error_max": float(rel.max()),
            "within_max_depth_error": float((rel <= 0.01).mean())}


def bench_e2e(N, reps):
    from roma_b200.synthetic import make_weights

    mw, dw = make_weights(0)
    model = roma_outdoor("cuda", weights=mw, dinov2_weights=dw, amp_dtype=torch.float16)
    g = torch.Generator().manual_seed(0)
    ims = torch.rand(N, 3, 560, 560, generator=g).cuda()
    his = torch.rand(N, 3, 864, 864, generator=g).cuda()
    views = synthetic.depth_views(1, N, (64, 64))
    K, R, t = views["K"] * 864 / 64, views["R"], views["t"]
    K[:, 2, 2] = 1.0
    sizes = [(864, 864)] * N
    pairs = [(i, j) for i in range(N) for j in range(i + 1, N)]

    def run_match():
        model.match_pairs(ims, pairs, his, max_batch=8, on_batch=lambda *a: None)

    def run_cloud():
        return model.dense_cloud(ims, pairs, K, R, t, image_sizes=sizes, images_high_res=his, max_batch=8)

    run_match(), run_cloud()
    torch.cuda.synchronize()
    times = {"match_pairs": [], "dense_cloud": []}
    for _ in range(reps):                   # alternating, so both see the same machine state
        for name, fn in (("match_pairs", run_match), ("dense_cloud", run_cloud)):
            torch.cuda.synchronize()
            s = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[name].append(time.perf_counter() - s)
    m, c = np.median(times["match_pairs"]), np.median(times["dense_cloud"])
    return {"e2e_images": N, "pairs": len(pairs), "match_pairs_s": round(float(m), 4), "dense_cloud_s": round(float(c), 4),
            "dense_overhead_ms_per_pair": round(1e3 * (c - m) / len(pairs), 3),
            "spread_match_pairs_s": [round(float(min(times["match_pairs"])), 4), round(float(max(times["match_pairs"])), 4)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[16, 50])
    ap.add_argument("--grid", type=int, default=864)
    ap.add_argument("--chunk", type=int, default=8)
    ap.add_argument("--oracle-pairs", type=int, default=2)
    ap.add_argument("--oracle-images", type=int, default=1)
    ap.add_argument("--e2e", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    gpu, pl = _gpu()
    for N in args.sizes:
        print(json.dumps({"gpu": gpu, "power_limit": pl, **bench_scene(N, args.grid, args.chunk, args.oracle_pairs, args.oracle_images)}),
              flush=True)
    if args.e2e:
        print(json.dumps({"gpu": gpu, "power_limit": pl, **bench_e2e(args.e2e, args.reps)}), flush=True)


if __name__ == "__main__":
    main()
