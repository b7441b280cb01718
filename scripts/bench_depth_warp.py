"""The MegaDepth dense metric step on one H100: the fused float64 kernels (`roma_b200.dense_geometric_dist`, csrc/depth_warp.cu)
against the eager torch statement of the same step (oracle/depth_warp.py, which is what the reference's harness runs) on the same GPU.

    python scripts/bench_depth_warp.py [--reps 30] [--sizes 8x384x512,8x864x864]

Inputs: `synthetic.depth_scene` (float32 depth maps with holes, a large camera motion) and a warp that is the ground truth plus
noise, so every class of pixel occurs.  Per size one JSON line:
  - device_ms / torch_ms: one call from CUDA events after warm-up; the two are alternated in one loop and the medians of --reps
    calls each are reported (with the quartiles, to show the spread);
  - *_launches: kernels per call (the library's launch counter; torch.profiler CUDA kernel events for the torch statement);
  - *_peak_mb: growth of torch.cuda.max_memory_allocated during one call, outputs included;
  - compulsory_mb: the bytes the step has to move, from the shapes: the warp (16 B per pixel) and both depth maps read once, gd
    (8 B) and prob (4 B) written once; device_gbps = compulsory bytes / device time, and its share of the HBM bound, which is the
    bound of this step (3.35 TB/s on the H100 SXM data sheet; the ~150 float64 operations per pixel are far below the FP64 rate).
Then one step of the MegaDepth dense protocol, TinyRoMa `match` of 8 pairs at 384 x 512 followed by the metric, with the device
metric and with the torch statement, and a last line with the GPU's name, power limit and maximum SM clock.
Fails without a GPU.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12       # NVIDIA's data sheet for the H100 SXM; never reached, named as the bound


def gpu_info():
    import torch
    props = torch.cuda.get_device_properties(0)
    info = {"gpu": props.name, "sms": props.multi_processor_count}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["max_sm_clock_mhz"] = float(out[0]), float(out[1])
    except Exception as e:     # the numbers are still printed, without the card's limits
        info["nvidia_smi_error"] = repr(e)
    return info


def compulsory_bytes(B, H, W, depth0, depth1):
    return B * H * W * (16 + 8 + 4) + depth0.numel() * depth0.element_size() + depth1.numel() * depth1.element_size()


def alternate(fns, reps):
    """Median and quartiles (ms) of each callable, timed with CUDA events, one call of each per round."""
    import torch
    for f in fns:
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            ts[i].append(e0.elapsed_time(e1))
    out = []
    for t in ts:
        t.sort()
        out.append({"median": round(t[len(t) // 2], 4), "q1": round(t[len(t) // 4], 4), "q3": round(t[(3 * len(t)) // 4], 4)})
    return out


def peak_mb(f):
    import torch
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = f()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    del out
    return round(peak, 1)


def torch_kernel_count(f):
    """CUDA kernels (and memcpys / memsets) one call enqueues, from torch.profiler."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA)


def make_case(B, H, W, dev):
    import torch
    from oracle import depth_warp as oracle
    from roma_b200 import synthetic
    views = [v.to(dev) for v in synthetic.depth_scene(100, B, H, W)]
    x2, _ = oracle.get_gt_warp(*views)
    xs, ys = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n, device=dev) for n in (W, H))
    grid = torch.stack((xs[None].expand(H, W), ys[:, None].expand(H, W)), -1)[None].expand(B, -1, -1, -1)
    g = torch.Generator(device=dev).manual_seed(3)
    x2 = torch.where(torch.isfinite(x2), x2, torch.zeros((), device=dev, dtype=x2.dtype)).float()
    return views, torch.cat((grid, x2 + 4e-3 * torch.randn(B, H, W, 2, device=dev, generator=g)), dim=-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--sizes", default="8x384x512,8x864x864")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_depth_warp measures on a GPU"
    assert args.reps >= 20, "medians of fewer than 20 calls are not reported"
    from oracle import depth_warp as oracle
    from roma_b200 import cabi, dense_geometric_dist, synthetic, tiny_roma_v1_outdoor
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    for B, H, W in (tuple(int(x) for x in s.split("x")) for s in args.sizes.split(",")):
        views, dm = make_case(B, H, W, dev)
        device = lambda: dense_geometric_dist(*views, dm)            # noqa: E731
        eager = lambda: oracle.dense_geometric_dist(*views, dm)      # noqa: E731
        res, ref = device(), eager()
        same = bool(torch.equal(res.prob, ref["prob"]) and torch.equal(res.pair_count, ref["pair_count"]))
        gd_err = ((res.gd - ref["gd"]).nan_to_num().abs().max() / ref["gd"].nan_to_num().max()).item()
        n0 = cabi.kernel_launches()
        device()
        dev_launches = cabi.kernel_launches() - n0
        t_dev, t_torch = alternate((device, eager), args.reps)
        nbytes = compulsory_bytes(B, H, W, views[0], views[1])
        rate = nbytes / (t_dev["median"] / 1e3)
        print(json.dumps({
            "size": f"{B}x{H}x{W}", "pixels": B * H * W, "valid_fraction": round(res.prob.mean().item(), 3), "epe_px": round(res.epe.item(), 4),
            "same_counts_as_torch": same, "gd_max_rel_err_vs_torch": gd_err,
            "device_ms": t_dev, "torch_ms": t_torch, "speedup": round(t_torch["median"] / t_dev["median"], 1),
            "device_launches": dev_launches, "torch_launches": torch_kernel_count(eager),
            "device_peak_mb": peak_mb(device), "torch_peak_mb": peak_mb(eager),
            "compulsory_mb": round(nbytes / 1e6, 1), "device_gbps": round(rate / 1e9, 1), "bound": "HBM",
            "share_of_hbm_data_sheet": round(rate / HBM_BYTES_PER_S, 3)}), flush=True)
        del views, dm, res, ref
        torch.cuda.empty_cache()
    # one step of the MegaDepth dense protocol with TinyRoMa: match of 8 pairs + the metric
    B, H, W = 8, 384, 512
    xf = synthetic.xfeat_standin()
    model = tiny_roma_v1_outdoor("cuda:0", weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    views = [v.to(dev) for v in synthetic.depth_scene(100, B, H, W)]
    g = torch.Generator(device=dev).manual_seed(5)
    a, b = torch.rand(B, 3, H, W, device=dev, generator=g), torch.rand(B, 3, H, W, device=dev, generator=g)
    match_only = lambda: model.match(a, b)                                                      # noqa: E731
    step_device = lambda: dense_geometric_dist(*views, model.match(a, b)[0])                    # noqa: E731
    step_torch = lambda: oracle.dense_geometric_dist(*views, model.match(a, b)[0])              # noqa: E731
    t_match, t_dev, t_torch = alternate((match_only, step_device, step_torch), args.reps)
    print(json.dumps({"protocol_step": f"tiny_roma_v1_outdoor match of {B} pairs at {H}x{W} + metric", "match_only_ms": t_match,
                      "with_device_metric_ms": t_dev, "with_torch_metric_ms": t_torch}), flush=True)
    print(json.dumps(info), flush=True)


if __name__ == "__main__":
    main()
