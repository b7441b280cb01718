"""`match_keypoints` on one H100: the device path (csrc/keypoints.cu) against the reference's torch statement (grid_sample + cdist +
mutual-minimum masks + nonzero) at N_A = N_B = N keypoints.

    python scripts/bench_keypoints.py [--sizes 2000,10000,30000,100000] [--reps 10] [--torch-max 30000]

Inputs: x_A uniform in [-1, 1]^2, x_B half x_A moved by N(0, 2e-3) and half uniform, a 512 x 512 warp close to the identity, random
certainty, max_dist = 0.005, cert_th = 0.1: a typical keypoint-matching call with tens of percent of the points matched.
Prints one JSON line per N and a summary line with the GPU name, power limit and max SM clock:
  - device_ms: one call from CUDA events, median over --reps, including the read of the match count;
  - device_peak_mb: growth of torch.cuda.max_memory_allocated during the call;
  - min_sweeps_ms: the two min sweeps (kernel time from torch.profiler), rate = 2 N^2 distances over that time, against the
    instruction-issue bound of the GPU (SMs x 128 lanes x max SM clock / 6 instructions per distance: 2 FADD differences, 2 FMUL,
    1 FADD and one FMNMX; the five FP32 operations alone give the FP32 bound, also printed);
  - torch_ms / torch_peak_mb: the torch statement, for N <= --torch-max (its N x N fp32 distance matrix plus the same-size
    temporaries of cdist and the masks; at 100 000 the matrix alone is 40 GB) and whether it returned the same pairs.
Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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


def make_inputs(n, dev):
    import torch
    g = torch.Generator(device=dev).manual_seed(n)
    x_A = torch.rand(n, 2, device=dev, generator=g) * 2 - 1
    h = n // 2
    x_B = torch.cat((x_A[:h] + 2e-3 * torch.randn(h, 2, device=dev, generator=g), torch.rand(n - h, 2, device=dev, generator=g) * 2 - 1))
    x_B = x_B[torch.randperm(n, device=dev, generator=g)]
    s = torch.linspace(-1 + 1 / 512, 1 - 1 / 512, 512, device=dev)
    gy, gx = torch.meshgrid(s, s, indexing="ij")
    grid = torch.stack((gx, gy), dim=-1)
    warp = torch.cat((grid, grid + 1e-3 * torch.sin(3 * grid)), dim=-1)
    cert = torch.rand(512, 512, device=dev, generator=g)
    return x_A, x_B, warp, cert


def torch_statement(x_A, x_B, warp, certainty, max_dist, cert_th):
    import torch
    import torch.nn.functional as F
    x_A_to_B = F.grid_sample(warp[..., -2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False, mode="bilinear")[0, :, 0].mT
    cert = F.grid_sample(certainty[None, None], x_A[None, None], align_corners=False, mode="bilinear")[0, 0, 0]
    D = torch.cdist(x_A_to_B, x_B)
    mutual = (D == D.min(dim=-1, keepdim=True).values) * (D == D.min(dim=-2, keepdim=True).values)
    return torch.nonzero(mutual * (cert[:, None] > cert_th) * (D < max_dist), as_tuple=True)


def timed(fn, reps):
    """(median ms of one call from CUDA events, peak allocation growth in MB of one call)."""
    import torch
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    return sorted(ts)[len(ts) // 2], peak, out


def kernel_ms(fn):
    """Device time per kernel name of one call (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.device_type == torch.autograd.DeviceType.CUDA or getattr(ev, "device_time_total", 0) > 0:
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            out[ev.key] = out.get(ev.key, 0.0) + t / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2000,10000,30000,100000")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--torch-max", type=int, default=30000)
    args = ap.parse_args()
    import torch
    from roma_b200.matcher import RegressionMatcher
    torch.backends.cuda.matmul.allow_tf32 = False
    assert torch.cuda.is_available(), "bench_keypoints measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    m = RegressionMatcher.__new__(RegressionMatcher)
    clock_hz = info.get("max_sm_clock_mhz", 0) * 1e6
    lanes = info["sms"] * 128
    for n in (int(s) for s in args.sizes.split(",")):
        x_A, x_B, warp, cert = make_inputs(n, dev)
        call = lambda: m.match_keypoints(x_A, x_B, warp, cert, return_inds=True, max_dist=0.005, cert_th=0.1)   # noqa: E731
        dev_ms, dev_peak, (ia, ib) = timed(call, args.reps)
        kms = kernel_ms(call)
        sweep_ms = sum(t for k, t in kms.items() if "kp_min_kernel" in k)
        res = {"n": n, "matches": int(ia.numel()), "device_ms": round(dev_ms, 3), "device_peak_mb": round(dev_peak, 2),
               "kernels_ms": {k.split("(")[0][-40:]: round(t, 4) for k, t in kms.items() if "kp_" in k},
               "min_sweeps_ms": round(sweep_ms, 4)}
        if sweep_ms > 0:
            rate = 2.0 * n * n / (sweep_ms / 1e3)
            res["sweep_distances_per_s"] = f"{rate:.3e}"
            if clock_hz:
                res["issue_bound_distances_per_s"] = f"{lanes * clock_hz / 6:.3e}"
                res["fp32_bound_distances_per_s"] = f"{lanes * clock_hz / 5:.3e}"
                res["share_of_issue_bound"] = round(rate / (lanes * clock_hz / 6), 3)
        if n <= args.torch_max:
            t_ms, t_peak, (ta, tb) = timed(lambda: torch_statement(x_A, x_B, warp, cert, 0.005, 0.1), max(3, args.reps // 2))
            res.update(torch_ms=round(t_ms, 3), torch_peak_mb=round(t_peak, 1), same_pairs_as_torch=bool(torch.equal(ia, ta) and torch.equal(ib, tb)))
        else:
            res.update(torch_ms=None, torch_note=f"not run: its {n}x{n} fp32 distance matrix alone is {4 * n * n / 1e9:.0f} GB")
        print(json.dumps(res), flush=True)
        del x_A, x_B, warp, cert, ia, ib
        torch.cuda.empty_cache()
    print(json.dumps(info), flush=True)


if __name__ == "__main__":
    main()
