"""TinyRoMa throughput on one H100: BASELINE config 5 (tiny_roma_v1_outdoor, batch of 560x560 pairs) on a single GPU.

    python scripts/bench_tiny.py [--pairs-per-gpu 32] [--steps K] [--warmup W] [--no-sample] [--no-library-baseline] [--no-cpu-baseline]

Prints one JSON line: pairs/s of match() + sample(5000) per pair, live parity against the reference golden `tests/golden/tiny_full.npz`,
the fused correlation / soft-argmax kernel's time and FLOP rate (from the shapes), stock PyTorch on the same GPU running the oracle
(`gpu_library_baseline`, TF32 off) and the oracle on the host cores (`cpu_baseline`).  Writes nothing to disk.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def run_tiny(args):
    """BASELINE config 5 on one GPU: TinyRoMa around the stand-in XFeat backbone (`synthetic.xfeat_standin`, unverified against the real
    network; seeded synthetic checkpoint) on rand(B, 3, 560, 560) pairs, which the model resizes to 544 x 544 (multiples of 32); one step =
    match() of `--pairs-per-gpu` pairs + sample(num=5000) of every pair.  Multi-GPU scaling of config 5 is not part of this leg."""
    import numpy as np
    import torch
    from oracle.tiny_oracle import TinyOracle
    from roma_b200 import synthetic, tiny_roma_v1_outdoor
    from roma_b200.cabi import call
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    xf = synthetic.xfeat_standin()
    sd = synthetic.make_tiny_weights(0, xf)
    model = tiny_roma_v1_outdoor(dev, weights=sd, xfeat=xf)
    B, size, num = args.pairs_per_gpu, 560, 5000
    g = torch.Generator().manual_seed(0)
    im_a, im_b = torch.rand(B, 3, size, size, generator=g).to(dev), torch.rand(B, 3, size, size, generator=g).to(dev)

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps

    def step(m=model, a=im_a, b=im_b):
        warp, cert = m.match(a, b)
        if not args.no_sample:
            for i in range(a.shape[0]):
                m.sample(warp[i], cert[i], num=num)
    dt = timed(step, args.steps, max(args.warmup, 2))
    line = {"impl": "ours", "model": "tiny_roma_v1_outdoor", "metric": "image-pairs/sec match()+sample(5000) 560x560 (544 after resize)",
            "unit": "pairs/s", "n_gpus": 1, "pairs_per_gpu": B, "value": round(B / dt, 3), "ms_per_step": round(dt * 1e3, 3),
            "device": torch.cuda.get_device_name(dev)}
    # live parity against the full-size golden of the unmodified reference (tests/golden/tiny_full.npz)
    gd = np.load(os.path.join(ROOT, "tests", "golden", "tiny_full.npz"))
    gg = torch.Generator().manual_seed(int(gd["meta"][0]))
    a1, b1 = torch.rand(*gd["shape0"], generator=gg), torch.rand(*gd["shape1"], generator=gg)
    warp, cert = model.match(a1.to(dev), b1.to(dev))
    st = int(gd["meta"][2])
    line["parity_vs_reference_golden"] = {"warp_max_abs": float(np.abs(warp[:, ::st, ::st].cpu().numpy() - gd["warp"]).max()),
                                          "certainty_max_abs": float(np.abs(cert[:, ::st, ::st].cpu().numpy() - gd["certainty"]).max()),
                                          "tolerance": 1e-4}
    # the fused correlation / argmax / soft-argmax kernel on the shapes of one step (68 x 68 coarse maps, 64-d features), in one CUDA graph
    h = size // 32 * 32 // 8
    f0, f1 = torch.randn(B, h * h, 64, device=dev), torch.randn(B, h * h, 64, device=dev)
    state = torch.empty(B, h * h, 3, device=dev)
    lin = lambda lo, n: torch.linspace(-1 + lo, 1 - lo, n).to(dev)
    gx, glx = lin(1 / h, h), lin(4 / h, h // 4)
    launch = lambda: call("romab200_tiny_pos_embed", "rb_tiny_pos_embed_args", f0=f0, f1=f1, state=state, batch=B, h0=h, w0=h, h1=h, w1=h, c=64,
                          scale=8.0, exact=0, grid_x=gx, grid_y=gx, grid_lr_x=glx, grid_lr_y=glx)
    launch()
    torch.cuda.synchronize()
    graph, reps = torch.cuda.CUDAGraph(), 10
    with torch.cuda.graph(graph):
        for _ in range(reps):
            launch()
    ts = []
    for _ in range(7):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); graph.replay(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e) / reps)
    ms = sorted(ts)[3]
    flops = 2.0 * B * (h * h) ** 2 * 64
    line["pos_embed_kernel"] = {"ms_per_step": round(ms, 4), "pairs": B, "flops_per_pair": flops / B, "tflops": round(flops / ms / 1e9, 2),
                                "arithmetic": "fp32 FFMA (CUDA cores)"}
    if not args.no_library_baseline:
        orc = TinyOracle(sd, xf, device=dev)

        def lib_step():
            with torch.no_grad():
                warp, cert = orc.match(im_a, im_b)
            if not args.no_sample:
                for i in range(B):
                    orc.sample(warp[i], cert[i], num=num)
        ld = timed(lib_step, max(1, min(args.steps, 3)), 1)
        line["gpu_library_baseline"] = {"impl": "tiny oracle on stock PyTorch CUDA (cuDNN / cuBLAS, TF32 off)", "value": round(B / ld, 3),
                                        "unit": "pairs/s", "speedup": round(ld / dt, 2)}
        del orc
    if not args.no_cpu_baseline:
        orc = TinyOracle(sd, xf)
        a0, b0 = im_a[:1].cpu(), im_b[:1].cpu()
        t0 = time.perf_counter()
        with torch.no_grad():
            warp, cert = orc.match(a0, b0)
        if not args.no_sample:
            orc.sample(warp[0], cert[0], num=num)
        ct = time.perf_counter() - t0
        line["cpu_baseline"] = {"impl": f"tiny oracle on the host CPU ({torch.get_num_threads()} threads)", "value": round(1 / ct, 4), "unit": "pairs/s"}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pairs-per-gpu", type=int, default=32, help="pairs per match() call (BASELINE config 5: 256 pairs over 8 GPUs = 32)")
    ap.add_argument("--no-sample", action="store_true")
    ap.add_argument("--no-library-baseline", action="store_true", help="skip the stock-PyTorch-CUDA comparison leg (gpu_library_baseline)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    run_tiny(ap.parse_args())


if __name__ == "__main__":
    main()
