#!/usr/bin/env python
"""match_pairs against a match() loop over the same pairs: exhaustive symmetric graphs over N seeded synthetic images at 560 -> 864.

    python scripts/bench_match_pairs.py [--n 2 4 8 16] [--precision fp32 fp16] [--max-batch 8] [--reps 3]

For each precision and N: (a) match() over all N (N - 1) / 2 unordered pairs in batches of max_batch pairs, (b) match_pairs over the
same pairs with the same max_batch.  Both are warmed up until their CUDA graphs replay, then timed alternately (a, b, a, b, ...) with
CUDA events around whole calls; the median is reported.  A separate eager pass of (b) times the encode step per image and the bank
gather per chunk; peak memory is measured in passes of their own.  The max-abs difference between (a) and (b) must be 0.  Prints a
markdown table and one JSON line; writes nothing else.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from roma_b200 import roma_outdoor, synthetic  # noqa: E402

AMP = {"fp32": torch.float32, "fp16": torch.float16, "bf16": torch.bfloat16}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:              # nvidia-smi missing: the numbers still carry the device name
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), out


def peak(model, fn):
    """Peak device memory of one call from a freed arena (activation buffers, feature bank, outputs), above weights and inputs."""
    model.free_buffers()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 30, out


def run(precision, n_images, max_batch, reps, coarse, up):
    model = roma_outdoor("cuda", weights=WEIGHTS[0], dinov2_weights=WEIGHTS[1], coarse_res=coarse, upsample_res=up, amp_dtype=AMP[precision])
    A, B, Ah, Bh = synthetic.make_pair((n_images + 1) // 2, coarse, up, seed=n_images)
    ims, his = torch.cat((A, B))[:n_images].cuda(), torch.cat((Ah, Bh))[:n_images].cuda()
    pairs = [(i, j) for i in range(n_images) for j in range(i + 1, n_images)]
    ia = torch.tensor([i for i, _ in pairs], device="cuda")
    ib = torch.tensor([j for _, j in pairs], device="cuda")

    def loop():
        outs = [model.match(ims[ia[k:k + max_batch]], ims[ib[k:k + max_batch]], im_A_high_res=his[ia[k:k + max_batch]],
                            im_B_high_res=his[ib[k:k + max_batch]]) for k in range(0, len(pairs), max_batch)]
        return torch.cat([w for w, _ in outs]), torch.cat([c for _, c in outs])

    def pairs_call(on_batch=None):
        return model.match_pairs(ims, pairs, his, max_batch=max_batch, on_batch=on_batch)
    diff = []
    for _ in range(3):                   # call 3 of every graph key replays
        ref = loop()

        def compare(k, w, c):            # chunk by chunk, so that only one copy of the dense outputs is alive
            diff.append(max((w - ref[0][k:k + w.shape[0]]).abs().max().item(), (c - ref[1][k:k + c.shape[0]]).abs().max().item()))
        pairs_call(compare)
        del ref
    diff = max(diff)
    ta, tb = [], []
    for _ in range(reps):
        ta.append(timed(loop)[0])
        tb.append(timed(pairs_call)[0])
    mem_a, _ = peak(model, loop)
    mem_b, _ = peak(model, pairs_call)
    # eager pass of (b): the encode step per image (CUDA events around each encode batch) and the bank gather per chunk
    eng = model.engine
    enc, orig = [], eng.encode_images        # the bound method; the wrapper below shadows it on the instance until `del`

    def encode(images, *a):
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        orig(images, *a)
        t1.record()
        enc.append((images.shape[0], t0, t1))
    eng.encode_images, eng.profile = encode, {}
    pairs_call()
    torch.cuda.synchronize()
    del eng.encode_images
    prof, eng.profile = eng.profile, None
    enc_ms = sum(t0.elapsed_time(t1) for _, t0, t1 in enc) / sum(e for e, _, _ in enc)
    gathers = [s.elapsed_time(e) for s, e in prof["bank.gather"]]
    ma, mb = statistics.median(ta), statistics.median(tb)
    res = dict(precision=precision, n_images=n_images, pairs=len(pairs), max_batch=max_batch, match_loop_pairs_s=len(pairs) / ma * 1e3,
               match_pairs_pairs_s=len(pairs) / mb * 1e3, speedup=ma / mb, match_loop_ms=ta, match_pairs_ms=tb, encode_ms_per_image=enc_ms,
               gather_ms_per_chunk=statistics.mean(gathers), chunk_ms=mb / len(gathers), peak_gb_match_loop=mem_a, peak_gb_match_pairs=mem_b,
               max_abs_diff=diff)
    model.free_buffers()
    del model, eng, loop, pairs_call
    gc.collect()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, nargs="+", default=[2, 4, 8, 16])
    ap.add_argument("--precision", nargs="+", default=["fp32", "fp16"], choices=list(AMP))
    ap.add_argument("--max-batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--coarse", type=int, default=560)
    ap.add_argument("--upsample", type=int, default=864)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_match_pairs.py needs a CUDA device")
    global WEIGHTS
    WEIGHTS = synthetic.make_weights(0)
    info = card()
    rows = [run(p, n, args.max_batch, args.reps, args.coarse, args.upsample) for p in args.precision for n in args.n]
    print(f"{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}; {args.coarse} -> {args.upsample}, "
          f"symmetric, max_batch {args.max_batch}, median of {args.reps}")
    print("| precision | N | pairs | match() loop pairs/s | match_pairs pairs/s | speed-up | encode ms/image | gather ms/chunk (call ms/chunk) "
          "| peak GB loop / pairs | max-abs diff |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['precision']} | {r['n_images']} | {r['pairs']} | {r['match_loop_pairs_s']:.2f} | {r['match_pairs_pairs_s']:.2f} | "
              f"{r['speedup']:.2f}x | {r['encode_ms_per_image']:.1f} | {r['gather_ms_per_chunk']:.2f} ({r['chunk_ms']:.0f}) | "
              f"{r['peak_gb_match_loop']:.1f} / {r['peak_gb_match_pairs']:.1f} | {r['max_abs_diff']:.1e} |")
    print(json.dumps({"card": info, "results": rows}))


if __name__ == "__main__":
    main()
