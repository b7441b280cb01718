#!/usr/bin/env python
"""Retrieval: what `global_descriptors` costs, `select_pairs` against the torch statement, and what retrieval saves end to end.

    python scripts/bench_retrieval.py [--reps 5] [--select-n 1000 10000 50000] [--e2e-n 50]

(a) `global_descriptors` of 16 seeded synthetic images at 560 x 560, batch 8, fp32 (parity mode) and fp16: ms per image, warmed up
    until the CUDA graphs replay, the median of `reps` calls timed with CUDA events.
(b) `select_pairs` on N random unit descriptors (D = 2048, k = 20): the whole call, and an instrumented pass of the same launches
    split into the score GEMMs and the selection (neighbours + pair list), with the GEMM's FP32 rate against the 67 TFLOP/s data-sheet
    figure (2 N^2 D operations); peak device memory of one call; and the torch statement on the same GPU (chunked torch.mm with the
    same rows per block + torch.topk + torch.unique), whose pairs must equal ours wherever no score tie sits at the k-th place.
(c) End to end on N synthetic images (560 -> 864, fp16): `match_graph` over the exhaustive graph against `global_descriptors` +
    `select_pairs(k=10)` + `match_graph` over the selected pairs; wall time (host clock around calls that end in a synchronise)
    and pair counts.
The card's name, power limit and maximum SM clock are read in the same run.  Prints markdown tables and one JSON line; writes nothing.
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

import torch  # noqa: E402

from roma_b200 import cabi, roma_outdoor, select_pairs, synthetic  # noqa: E402
from roma_b200.match_graph import WORKSPACE_BYTES  # noqa: E402

AMP = {"fp32": torch.float32, "fp16": torch.float16}
FP32_PEAK = 67e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(), "power_limit": f"unknown ({e})", "max_sm_clock": "unknown"}


def timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end), out


def median_ms(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    return statistics.median(timed(fn)[0] for _ in range(reps))


def bench_descriptors(weights, reps):
    images = synthetic.make_pair(8, 560, 864, seed=11)[0]
    images = torch.cat((images, synthetic.make_pair(8, 560, 864, seed=12)[0])).cuda()
    rows = {}
    for prec, amp in AMP.items():
        model = roma_outdoor("cuda", weights=weights[0], dinov2_weights=weights[1], coarse_res=560, upsample_res=864, amp_dtype=amp)
        ms = median_ms(lambda: model.global_descriptors(images, max_batch=8), reps)
        rows[prec] = ms / images.shape[0]
        del model
        torch.cuda.empty_cache()
    return rows


def select_split(X, k, workspace_bytes=WORKSPACE_BYTES):
    """The launches of select_pairs with CUDA events around the GEMMs and around the selection (select + pair list)."""
    N, D = X.shape
    rows = min(N, workspace_bytes // (4 * N))
    block = torch.empty(rows * N, device="cuda")
    nb = torch.empty(N, k, dtype=torch.int64, device="cuda")
    sc = torch.empty(N, k, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    gemm = sel = 0.0
    for r0 in range(0, N, rows):
        r1 = min(N, r0 + rows)
        t, _ = timed(lambda: cabi.call("romab200_gemm", "rb_gemm_args", A=X[r0:r1], B=X, C=block, M=r1 - r0, N=N, K=D, lda=D, ldb=D, ldc=N,
                                       batch0=1, batch1=1, ntaps=1, alpha=1.0, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32))
        gemm += t
        t, _ = timed(lambda: cabi.call("romab200_retrieval_select", "rb_retrieval_args", num_images=N, k=k, scores=block, ld_scores=N,
                                       row_begin=r0, row_end=r1, neighbors=nb, neighbor_scores=sc, status=status))
        sel += t
    total = N * k
    kw = dict(num_images=N, k=k, neighbors=nb, keys=torch.empty(total, dtype=torch.int64, device="cuda"),
              keys_alt=torch.empty(total, dtype=torch.int64, device="cuda"),
              hist=torch.empty(256 * (-(-total // cabi.RB_RETRIEVAL_TILE)) + 1, dtype=torch.int32, device="cuda"),
              offsets=torch.empty(total + 1, dtype=torch.int64, device="cuda"))
    t, _ = timed(lambda: cabi.call("romab200_retrieval_pairs_count", "rb_retrieval_args", **kw))
    P = int(kw["offsets"][total])
    pairs = torch.empty(P, 2, dtype=torch.int64, device="cuda")
    t2, _ = timed(lambda: cabi.call("romab200_retrieval_pairs_emit", "rb_retrieval_args", num_pairs=P, pairs=pairs, **kw))
    return gemm, sel + t + t2


def torch_statement(X, k, rows):
    N = X.shape[0]
    nbs = []
    for r0 in range(0, N, rows):
        S = torch.mm(X[r0:r0 + rows], X.T)
        S[torch.arange(S.shape[0], device="cuda"), torch.arange(r0, r0 + S.shape[0], device="cuda")] = -float("inf")
        nbs.append(torch.topk(S, k, dim=1).indices)
    nb = torch.cat(nbs)
    i = torch.arange(N, device="cuda")[:, None].expand(N, k)
    return torch.unique(torch.stack((torch.minimum(i, nb), torch.maximum(i, nb)), -1).reshape(-1, 2), dim=0)


def bench_select(ns, reps):
    out = []
    for N in ns:
        D, k = 2048, 20
        g = torch.Generator(device="cuda").manual_seed(N)
        X = torch.randn(N, D, device="cuda", generator=g)
        X = X / X.norm(dim=1, keepdim=True)
        ms = median_ms(lambda: select_pairs(X, k), reps, warmup=1)
        splits = [select_split(X, k) for _ in range(reps)]
        gemm = statistics.median(s[0] for s in splits)
        sel = statistics.median(s[1] for s in splits)
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        res = select_pairs(X, k)
        torch.cuda.synchronize()
        mem = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        rows = min(N, WORKSPACE_BYTES // (4 * N))
        t_ms = median_ms(lambda: torch_statement(X, k, rows), reps, warmup=1)
        tp = torch_statement(X, k, rows)
        same = torch.equal(tp, res.pairs)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        torch_statement(X, k, rows)
        torch.cuda.synchronize()
        t_mem = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
        flops = 2.0 * N * N * D
        out.append(dict(N=N, ms=ms, gemm_ms=gemm, select_ms=sel, gemm_tflops=flops / gemm / 1e9, gemm_peak_share=flops / gemm / 1e9 / (FP32_PEAK / 1e12),
                        peak_gib=mem, pairs=int(res.pairs.shape[0]), torch_ms=t_ms, torch_peak_gib=t_mem, torch_pairs_equal=same))
        del X, res
        torch.cuda.empty_cache()
    return out


def bench_e2e(weights, n, k):
    A, B, Ah, Bh = synthetic.make_pair((n + 1) // 2, 560, 864, seed=13)
    ims, his = torch.cat((A, B))[:n].cuda(), torch.cat((Ah, Bh))[:n].cuda()
    sizes = [(864, 864)] * n
    model = roma_outdoor("cuda", weights=weights[0], dinov2_weights=weights[1], coarse_res=560, upsample_res=864, amp_dtype=torch.float16)
    ring = [(i, (i + 1) % n) for i in range(n)]
    for _ in range(2):                       # warm-up: every image encoded, the batch-8 graphs captured
        model.match_graph(ims, ring, his, image_sizes=sizes, num=1000)
        model.global_descriptors(ims)
    torch.cuda.synchronize()
    exhaustive = [(i, j) for i in range(n) for j in range(i + 1, n)]
    t0 = time.perf_counter()
    model.match_graph(ims, exhaustive, his, image_sizes=sizes, num=1000)
    torch.cuda.synchronize()
    t_exh = time.perf_counter() - t0
    t0 = time.perf_counter()
    d = model.global_descriptors(ims)
    torch.cuda.synchronize()
    t_desc = time.perf_counter() - t0
    res = select_pairs(d, k)
    torch.cuda.synchronize()
    t_sel = time.perf_counter() - t0 - t_desc
    model.match_graph(ims, res.pairs, his, image_sizes=sizes, num=1000)
    torch.cuda.synchronize()
    t_ret = time.perf_counter() - t0
    return dict(n=n, k=k, exhaustive_pairs=len(exhaustive), exhaustive_s=t_exh, retrieval_pairs=int(res.pairs.shape[0]), retrieval_s=t_ret,
                descriptors_s=t_desc, select_s=t_sel)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--select-n", type=int, nargs="+", default=[1000, 10000, 50000])
    ap.add_argument("--e2e-n", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_retrieval needs a CUDA device")
    info = card()
    weights = synthetic.make_weights(0)
    desc = bench_descriptors(weights, args.reps)
    sel = bench_select(args.select_n, args.reps)
    e2e = bench_e2e(weights, args.e2e_n, 10)
    print(f"card: {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}\n")
    print("| global_descriptors, 560 x 560, batch 8 | ms / image |\n|---|---|")
    for p, v in desc.items():
        print(f"| {p} | {v:.2f} |")
    print("\n| N | select_pairs ms | GEMM ms | select ms | GEMM TFLOP/s (share of 67) | peak GiB | pairs | torch ms | torch peak GiB | same pairs |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for r in sel:
        print(f"| {r['N']} | {r['ms']:.1f} | {r['gemm_ms']:.1f} | {r['select_ms']:.1f} | {r['gemm_tflops']:.1f} ({100 * r['gemm_peak_share']:.0f} %) | "
              f"{r['peak_gib']:.2f} | {r['pairs']} | {r['torch_ms']:.1f} | {r['torch_peak_gib']:.2f} | {r['torch_pairs_equal']} |")
    print(f"\nend to end, {e2e['n']} images 560 -> 864 fp16: exhaustive match_graph {e2e['exhaustive_pairs']} pairs {e2e['exhaustive_s']:.1f} s; "
          f"descriptors {e2e['descriptors_s']:.2f} s + select_pairs(k={e2e['k']}) {e2e['select_s']:.3f} s + match_graph "
          f"{e2e['retrieval_pairs']} pairs = {e2e['retrieval_s']:.1f} s")
    print(json.dumps(dict(card=info, descriptors_ms_per_image=desc, select=sel, e2e=e2e)))


if __name__ == "__main__":
    main()
