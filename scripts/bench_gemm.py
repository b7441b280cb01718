"""Where the tensor-core GEMM's time goes in the parity-mode (split-fp16) step, on one GPU.

    python scripts/bench_gemm.py [--reps 20] [--out FILE]

1. Runs one eager parity-mode `match()` at 560 -> 864 (seeded synthetic weights, seed-1 pair) and records the arguments of every
   `romab200_gemm` call the engine makes (by wrapping `roma_b200.engine.call`).  Each distinct launch is replayed `--reps` times from
   one CUDA graph, so the table holds device time only: shape, tile width, epilogue, output dtype, row map, ms per launch, TFLOP/s
   counted as 3 * 2MNK (three MMAs per k-step) and the share of the summed GEMM time.  GEMMs issued from inside the GP solve's C++
   chain do not pass through Python and are not in the table.  Per launch also the tile order (m-fastest or bands of M-tiles),
   the compulsory HBM bytes (A once, B once, C, R), the bytes under the order used, achieved GB/s, and the least time at the
   data-sheet HBM bandwidth and fp16 tensor rate: the larger of the two says whether the launch is HBM- or tensor-bound.
2. K-sweep: for the step's dominant GEMM groups, times the same launch (same M, N, epilogue, output dtype and row map) on fresh
   operands at several K and fits t = a + b K.  The intercept `a` (per tile wave) is the fixed cost per tile, epilogue and set-up;
   the slope `b` gives the main-loop rate.
3. Records the card name, power limit and maximum SM clock.

Prints one JSON document (and writes it to --out if given).
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

COARSE, UPSAMPLE = 560, 864
EPI = {0: "linear", 1: "coskernel"}
ACT = {0: "none", 1: "relu", 2: "gelu"}
DT = {0: "f32", 1: "f16", 2: "bf16", 3: "f16s"}
ROWMAP = {0: "none", 1: "pad_keep", 2: "pad_to_compact", 3: "segment"}
# NVIDIA H100 SXM data sheet (a card allowed 700 W): HBM3 bandwidth and dense fp16 tensor rate
DATASHEET_HBM_GBS, DATASHEET_F16_TFLOPS = 3350.0, 989.0


def tile_width(N, M, z, trans_b, split, sms, max_split_bn):
    """Tile width gemm_tc() picks (gemm_tc.cu); max_split_bn = 128 reproduces builds without 144-wide split tiles."""
    bn = 32 if N <= 32 and not trans_b else (64 if N <= 64 else 128)
    if trans_b or N <= 128:
        return bn
    if split:
        if max_split_bn < 144:
            return 128
        bn = 144 if -N % 144 < -N % 128 else 128
    elif N <= 144:
        bn = 144
    elif N <= 192:
        bn = 192
    else:
        bn = 192 if (-N % 192) + N // 20 < -N % 256 else 256
    if math.ceil(M / 128) * math.ceil(N / bn) * z < sms * 2 // 3:
        bn = 128
    return bn


def operand_bytes(kw):
    """HBM bytes of one pass over A (per z: rows x K-extent, the map of a 9-tap launch once), B (per z), C and R (all z)."""
    M, N, K = kw["M"], kw["N"], kw["K"]
    z = (kw.get("batch0") or 1) * (kw.get("batch1") or 1)
    ntaps = kw.get("ntaps", 1) or 1
    planes = 2 if kw.get("dtype_ab") == 3 else 1
    es = {0: 4, 1: 2, 2: 2, 3: 4}                        # RB_F16S: two fp16 planes
    a = M * (K // ntaps if ntaps > 1 else K) * planes * 2
    b = N * K * planes * 2
    c = M * N * z * es[kw.get("dtype_c", 0)]
    r = M * N * z * es[kw.get("dtype_r", 0)] if kw.get("R") is not None else 0
    return a, b, c, r


def tile_order(kw, tiles_m, tiles_n, sms, l2, bands_enabled):
    """(order, M-tiles per band) gemm_tc() picks (launch_tc in gemm_tc.cu); bands_enabled = False reproduces builds that always walk
    the tiles m-fastest."""
    z = (kw.get("batch0") or 1) * (kw.get("batch1") or 1)
    a, b, _, _ = operand_bytes(kw)
    resident = min(sms, kw["max_ctas"]) if kw.get("max_ctas") else sms
    grid = min(tiles_m * tiles_n * z, resident)
    band_m = max(1, grid // tiles_n)
    if bands_enabled and tiles_n > 1 and 2 * a > l2 and 2 * b <= l2 and band_m < tiles_m:
        return "bands", band_m
    return "m_fastest", tiles_m


def hbm_bytes(kw, order, tiles_n, n_bands, l2):
    """(compulsory, scheduled) HBM bytes of one launch.  Compulsory: A once + B once + C + R (R is read even when it is C).
    Scheduled, by the model the order rule rests on: m-fastest reads A once per N-tile when A exceeds half the L2 (the sweep over
    all of A evicts a row before its next N-tile comes back to it); bands read A once and B once per band when B exceeds half the L2."""
    a, b, c, r = operand_bytes(kw)
    z = (kw.get("batch0") or 1) * (kw.get("batch1") or 1)
    compulsory = (a + b) * z + c + r
    a_reads = tiles_n if order == "m_fastest" and 2 * a > l2 else 1
    b_reads = n_bands if order == "bands" and 2 * b > l2 else 1
    return compulsory, (a * a_reads + b * b_reads) * z + c + r


def gpu_info():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [s.strip() for s in out.split(",")]
        info.update(smi_name=name, power_limit=power, clocks_max_sm=clock)
    except Exception as exc:                       # the numbers are still device times; the card's settings are then unknown
        info["smi_error"] = f"{type(exc).__name__}: {exc}"[:200]
    return info


def record_step():
    """One eager parity-mode match() with every romab200_gemm call's keyword arguments recorded (tensors kept alive)."""
    import torch
    from roma_b200 import engine, roma_outdoor, synthetic
    mw, dw = synthetic.make_weights(0)
    model = roma_outdoor("cuda:0", weights=mw, dinov2_weights=dw, coarse_res=COARSE, upsample_res=UPSAMPLE, amp_dtype=torch.float32)
    model.use_cuda_graph = False
    A, B, Ah, Bh = (t.cuda() for t in synthetic.make_pair(1, COARSE, UPSAMPLE, seed=1))
    model.match(A, B, im_A_high_res=Ah, im_B_high_res=Bh)          # warm: buffers, constants, function attributes
    torch.cuda.synchronize()
    calls = []
    inner = engine.call

    def spy(fn_name, struct_name, **kw):
        if fn_name == "romab200_gemm":
            calls.append(dict(kw))
        return inner(fn_name, struct_name, **kw)
    engine.call = spy
    try:
        model.match(A, B, im_A_high_res=Ah, im_B_high_res=Bh)
        torch.cuda.synchronize()
    finally:
        engine.call = inner
    return model, calls


def launch_key(kw):
    """Everything but the operand addresses: launches with equal keys do the same work."""
    import torch
    addresses = ("A", "B", "C", "A_lo", "B_lo", "C_lo", "R", "bias", "col_scale", "norm_a", "norm_b")
    scalars = sorted((k, tuple(v) if isinstance(v, (list, tuple)) else v) for k, v in kw.items()
                     if not isinstance(v, torch.Tensor) and k not in addresses)
    flags = [(k, kw.get(k) is not None) for k in ("R", "bias", "col_scale")]
    return tuple(scalars + flags + [("R_is_C", kw.get("R") is not None and _same(kw.get("R"), kw.get("C")))])


def _same(a, b):
    return a.data_ptr() == b.data_ptr()


def time_launch(kw, reps, trials=5):
    """ms per launch: `reps` launches captured in one CUDA graph, best of `trials` replays."""
    import torch
    from roma_b200.cabi import call
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call("romab200_gemm", "rb_gemm_args", **kw)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            call("romab200_gemm", "rb_gemm_args", **kw)
    g.replay()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(trials):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1) / reps)
    del g
    return best


def describe(kw, sms, max_split_bn, l2, bands_enabled):
    M, N, K = kw["M"], kw["N"], kw["K"]
    z = (kw.get("batch0") or 1) * (kw.get("batch1") or 1)
    split = kw.get("dtype_ab") == 3
    bn = tile_width(N, M, z, kw.get("trans_b", 0), split, sms, max_split_bn)
    tiles_m, tiles_n = math.ceil(M / 128), math.ceil(N / bn)
    tiles = tiles_m * tiles_n * z
    order, band_m = tile_order(kw, tiles_m, tiles_n, sms, l2, bands_enabled)
    compulsory, scheduled = hbm_bytes(kw, order, tiles_n, math.ceil(tiles_m / band_m), l2)
    return dict(M=M, N=N, K=K, batch=z, ntaps=kw.get("ntaps", 1) or 1, trans_b=kw.get("trans_b", 0), operands=DT[kw.get("dtype_ab", 0)],
                bn=bn, tiles=tiles, tiles_n=tiles_n, waves=math.ceil(tiles / sms), order=order, band_m=band_m,
                epi=EPI[kw.get("epi", 0)], act=ACT[kw.get("act", 0)],
                out=DT[kw.get("dtype_c", 0)], rowmap=ROWMAP[kw.get("rowmap", 0)], residual=kw.get("R") is not None,
                residual_is_c=kw.get("R") is not None and _same(kw.get("R"), kw.get("C")),
                bias=kw.get("bias") is not None, col_scale=kw.get("col_scale") is not None,
                a_mb=operand_bytes(kw)[0] / 1e6, hbm_mb_compulsory=compulsory / 1e6, hbm_mb_scheduled=scheduled / 1e6)


def sweep_case(kw, Ks):
    """The launch `kw` on fresh split-fp16 operands at every K in Ks (9-tap launches: K = 9 * k_per_tap); same epilogue arguments."""
    import torch
    M, N = kw["M"], kw["N"]
    ntaps = kw.get("ntaps", 1) or 1
    a_rows = kw.get("a_rows") or M
    out = []
    for K in Ks:
        kin = K // ntaps
        A = torch.randn(a_rows, kin, device="cuda").to(torch.float16)
        B = torch.randn(N, K, device="cuda").to(torch.float16)
        args = {k: v for k, v in kw.items() if k not in ("A", "A_lo", "B", "B_lo")}
        args.update(A=A, A_lo=A, B=B, B_lo=B, K=K, lda=kin, ldb=K)
        out.append((K, time_launch(args, reps=10, trials=3)))
        del A, B
    return out


def fit(points):
    n = len(points)
    sx = sum(k for k, _ in points); sy = sum(t for _, t in points)
    sxx = sum(k * k for k, _ in points); sxy = sum(k * t for k, t in points)
    b = (n * sxy - sx * sy) / (n * sxx - sx * sx)
    return (sy - b * sx) / n, b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="launches per CUDA graph in the per-launch table")
    ap.add_argument("--max-split-bn", type=int, default=144, choices=[128, 144],
                    help="widest split-fp16 tile of the build being measured (labels the table only)")
    ap.add_argument("--no-bands", action="store_true",
                    help="the build being measured always walks its tiles m-fastest (labels the table only)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_gemm.py needs a GPU"
    torch.cuda.set_device(0)
    props = torch.cuda.get_device_properties(0)
    sms, l2 = props.multi_processor_count, props.L2_cache_size
    doc = {"gpu": dict(gpu_info(), l2_bytes=l2, datasheet_hbm_gbs=DATASHEET_HBM_GBS, datasheet_f16_tflops=DATASHEET_F16_TFLOPS),
           "workload": f"parity-mode match() at {COARSE} -> {UPSAMPLE}, one symmetric pair"}
    model, calls = record_step()

    groups = {}
    for kw in calls:
        key = launch_key(kw)
        if key in groups:
            groups[key]["count"] += 1
        else:
            groups[key] = {"kw": kw, "count": 1}
    rows = []
    for g in groups.values():
        kw = g["kw"]
        ms = time_launch(kw, args.reps)
        d = describe(kw, sms, args.max_split_bn, l2, not args.no_bands)
        flop = (3 if kw.get("dtype_ab") == 3 else 1) * 2.0 * d["M"] * d["N"] * d["K"] * d["batch"]
        # least time at the data-sheet rates: which of the two bounds the launch (labelled as data-sheet figures)
        ms_hbm = d["hbm_mb_scheduled"] * 1e6 / (DATASHEET_HBM_GBS * 1e9) * 1e3
        ms_tc = flop / (DATASHEET_F16_TFLOPS * 1e12) * 1e3
        d.update(count=g["count"], ms=ms, ms_total=ms * g["count"], tflops=flop / (ms * 1e-3) / 1e12,
                 gbs_scheduled=d["hbm_mb_scheduled"] / ms, gbs_compulsory=d["hbm_mb_compulsory"] / ms,
                 hbm_share_scheduled=d["hbm_mb_scheduled"] / ms / DATASHEET_HBM_GBS,
                 datasheet_min_ms_hbm=ms_hbm, datasheet_min_ms_tc=ms_tc, bound="hbm" if ms_hbm > ms_tc else "tensor")
        rows.append(d)
    total = sum(r["ms_total"] for r in rows)
    for r in rows:
        r["share"] = r["ms_total"] / total
    rows.sort(key=lambda r: -r["ms_total"])
    split_flop = sum((3 * 2.0 * r["M"] * r["N"] * r["K"] * r["batch"]) * r["count"] for r in rows if r["operands"] == "f16s")
    split_ms = sum(r["ms_total"] for r in rows if r["operands"] == "f16s")
    doc["launches"] = {"calls": len(calls), "distinct": len(rows), "gemm_ms_sum": total, "split_ms_sum": split_ms,
                       "split_tflops": split_flop / (split_ms * 1e-3) / 1e12 if split_ms else None, "table": rows}

    # K-sweep over the dominant groups
    def first(pred):
        for kw in calls:
            if pred(kw):
                return kw
        return None
    lin = lambda kw: (kw.get("ntaps", 1) or 1) == 1 and not kw.get("trans_b", 0) and (kw.get("batch0") or 1) * (kw.get("batch1") or 1) == 1
    cases = {
        "vit_qkv": first(lambda kw: lin(kw) and kw["N"] == 3072 and kw["K"] == 1024),
        "vit_fc1": first(lambda kw: lin(kw) and kw["N"] == 4096 and kw["K"] == 1024),
        "vit_fc2": first(lambda kw: lin(kw) and kw["N"] == 1024 and kw["K"] == 4096),
        "refiner_pw_c144": first(lambda kw: lin(kw) and kw["N"] == 144 and kw["K"] == 144),
        "refiner_pw_c569": first(lambda kw: lin(kw) and kw["N"] == 569 and kw["K"] == 569),
        "refiner_pw_c1137": first(lambda kw: lin(kw) and kw["N"] == 1137 and kw["K"] == 1137),
        "vgg_tap_n64": first(lambda kw: (kw.get("ntaps", 1) or 1) == 9 and kw["N"] == 64),
    }
    sweep = {}
    for name, kw in cases.items():
        if kw is None:
            sweep[name] = {"error": "no such launch in the step"}
            continue
        ntaps = kw.get("ntaps", 1) or 1
        Ks = [ntaps * k for k in ((64, 128, 256) if ntaps > 1 else (64, 128, 256, 512, 1024))]
        pts = sweep_case(kw, Ks)
        a, b = fit(pts)
        d = describe(kw, sms, args.max_split_bn, l2, not args.no_bands)
        t_at_k = a + b * kw["K"]
        sweep[name] = {"M": d["M"], "N": d["N"], "K_in_step": kw["K"], "bn": d["bn"], "tiles": d["tiles"], "waves": d["waves"],
                       "epi": d["epi"], "act": d["act"], "out": d["out"], "rowmap": d["rowmap"], "residual": d["residual"],
                       "points_ms": pts, "intercept_ms": a, "intercept_us_per_wave": a * 1e3 / d["waves"],
                       "slope_us_per_kblock_per_wave": b * 64 * 1e3 / d["waves"],
                       "mainloop_tflops": 3 * 2.0 * d["M"] * d["N"] / (b * 1e-3) / 1e12 if b > 0 else None,
                       "intercept_share_at_step_K": a / t_at_k if t_at_k > 0 else None}
    doc["k_sweep"] = sweep
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
