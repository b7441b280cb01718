"""Device time of the parity-mode refiner blocks at C = 144 (the stride-2 maps of the 560 -> 864 step), fused and un-fused.

    python scripts/bench_refiner.py [--reps 20] [--unfused-only] [--out FILE]

For the two stride-2 shapes of a symmetric pair (2 x 432 x 432 at 864, 2 x 280 x 280 at 560) on seeded random fp32 maps and weights:
1. Replays the 9-block chain of the parity mode from CUDA graphs, un-fused (`romab200_dwconv5x5_relu` writing the split-fp16 A
   operand, then the split-fp16 pointwise `romab200_gemm`) and fused (`romab200_refiner_block_c144_split`, ping-ponging two fp32
   maps), and times each of the two un-fused launches on its own.
2. Prints device ms per block, the byte model (8 B per map element and block fused: read the map once, write it once; 16 B
   un-fused: the depthwise kernel reads 4 B and writes the 4-B split pair, the GEMM reads the pair and writes 4 B), achieved
   GB/s, and the share of the least time at the data-sheet rates: the larger of bytes over HBM bandwidth and 3 x 2 MNK over the
   fp16 tensor rate (three MMAs per k-step).
3. Records the card name, power limit and maximum SM clock.

--unfused-only measures the two-launch chain alone, e.g. on a build without the fused kernel.  Prints one JSON document (and
writes it to --out if given).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_gemm import DATASHEET_F16_TFLOPS, DATASHEET_HBM_GBS, gpu_info  # noqa: E402

C, BLOCKS = 144, 9
SHAPES = {"864": (2, 432, 432), "560": (2, 280, 280)}


def make_blocks(seed=0):
    """BLOCKS sets of (depthwise taps [25][C], depthwise bias, pointwise split planes [C][C], pointwise bias), packed as the engine does."""
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    blocks = []
    for _ in range(BLOCKS):
        dw = (torch.randn(25, C, generator=g) * 0.2).cuda()
        db = (torch.randn(C, generator=g) * 0.1).cuda()
        pw = torch.randn(C, C, generator=g) * (1.0 / C ** 0.5)
        hi = pw.half()
        lo = ((pw - hi.float()) * 2048.0).half()
        pb = (torch.randn(C, generator=g) * 0.1).cuda()
        blocks.append(dict(dw=dw, db=db, pw_hi=hi.cuda(), pw_lo=lo.cuda(), pb=pb))
    return blocks


def dw_launch(x, ts_hi, ts_lo, blk, D, h, w):
    from roma_b200 import cabi
    cabi.call("romab200_dwconv5x5_relu", "rb_dwconv_args", **{"in": x}, out=ts_hi, out_lo=ts_lo, ldi=C, ldo=C, weight=blk["dw"], ldw=C,
              bias=blk["db"], batch=D, h=h, w=w, c=C, dtype=cabi.RB_F32)


def gemm_launch(ts_hi, ts_lo, y, blk, rows):
    from roma_b200 import cabi
    cabi.call("romab200_gemm", "rb_gemm_args", A=ts_hi, A_lo=ts_lo, B=blk["pw_hi"], B_lo=blk["pw_lo"], C=y, M=rows, N=C, K=C, lda=C, ldb=C,
              ldc=C, batch0=1, batch1=1, ntaps=1, alpha=1.0, bias=blk["pb"], dtype_ab=cabi.RB_F16S, dtype_c=cabi.RB_F32)


def fused_launch(x, y, blk, D, h, w):
    from roma_b200 import cabi
    cabi.call("romab200_refiner_block_c144_split", "rb_refiner_block_c144_split_args", **{"in": x}, out=y, ld=C, dw_weight=blk["dw"],
              ldw=C, dw_bias=blk["db"], pw_weight=blk["pw_hi"], pw_weight_lo=blk["pw_lo"], ld_pw=C, pw_bias=blk["pb"], batch=D, h=h, w=w, c=C)


def time_graph(fn, reps, trials=5):
    """ms per call of fn(): `reps` calls captured in one CUDA graph, best of `trials` replays."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
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


def row(ms_per_block, bytes_per_block, flop_per_block):
    ms_hbm = bytes_per_block / (DATASHEET_HBM_GBS * 1e9) * 1e3
    ms_tc = flop_per_block / (DATASHEET_F16_TFLOPS * 1e12) * 1e3
    return {"ms_per_block": ms_per_block, "ms_chain": ms_per_block * BLOCKS, "mb_per_block": bytes_per_block / 1e6,
            "gbs": bytes_per_block / (ms_per_block * 1e-3) / 1e9, "datasheet_min_ms_hbm": ms_hbm, "datasheet_min_ms_tc": ms_tc,
            "bound": "hbm" if ms_hbm > ms_tc else "tensor", "share_of_floor": max(ms_hbm, ms_tc) / ms_per_block}


def measure(shape, blocks, reps, unfused_only):
    import torch
    D, h, w = shape
    rows = D * h * w
    elems = rows * C
    flop = 3 * 2.0 * rows * C * C
    g = torch.Generator(device="cpu").manual_seed(1)
    d = torch.randn(rows, C, generator=g).cuda()
    t = torch.empty_like(d)
    ts_hi, ts_lo = torch.empty(rows, C, dtype=torch.float16, device="cuda"), torch.empty(rows, C, dtype=torch.float16, device="cuda")

    def unfused_chain():
        for blk in blocks:
            dw_launch(d, ts_hi, ts_lo, blk, D, h, w)
            gemm_launch(ts_hi, ts_lo, d, blk, rows)

    out = {"batch": D, "h": h, "w": w, "rows": rows, "map_mb_fp32": elems * 4 / 1e6}
    chain_reps = max(1, reps // BLOCKS)
    out["unfused"] = row(time_graph(unfused_chain, chain_reps) / BLOCKS, 16 * elems, flop)
    out["unfused_dwconv_launch"] = row(time_graph(lambda: dw_launch(d, ts_hi, ts_lo, blocks[0], D, h, w), reps), 8 * elems, 0.0)
    out["unfused_gemm_launch"] = row(time_graph(lambda: gemm_launch(ts_hi, ts_lo, t, blocks[0], rows), reps), 8 * elems, flop)
    if not unfused_only:
        def fused_chain():
            x, y = d, t
            for blk in blocks:
                fused_launch(x, y, blk, D, h, w)
                x, y = y, x
        out["fused"] = row(time_graph(fused_chain, chain_reps) / BLOCKS, 8 * elems, flop)
        out["saved_ms_per_chain"] = out["unfused"]["ms_chain"] - out["fused"]["ms_chain"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=36, help="launches per CUDA graph")
    ap.add_argument("--unfused-only", action="store_true", help="time the two-launch chain only (a build without the fused kernel)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_refiner.py needs a GPU"
    torch.cuda.set_device(0)
    from roma_b200 import cabi
    cabi.load_library()
    doc = {"gpu": dict(gpu_info(), datasheet_hbm_gbs=DATASHEET_HBM_GBS, datasheet_f16_tflops=DATASHEET_F16_TFLOPS),
           "workload": f"parity-mode refiner, {BLOCKS} blocks at C = {C}, seeded random fp32 maps and weights"}
    blocks = make_blocks()
    doc["shapes"] = {name: measure(shape, blocks, args.reps, args.unfused_only) for name, shape in SHAPES.items()}
    text = json.dumps(doc, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
