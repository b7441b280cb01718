"""Device JPEG decoding (roma_b200/csrc/jpeg.cu) against Pillow on the same host, and `match` from paths through both routes.

    python scripts/bench_jpeg.py [--reps 20]

Prints one JSON line per measurement and a summary line with the GPU name, power limit and max SM clock:
  - single-image latency of the device decode (file read + host parse + H2D of the compressed bytes + decode + status read)
    for the fixtures, the 6000 x 4000 q90 4:2:0 corpus entry and a 6000 x 4000 q100 4:4:4 file without restart markers (the
    most compressed bits per pixel, the longest Huffman sync chains), next to Pillow's `np.asarray(Image.open(p))` on this
    host, and the sync passes;
  - batched throughput for 64 x 640 x 480 in images/s, compressed MB/s and output MP/s;
  - `match(path, path)` pairs/s for RoMa 560 -> 864 and TinyRoMa: device route (paths) vs host route (PIL images opened and
    converted by the caller in the timed loop, which is what the path route did before).
Nothing is written to the repository: synthetic files go to a temporary directory.
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_keypoints import gpu_info  # noqa: E402


def _timed(fn, reps, sync):
    fn()
    sync()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        sync()
        ts.append(time.perf_counter() - t)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image

    from roma_b200 import jpeg, roma_outdoor, synthetic, tiny_roma_v1_outdoor
    sync = torch.cuda.synchronize
    nosync = lambda: None      # noqa: E731
    tmp = tempfile.mkdtemp()
    fixtures = [os.path.join(ROOT, "tests", "golden", "jpeg", f) for f in ("sacre_coeur_A.jpg", "sacre_coeur_B.jpg", "toronto_A.jpg")]
    corpus = {n: d for n, d, dec in synthetic.jpeg_corpus(0) if dec is None}
    big = os.path.join(tmp, "synthetic_6000x4000.jpg")
    with open(big, "wb") as f:
        f.write(corpus["rgb_6000x4000_q90_s2"])
    big444 = os.path.join(tmp, "synthetic_6000x4000_q100_444.jpg")
    Image.fromarray(synthetic._jpeg_image(np.random.RandomState(5), 6000, 4000, False)).save(big444, "JPEG", quality=100,
                                                                                                 subsampling=0)
    stats = {}

    def device_decode(srcs):
        datas = [jpeg.read_source(p) for p in srcs]
        res, stats["passes"] = jpeg.decode_device(datas, [jpeg.parse(d) for d in datas], "cuda", [False] * len(datas))
        assert not any(isinstance(r, str) for r in res), res
        return res

    rows = []
    for p in fixtures + [big, big444]:
        reps = max(3, args.reps // 4) if p in (big, big444) else args.reps
        dev = _timed(lambda: device_decode([p]), reps, sync)
        passes = stats["passes"]
        pil = _timed(lambda: np.asarray(Image.open(p)), reps, nosync)
        w, h = Image.open(p).size
        rows.append({"bench": "decode_single", "file": os.path.basename(p), "size": f"{w}x{h}", "bytes": os.path.getsize(p),
                     "device_ms": round(dev * 1e3, 3), "pillow_ms": round(pil * 1e3, 3), "sync_passes": passes})
    batch = [corpus["rgb_640x480_q90_s2"]] * 64
    t = _timed(lambda: device_decode(batch), args.reps, sync)
    mb = sum(len(b) for b in batch) / 1e6
    pil = _timed(lambda: [np.asarray(Image.open(__import__("io").BytesIO(b))) for b in batch], max(3, args.reps // 4), nosync)
    rows.append({"bench": "decode_batch64_640x480", "device_images_per_s": round(64 / t, 1), "device_MB_per_s": round(mb / t, 1),
                 "device_MP_per_s": round(64 * 0.3072 / t, 1), "pillow_images_per_s_one_core": round(64 / pil, 1),
                 "sync_passes": stats["passes"]})
    mw, dw = synthetic.make_weights(0)
    roma = roma_outdoor("cuda:0", weights=mw, dinov2_weights=dw, amp_dtype=torch.float32)
    xf = synthetic.xfeat_standin()
    tiny = tiny_roma_v1_outdoor("cuda:0", weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    a, b = fixtures[:2]
    reps = max(3, args.reps // 4)
    for name, dev_fn, host_fn in (
            ("roma_560_864", lambda: roma.match(a, b),
             lambda: roma.match(Image.open(a).convert("RGB"), Image.open(b).convert("RGB"))),
            ("tiny_roma", lambda: tiny.match_from_path(a, b), lambda: tiny.match(Image.open(a), Image.open(b)))):
        td = _timed(dev_fn, reps, sync)
        th = _timed(host_fn, reps, sync)
        rows.append({"bench": f"match_paths_{name}", "pair": "sacre_coeur_A/B", "device_route_pairs_per_s": round(1 / td, 2),
                     "host_route_pairs_per_s": round(1 / th, 2)})
    for r in rows:
        print(json.dumps(r))
    print(json.dumps({"summary": gpu_info(), "host_cpu_threads": os.cpu_count()}))


if __name__ == "__main__":
    main()
