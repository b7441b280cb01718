"""Golden vectors for the depth-based warps, FROM THE UNMODIFIED REFERENCE (`romatch.utils.utils.warp_kpts`, `get_gt_warp`,
romatch/utils/utils.py:325-454), on the CPU in float64.

Run where the reference is importable (it is not needed by any test):

    PYTHONPATH=<reference tree> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_depth_warp.py

Two pairs of `synthetic.depth_scene(5, 2, 48, 64, 60, 80)` (the two views differ in size) and 3000 points per pair: uniform in
[-1.1, 1.1]^2, so some lie outside view 0, plus a few at the corners and far outside both images.  depth_warp.npz holds the inputs
and, for the modes `bilinear` and `nearest`, `warp_kpts`'s (valid, warped) on the points and `get_gt_warp`'s (x2, prob) at the depth
map's own size and at H, W = 30, 44.  The harness's metric (`romatch.benchmarks`) cannot be imported without its dataset
dependencies; it is pinned through oracle/depth_warp.py, which these vectors pin.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
from romatch.utils.utils import get_gt_warp, warp_kpts  # noqa: E402  (the reference)

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from roma_b200 import synthetic  # noqa: E402


def main():
    depth0, depth1, T, K0, K1 = synthetic.depth_scene(5, 2, 48, 64, 60, 80)
    g = torch.Generator().manual_seed(11)
    kpts = torch.rand(2, 3000, 2, generator=g, dtype=torch.float64) * 2.2 - 1.1
    kpts[:, :6] = torch.tensor([[-1.0, -1.0], [1.0, 1.0], [-1.0, 1.0], [0.0, 0.0], [7.5, -3.0], [-40.0, 90.0]], dtype=torch.float64)
    out = {"depth0": depth0.numpy(), "depth1": depth1.numpy(), "T": T.numpy(), "K0": K0.numpy(), "K1": K1.numpy(), "kpts": kpts.numpy()}
    for mode in ("bilinear", "nearest"):
        valid, warped = warp_kpts(kpts, depth0.double(), depth1.double(), T, K0, K1, depth_interpolation_mode=mode)
        out[f"valid_{mode}"], out[f"warped_{mode}"] = valid.numpy(), warped.numpy()
        x2, prob = get_gt_warp(depth0, depth1, T, K0, K1, depth_interpolation_mode=mode)
        out[f"x2_{mode}"], out[f"prob_{mode}"] = x2.numpy(), prob.numpy()
        x2, prob = get_gt_warp(depth0, depth1, T, K0, K1, depth_interpolation_mode=mode, H=30, W=44)
        out[f"x2_hw_{mode}"], out[f"prob_hw_{mode}"] = x2.numpy(), prob.numpy()
    path = os.path.join(HERE, "depth_warp.npz")
    np.savez_compressed(path, **out)
    print({k: (v.shape, str(v.dtype)) for k, v in out.items()}, os.path.getsize(path), "bytes;",
          "valid fraction", float(out["valid_bilinear"].mean()), "prob mean", float(out["prob_bilinear"].mean()))


if __name__ == "__main__":
    main()
