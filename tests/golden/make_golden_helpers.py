"""Golden vectors for the pure-Python API helpers of the path (SURVEY §8 a14), FROM THE UNMODIFIED REFERENCE.

Run where the reference is importable (it is not needed by any test):

    PYTHONPATH=<reference tree> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_helpers.py

`RegressionMatcher.to_pixel_coordinates / to_normalized_coordinates / match_keypoints / conf_from_fb_consistency`
(romatch/models/matcher.py:672-773) use nothing of the model but `self`, so they are called unbound on a bare
`RegressionMatcher.__new__` instance with seeded inputs; inputs and outputs go to helpers.npz.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
from romatch.models.matcher import RegressionMatcher  # noqa: E402  (the reference)


def main():
    g = torch.Generator().manual_seed(7)
    ref = RegressionMatcher.__new__(RegressionMatcher)
    H, W = 24, 32
    out = {}
    # a smooth symmetric warp [H, 2W, 4] (identity + small seeded perturbation) and a certainty map
    xs = torch.linspace(-1 + 1 / W, 1 - 1 / W, W)
    ys = torch.linspace(-1 + 1 / H, 1 - 1 / H, H)
    grid = torch.stack(torch.meshgrid(xs, ys, indexing="xy"), dim=-1)                 # [H, W, 2]
    pert = 0.03 * torch.randn(H, W, 2, generator=g)
    a_to_b = (grid + 0.1 + pert).clamp(-1, 1)
    b_to_a = (grid - 0.1 - pert).clamp(-1, 1)
    warp = torch.cat((torch.cat((grid, a_to_b), dim=-1), torch.cat((b_to_a, grid), dim=-1)), dim=1)   # [H, 2W, 4]
    certainty = torch.rand(H, 2 * W, generator=g)
    out["warp"], out["certainty"] = warp.numpy(), certainty.numpy()
    # coordinates
    coords = torch.rand(50, 4, generator=g) * 2 - 1
    pa, pb = ref.to_pixel_coordinates(coords, 480, 640, 600, 800)
    out["coords"], out["pix_A"], out["pix_B"] = coords.numpy(), pa.numpy(), pb.numpy()
    out["pix_single"] = ref.to_pixel_coordinates(coords[:, :2], 480, 640).numpy()
    na, nb = ref.to_normalized_coordinates(torch.cat((pa, pb), dim=-1), 480, 640, 600, 800)
    out["norm_A"], out["norm_B"] = na.numpy(), nb.numpy()
    # match_keypoints on the A half of the warp: keypoints in A, their warped positions (+ noise / outliers) in B
    x_A = torch.rand(40, 2, generator=g) * 1.6 - 0.8
    wA, cA = warp[:, :W], certainty[:, :W]
    x_B_true = torch.nn.functional.grid_sample(wA[..., -2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False,
                                               mode="bilinear")[0, :, 0].mT
    x_B = x_B_true + 0.001 * torch.randn(40, 2, generator=g)
    x_B[::5] += 0.3                                             # every fifth keypoint has no counterpart
    x_B = x_B[torch.randperm(40, generator=g)]
    out["x_A"], out["x_B"] = x_A.numpy(), x_B.numpy()
    ia, ib = ref.match_keypoints(x_A, x_B, wA, cA, return_tuple=True, return_inds=True, max_dist=0.005, cert_th=0.2)
    out["kp_inds_A"], out["kp_inds_B"] = ia.numpy(), ib.numpy()
    m = ref.match_keypoints(x_A, x_B, wA, cA, return_tuple=False, return_inds=False, max_dist=0.005, cert_th=0.2)
    out["kp_cat"] = m.numpy()
    # forward-backward consistency (un-batched and batched)
    fb = ref.conf_from_fb_consistency(a_to_b, b_to_a, th=2)
    out["fb"] = fb.numpy()
    fb2 = ref.conf_from_fb_consistency(torch.stack((a_to_b, grid)), torch.stack((b_to_a, grid)), th=1)
    out["fb_batched"] = fb2.numpy()
    np.savez_compressed(os.path.join(HERE, "helpers.npz"), **out)
    print({k: v.shape for k, v in out.items()}, "matches:", len(out["kp_inds_A"]), "fb mean:", float(fb.mean()))
    # visualize_warp (matcher.py:936-989) on CPU: PIL inputs (symmetric and one-directional) and tensor inputs, plus the saved PNG
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from roma_b200 import synthetic
    import tempfile
    from PIL import Image
    im_a, im_b = synthetic.make_pil_pair(11, size_a=(50, 40), size_b=(45, 60))
    vis = {"vis_sym": ref.visualize_warp(warp, certainty, im_a, im_b, device="cpu").numpy(),
           "vis_one": ref.visualize_warp(warp[:, :W], certainty[:, :W], im_a, im_b, device="cpu", symmetric=False).numpy()}
    xa, xb = torch.rand(3, H, W, generator=g), torch.rand(3, H, W, generator=g)
    vis["x_A"], vis["x_B"] = xa.numpy(), xb.numpy()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "v.png")
        vis["vis_tensor"] = ref.visualize_warp(warp, certainty, xa, xb, device="cpu", save_path=path).numpy()
        vis["saved_png"] = np.asarray(Image.open(path))
    np.savez_compressed(os.path.join(HERE, "helpers_visualize.npz"), **vis)
    print({k: v.shape for k, v in vis.items()})


if __name__ == "__main__":
    main()
