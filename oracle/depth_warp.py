"""Torch float64 statement of the depth-based warps and of the MegaDepth dense metric, written from the formulas in
include/romab200.h: the oracle of `roma_b200.depth_warp` (csrc/depth_warp.cu).

It runs on whatever device its inputs live on.  On the CPU it is what the tests compare the kernels with; on a GPU it is the
eager torch statement a user would otherwise run (about 25 kernels over [B, L, 3] float64 temporaries), which
scripts/bench_depth_warp.py times against the fused kernels.

    valid, warped = warp_kpts(kpts0, depth0, depth1, T_0to1, K0, K1)
    x2, prob = get_gt_warp(depth1, depth2, T_1to2, K1, K2)
    out = dense_geometric_dist(depth1, depth2, T_1to2, K1, K2, dense_matches)     # dict: gd, prob, pck, epe, pair_sum, pair_count
"""
import torch
import torch.nn.functional as F

THRESHOLDS = (1.0, 3.0, 5.0)


def _sample(depth, pts, mode):
    """depth [B, h, w] at the normalised points [B, L, 2]: zero padding, align_corners=False -> [B, L]."""
    return F.grid_sample(depth[:, None], pts[:, :, None], mode=mode, align_corners=False)[:, 0, :, 0]


def _pixels(pts, h, w):
    """Normalised (x, y) -> pixel coordinates (w (x + 1) / 2, h (y + 1) / 2), in the dtype of `pts`."""
    return torch.stack((w * (pts[..., 0] + 1) / 2, h * (pts[..., 1] + 1) / 2), dim=-1)


@torch.no_grad()
def warp_kpts(kpts0, depth0, depth1, T_0to1, K0, K1, depth_interpolation_mode="bilinear", relative_depth_error_threshold=0.05, details=None):
    """(valid bool [B, L], warped float64 [B, L, 2]).  `details`, when a dict, receives u, v (pixel position in view 1) and rel (the
    relative depth error), with which a test can tell a point that sits on a decision boundary."""
    kpts0, depth0, depth1, T, K0, K1 = (a.double() for a in (kpts0, depth0, depth1, T_0to1, K0, K1))
    (h0, w0), (h1, w1) = depth0.shape[1:], depth1.shape[1:]
    d0 = _sample(depth0, kpts0, depth_interpolation_mode)
    homog = torch.cat((_pixels(kpts0, h0, w0), torch.ones_like(d0)[..., None]), dim=-1) * d0[..., None]      # [B, L, 3]
    cam0 = homog @ torch.linalg.inv(K0).mT
    cam1 = cam0 @ T[:, :3, :3].mT + T[:, None, :3, 3]
    z = cam1[..., 2]
    proj = cam1 @ K1.mT
    uv = proj[..., :2] / (proj[..., 2:] + 1e-4)
    u, v = uv[..., 0], uv[..., 1]
    covisible = (u > 0) & (u < w1 - 1) & (v > 0) & (v < h1 - 1)
    warped = torch.stack((2 * u / w1 - 1, 2 * v / h1 - 1), dim=-1)
    d1 = _sample(depth1, warped, depth_interpolation_mode)
    rel = ((d1 - z) / d1).abs()
    if details is not None:
        details.update(u=u, v=v, rel=rel, d0=d0)
    return (d0 != 0) & covisible & (rel < relative_depth_error_threshold), warped


@torch.no_grad()
def get_gt_warp(depth1, depth2, T_1to2, K1, K2, depth_interpolation_mode="bilinear", relative_depth_error_threshold=0.05, H=None, W=None,
                details=None):
    """(x2 float64 [B, H, W, 2], prob float32 [B, H, W]): `warp_kpts` at the pixel centres of an H x W image (default: depth1's size).
    The centres are float32 linspaces widened to float64, as the reference has them."""
    B = depth1.shape[0]
    if H is None:
        H, W = depth1.shape[1:]
    xs, ys = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n, device=depth1.device, dtype=torch.float32) for n in (W, H))
    grid = torch.stack((xs[None, :].expand(H, W), ys[:, None].expand(H, W)), dim=-1).reshape(1, H * W, 2).expand(B, -1, -1)
    valid, x2 = warp_kpts(grid.double(), depth1, depth2, T_1to2, K1, K2, depth_interpolation_mode, relative_depth_error_threshold, details)
    return x2.reshape(B, H, W, 2), valid.float().reshape(B, H, W)


@torch.no_grad()
def dense_geometric_dist(depth1, depth2, T_1to2, K1, K2, dense_matches, details=None):
    """The metric step of the MegaDepth dense harness on a warp `dense_matches` [B, H, W, 4] float32.  Returns a dict:
    gd float64 [B, H, W] (the end-point error in pixels, NaN where prob != 1), prob float32 [B, H, W], pck float32 [3] (the
    fraction of valid pixels with gd < 1, 3, 5), epe float64 (mean gd over valid pixels), pair_sum float64 [B] and pair_count
    int64 [B, 4] (valid, < 1, < 3, < 5 per pair).  The harness's compacted vector is gd[prob == 1]."""
    B, H, W, _ = dense_matches.shape
    valid, x2 = warp_kpts(dense_matches[..., :2].reshape(B, H * W, 2), depth1, depth2, T_1to2, K1, K2, details=details)
    truth = _pixels(x2, H, W).reshape(B, H, W, 2)
    pred = _pixels(dense_matches[..., 2:], H, W)                      # float32 arithmetic, as the harness has it
    gd = (pred - truth).norm(dim=-1)
    prob = valid.float().reshape(B, H, W)
    on = prob == 1
    picked = gd[on]
    nan = torch.full_like(gd, float("nan"))
    return {"gd": torch.where(on, gd, nan), "prob": prob,
            "pck": torch.stack([(picked < t).float().mean() for t in THRESHOLDS]), "epe": picked.mean(),
            "pair_sum": torch.where(on, gd, torch.zeros_like(gd)).sum(dim=(1, 2)),
            "pair_count": torch.stack([on.sum(dim=(1, 2))] + [(on & (gd < t)).sum(dim=(1, 2)) for t in THRESHOLDS], dim=1)}
