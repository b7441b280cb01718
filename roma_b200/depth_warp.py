"""Depth-based ground-truth warps and the MegaDepth dense metric on the device: drop-ins for `romatch.utils.warp_kpts` and
`romatch.utils.get_gt_warp` (romatch/utils/utils.py:325-454), and the metric step of the MegaDepth dense harness,
`MegadepthDenseBenchmark.geometric_dist` (romatch/benchmarks/megadepth_dense_benchmark.py:17-42).

The reference casts the depth maps, the points, the pose and the intrinsics to float64 and runs about 25 eager kernels over
[B, L, 3] float64 temporaries.  Here the same float64 geometry is one kernel per call (`csrc/depth_warp.cu`, stated in
include/romab200.h): float32 depth maps and points are converted in registers, inv(K0) is computed on the device, and the harness's
mask gather and means are a fixed-order reduction.  Nothing is read back to the host and nothing synchronises, so a call can be
captured in a CUDA graph.  There is no CPU fallback.

    from roma_b200 import warp_kpts, get_gt_warp, dense_geometric_dist
    valid, warped = warp_kpts(kpts0, depth0, depth1, T_0to1, K0, K1)
    x2, prob = get_gt_warp(depth1, depth2, T_1to2, K1, K2)
    warp, certainty = model.match(im_A, im_B, batched=True)
    gd, pck_1, pck_3, pck_5, prob = res = dense_geometric_dist(depth1, depth2, T_1to2, K1, K2, warp[:, :, :W])
    res.epe, res.pair_sum, res.pair_count        # exact aggregation over a dataset: sum(pair_sum) / sum(pair_count[:, 0])
"""
from __future__ import annotations

import torch

from . import cabi
from .geometry import _device

# include/romab200.h: RB_DEPTH_WARP_MAX_CTAS
MAX_CTAS = 512
_MODES = {"bilinear": 0, "nearest": 1}
_DEPTH_CODE = {torch.float32: cabi.RB_F32, torch.float64: cabi.RB_F64}


class DenseGeometricDist(tuple):
    """The result of `dense_geometric_dist`: the tuple (gd, pck_1, pck_3, pck_5, prob) of the harness, whose items are also fields,
    plus `epe` (0-dim float64, the mean of gd over valid pixels), `pair_sum` (float64 [B], the sum of gd over the valid pixels of
    each pair) and `pair_count` (int64 [B, 4]: valid pixels and those with gd < 1, < 3, < 5 of each pair)."""

    def __new__(cls, gd, pck_1, pck_3, pck_5, prob, epe, pair_sum, pair_count):
        self = super().__new__(cls, (gd, pck_1, pck_3, pck_5, prob))
        self.gd, self.pck_1, self.pck_3, self.pck_5, self.prob = gd, pck_1, pck_3, pck_5, prob
        self.epe, self.pair_sum, self.pair_count = epe, pair_sum, pair_count
        return self


def _mode(depth_interpolation_mode):
    """The mode code of the kernels; what `F.grid_sample` rejects is rejected with its exception ("combined" in the reference runs
    `nearest-exact`, which `F.grid_sample` does not have, so it fails there too)."""
    if depth_interpolation_mode in _MODES:
        return _MODES[depth_interpolation_mode]
    if depth_interpolation_mode == "bicubic":
        raise NotImplementedError("depth_interpolation_mode='bicubic' is not implemented: the kernels sample 'bilinear' or 'nearest'")
    raise ValueError("nn.functional.grid_sample(): expected mode to be 'bilinear', 'nearest' or 'bicubic', but got: "
                     f"'{depth_interpolation_mode}'")


def _views(what, depth0, depth1, T, K0, K1, extra):
    """Validates the arguments the three functions share (shapes and dtypes first, then the device) and returns the keyword
    arguments of the C structs for them plus the device.  `extra`: name -> further tensor that must live on the same device."""
    named = dict(depth0=depth0, depth1=depth1, T=T, K0=K0, K1=K1, **extra)
    for name, t in named.items():
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{what}: `{name}` must be a torch.Tensor, got {type(t).__name__}")
    for name in ("depth0", "depth1"):
        d = named[name]
        if d.dim() != 3 or d.numel() == 0:
            raise ValueError(f"{what}: `{name}` must be a non-empty [B, H, W] depth map, got {tuple(d.shape)}")
        if d.dtype not in _DEPTH_CODE:
            raise TypeError(f"{what}: `{name}` must be float32 or float64, got {d.dtype}")
    B = depth0.shape[0]
    if depth1.shape[0] != B or B > 65535:
        raise ValueError(f"{what}: the depth maps must share a batch size of at most 65535, got {tuple(depth0.shape)} and {tuple(depth1.shape)}")
    if T.dim() != 3 or T.shape[0] != B or T.shape[1] not in (3, 4) or T.shape[2] != 4:
        raise ValueError(f"{what}: the pose must be [{B}, 3, 4] or [{B}, 4, 4], got {tuple(T.shape)}")
    for name in ("K0", "K1"):
        if tuple(named[name].shape) != (B, 3, 3):
            raise ValueError(f"{what}: `{name}` must be [{B}, 3, 3], got {tuple(named[name].shape)}")
    for name in ("T", "K0", "K1"):
        if not named[name].dtype.is_floating_point:
            raise TypeError(f"{what}: `{name}` must be a floating-point tensor, got {named[name].dtype}")
    _device(what)
    for name, t in named.items():
        if not t.is_cuda or t.device != depth0.device:
            raise RuntimeError(f"{what} runs on the GPU only (there is no CPU fallback): `{name}` lives on {t.device}, "
                               f"`depth0` on {depth0.device}")
    if depth0.dtype != depth1.dtype:              # one dtype code describes both maps; widening float32 is exact
        depth0, depth1 = depth0.double(), depth1.double()
    f64 = lambda t: t.detach().to(torch.float64).contiguous()      # noqa: E731
    return dict(depth0=depth0.detach().contiguous(), depth1=depth1.detach().contiguous(), depth_dtype=_DEPTH_CODE[depth0.dtype],
                h0=depth0.shape[1], w0=depth0.shape[2], h1=depth1.shape[1], w1=depth1.shape[2], T=f64(T), T_rows=T.shape[1],
                K0=f64(K0), K1=f64(K1), batch=B), depth0.device


def warp_kpts(kpts0, depth0, depth1, T_0to1, K0, K1, smooth_mask=False, return_relative_depth_error=False,
              depth_interpolation_mode="bilinear", relative_depth_error_threshold=0.05):
    """Drop-in for `romatch.utils.warp_kpts`: warps the normalised points kpts0 [B, L, 2] of view 0 into view 1 through depth0, the
    pose T_0to1 [B, 3 or 4, 4] and the intrinsics K0, K1 [B, 3, 3], and checks each for non-zero depth, covisibility (strictly
    inside depth1's image less one pixel) and depth consistency against depth1.  Returns (valid bool [B, L], warped float64
    [B, L, 2]); `warped` is defined for every point.  Depth maps and points may be float32 or float64 and are not copied.
    `smooth_mask` and `return_relative_depth_error` (used by the training losses only) raise NotImplementedError."""
    if smooth_mask:
        raise NotImplementedError("warp_kpts: smooth_mask is not implemented (it is used by the training losses only)")
    if return_relative_depth_error:
        raise NotImplementedError("warp_kpts: return_relative_depth_error is not implemented (it is used by the training losses only)")
    mode = _mode(depth_interpolation_mode)
    if isinstance(kpts0, torch.Tensor):
        if kpts0.dim() != 3 or kpts0.shape[2] != 2 or (isinstance(depth0, torch.Tensor) and kpts0.shape[0] != depth0.shape[0]):
            raise ValueError(f"warp_kpts: `kpts0` must be [B, L, 2] with the batch size of the depth maps, got {tuple(kpts0.shape)}")
        if kpts0.dtype not in _DEPTH_CODE:
            raise TypeError(f"warp_kpts: `kpts0` must be float32 or float64, got {kpts0.dtype}")
    kw, dev = _views("warp_kpts", depth0, depth1, T_0to1, K0, K1, dict(kpts0=kpts0))
    B, L = kpts0.shape[:2]
    with torch.cuda.device(dev):
        warped = torch.empty(B, L, 2, dtype=torch.float64, device=dev)
        valid = torch.empty(B, L, dtype=torch.uint8, device=dev)
        if L:
            cabi.call("romab200_warp_kpts", "rb_warp_kpts_args", **kw, mode=mode, rel_threshold=float(relative_depth_error_threshold),
                      kpts=kpts0.detach().contiguous(), kpts_dtype=_DEPTH_CODE[kpts0.dtype], L=L, warped=warped, valid=valid)
    return valid.bool(), warped


def get_gt_warp(depth1, depth2, T_1to2, K1, K2, depth_interpolation_mode="bilinear", relative_depth_error_threshold=0.05, H=None, W=None):
    """Drop-in for `romatch.utils.get_gt_warp`: `warp_kpts` at the pixel centres of an H x W image of view 1 (default: depth1's
    size), generated in the kernel from the two float32 linspaces the reference builds.  Returns (x2 float64 [B, H, W, 2], prob
    float32 [B, H, W])."""
    mode = _mode(depth_interpolation_mode)
    if (H is None) != (W is None):
        raise ValueError(f"get_gt_warp: give both H and W or neither, got H={H}, W={W}")
    kw, dev = _views("get_gt_warp", depth1, depth2, T_1to2, K1, K2, {})
    if H is None:
        H, W = depth1.shape[1:]
    H, W = int(H), int(W)
    if H < 1 or W < 1:
        raise ValueError(f"get_gt_warp: H and W must be positive, got H={H}, W={W}")
    B = kw["batch"]
    with torch.cuda.device(dev):
        grid_x, grid_y = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n, device=dev, dtype=torch.float32) for n in (W, H))
        x2 = torch.empty(B, H, W, 2, dtype=torch.float64, device=dev)
        prob = torch.empty(B, H, W, dtype=torch.float32, device=dev)
        cabi.call("romab200_gt_warp", "rb_gt_warp_args", **kw, mode=mode, rel_threshold=float(relative_depth_error_threshold),
                  grid_x=grid_x, grid_y=grid_y, H=H, W=W, x2=x2, prob=prob)
    return x2, prob


def dense_geometric_dist(depth1, depth2, T_1to2, K1, K2, dense_matches):
    """The metric step of the MegaDepth dense harness, `MegadepthDenseBenchmark.geometric_dist`: the end-point error in pixels
    between a dense warp and the depth-based ground truth, and PCK@1/3/5 over the valid pixels.  dense_matches [B, H, W, 4]
    float32 holds (x1, y1, x2, y2) in normalised coordinates and is read through its strides: pass the left half of a symmetric
    warp as the view `warp[:, :, :W]`.
    Returns (gd, pck_1, pck_3, pck_5, prob) in the harness's order, as a `DenseGeometricDist` that also has `epe`, `pair_sum` and
    `pair_count`.  One deliberate difference: gd is the dense float64 [B, H, W] map, NaN where prob != 1, not the harness's compacted
    vector, whose data-dependent length would cost a read back; the vector is `gd[prob == 1]` and its mean is `epe`.  pck_* are
    0-dim float32 tensors bit-equal to `(gd[prob == 1] < t).float().mean()`; without a valid pixel they and epe are NaN."""
    what = "dense_geometric_dist"
    if isinstance(dense_matches, torch.Tensor):
        if dense_matches.dim() != 4 or dense_matches.shape[3] != 4 or dense_matches.numel() == 0 or \
                (isinstance(depth1, torch.Tensor) and dense_matches.shape[0] != depth1.shape[0]):
            raise ValueError(f"{what}: `dense_matches` must be a non-empty [B, H, W, 4] warp with the batch size of the depth maps, "
                             f"got {tuple(dense_matches.shape)}")
        if dense_matches.dtype != torch.float32:
            raise TypeError(f"{what}: `dense_matches` must be float32, got {dense_matches.dtype}")
    kw, dev = _views(what, depth1, depth2, T_1to2, K1, K2, dict(dense_matches=dense_matches))
    B, H, W, _ = dense_matches.shape
    dm = dense_matches.detach()
    with torch.cuda.device(dev):
        f64 = dict(dtype=torch.float64, device=dev)
        gd, prob = torch.empty(B, H, W, **f64), torch.empty(B, H, W, dtype=torch.float32, device=dev)
        pair_sum, pair_count = torch.empty(B, **f64), torch.empty(B, 4, dtype=torch.int64, device=dev)
        pck, epe = torch.empty(3, dtype=torch.float32, device=dev), torch.empty(1, **f64)
        cabi.call("romab200_dense_geometric_dist", "rb_dense_geometric_dist_args", **kw, rel_threshold=0.05,
                  dense_matches=dm, dm_sb=dm.stride(0), dm_sy=dm.stride(1), dm_sx=dm.stride(2), dm_sc=dm.stride(3), H=H, W=W,
                  gd=gd, prob=prob, partial_sum=torch.empty(B, MAX_CTAS, **f64),
                  partial_cnt=torch.empty(B, MAX_CTAS, 4, dtype=torch.int32, device=dev), pair_sum=pair_sum, pair_cnt=pair_count,
                  pck=pck, epe=epe)
    return DenseGeometricDist(gd, pck[0], pck[1], pck[2], prob, epe[0], pair_sum, pair_count)
