"""SIMPLE_RADIAL cameras (COLMAP's camera model 2) and keypoint undistortion on the device.

Camera i has the intrinsics (f, cx, cy, k), in COLMAP's parameter order, and maps a camera-frame point p to the pixel

    x = p0 / p2,  y = p1 / p2,  r^2 = x^2 + y^2,  d = 1 + k r^2,  u = f d x + cx,  v = f d y + cy.

`undistort_graph` maps every keypoint of a match graph to where the same camera without distortion (the pinhole K of
`pinhole_K`) would see it, so that the stages that take pinhole cameras (`triangulate_tracks`, `register_images`,
`initialize_reconstruction`) can run on photographs with radial distortion.  The exact rules are in include/romab200.h;
`oracle/camera.py` restates them in numpy."""
from __future__ import annotations

import copy

import numpy as np
import torch

from . import cabi
from .match_graph import MatchGraph


def default_intrinsics(image_sizes) -> np.ndarray:
    """COLMAP's prior for images of unknown calibration, float64 [N, 4] (f, cx, cy, k): f = 1.2 max(W, H), the principal point at the
    image centre (W / 2, H / 2: the pixel frame of this project is COLMAP's, whose pixel (0, 0) covers [0, 1)^2) and k = 0.
    `image_sizes` is [N, 2] (H, W), as `consolidate_matches` takes it."""
    s = image_sizes.detach().cpu().numpy() if isinstance(image_sizes, torch.Tensor) else np.asarray(image_sizes)
    if s.ndim != 2 or s.shape[1] != 2 or s.shape[0] < 1 or s.dtype.kind not in "iuf" or not (np.isfinite(s).all() and (s > 0).all()):
        raise ValueError(f"default_intrinsics: image_sizes must be [N, 2] positive (H, W), got {s.dtype} {list(s.shape)}")
    H, W = s[:, 0].astype(np.float64), s[:, 1].astype(np.float64)
    return np.stack((1.2 * np.maximum(W, H), W / 2, H / 2, np.zeros_like(W)), 1)


def check_intrinsics(intrinsics, N: int, what: str) -> np.ndarray:
    """SIMPLE_RADIAL intrinsics (a float tensor or array) widened to float64 [N, 4] on the host: finite, with every f > 0."""
    if isinstance(intrinsics, torch.Tensor):
        if not intrinsics.dtype.is_floating_point:
            raise ValueError(f"{what}: intrinsics must have a float dtype, got {intrinsics.dtype}")
        v = intrinsics.detach().cpu().double().numpy()
    else:
        v = np.asarray(intrinsics)
        if v.dtype.kind != "f":
            raise ValueError(f"{what}: intrinsics must have a float dtype, got {v.dtype}")
        v = v.astype(np.float64)
    if v.shape != (N, 4):
        raise ValueError(f"{what}: intrinsics must have shape [{N}, 4] (f, cx, cy, k), got {list(v.shape)}")
    if not np.isfinite(v).all() or not (v[:, 0] > 0).all():
        raise ValueError(f"{what}: intrinsics must be finite with every focal length > 0")
    return v


def pinhole_K(intrinsics):
    """[N, 3, 3] [[f, 0, cx], [0, f, cy], [0, 0, 1]] of SIMPLE_RADIAL intrinsics [N, 4]: the camera of the undistorted keypoints.  A
    tensor gives a float64 tensor on its device, anything else a float64 numpy array."""
    if isinstance(intrinsics, torch.Tensor):
        c = intrinsics.double()
        K = torch.zeros(c.shape[0], 3, 3, dtype=torch.float64, device=c.device)
    else:
        c = np.asarray(intrinsics, np.float64)
        K = np.zeros((c.shape[0], 3, 3))
    if c.ndim != 2 or c.shape[1] != 4:
        raise ValueError(f"pinhole_K: intrinsics must be [N, 4] (f, cx, cy, k), got {list(c.shape)}")
    K[:, 0, 0] = K[:, 1, 1] = c[:, 0]
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = c[:, 1], c[:, 2], 1.0
    return K


def undistort_keypoints(graph: MatchGraph, intrinsics):
    """The graph's keypoints undistorted under `intrinsics` [N, 4] (include/romab200.h): (keypoints fp32 [K, 2], clamped int64 [1])
    on the graph's device.  clamped counts the keypoints at or beyond the turning point of a k < 0 camera, which are put at the
    turning radius in their own direction.  Arguments are checked before any device work."""
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"undistort_keypoints: graph must be a MatchGraph, got {type(graph).__name__}")
    kp_off = graph._kp_off
    N, Kr = len(kp_off) - 1, kp_off[-1]
    if N < 1:
        raise ValueError("undistort_keypoints: the graph has no images")
    kp = graph.keypoints
    if not isinstance(kp, torch.Tensor) or kp.dtype != torch.float32 or tuple(kp.shape) != (Kr, 2):
        raise ValueError(f"undistort_keypoints: graph.keypoints must be fp32 [{Kr}, 2], got {getattr(kp, 'dtype', None)} "
                         f"{tuple(getattr(kp, 'shape', ()))}")
    c = check_intrinsics(intrinsics, N, "undistort_keypoints")
    if not kp.is_cuda:
        raise ValueError(f"undistort_keypoints: graph.keypoints must be on a CUDA device, got {kp.device}")
    dev = kp.device
    with torch.cuda.device(dev):
        out = torch.empty_like(kp)
        clamped = torch.empty(1, dtype=torch.int64, device=dev)
        # the offsets the graph was built with (its host list), so nothing is read back
        cabi.call("romab200_undistort_keypoints", "rb_undistort_args", num_images=N, num_rows=Kr,
                  kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev), keypoints=kp.contiguous(),
                  intrinsics=torch.from_numpy(c).to(dev), out=out, clamped=clamped)
    return out, clamped


def undistort_graph(graph: MatchGraph, intrinsics) -> MatchGraph:
    """A MatchGraph whose keypoints are `graph`'s undistorted under SIMPLE_RADIAL `intrinsics` [N, 4]; every other tensor, and the
    host offset lists, are shared with `graph`.  Run the pinhole stages on it with `pinhole_K(intrinsics)`."""
    kp, _ = undistort_keypoints(graph, intrinsics)
    out = copy.copy(graph)                                # keeps the host offset lists: no read-back
    out.keypoints = kp
    return out
