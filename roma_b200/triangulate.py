"""Triangulation of feature tracks with known cameras on the device (`triangulate_tracks`), COLMAP's `point_triangulator` for cameras
that come from a calibrated rig, GPS/INS or ground truth: per track a two-view RANSAC over its observations, a multi-view DLT and
Gauss-Newton over the inliers, then reprojection and angle filters.  The exact rules are in include/romab200.h and INTEGRATION.md;
`oracle/triangulate.py` restates them in numpy."""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass

import numpy as np
import torch

from . import cabi
from .match_graph import MatchGraph
from .tracks import Tracks


@dataclass
class Points3D:
    """Per track k: X[k] float64 [3] world point, ok[k] bool, num_inliers[k] int32 and error[k] float64 (the mean reprojection error
    in px of the inliers); X, num_inliers and error are zero where the track is not ok.  inlier [E] bool, aligned with
    tracks.elements, is all false for a track that is not ok.  Tensors live on the graph's device."""
    X: torch.Tensor
    ok: torch.Tensor
    num_inliers: torch.Tensor
    error: torch.Tensor
    inlier: torch.Tensor


def _float64(name, v, shape, what="triangulate_tracks"):
    """A float camera array (tensor on any device, or array-like) widened to a float64 numpy array of `shape`, all finite."""
    if isinstance(v, torch.Tensor):
        if not v.dtype.is_floating_point:
            raise ValueError(f"{what}: {name} must have a float dtype, got {v.dtype}")
        v = v.detach().cpu().double().numpy()
    else:
        v = np.asarray(v)
        if v.dtype.kind != "f":
            raise ValueError(f"{what}: {name} must have a float dtype, got {v.dtype}")
        v = v.astype(np.float64)
    if v.shape != shape:
        raise ValueError(f"{what}: {name} must have shape {list(shape)}, got {list(v.shape)}")
    if not np.isfinite(v).all():
        raise ValueError(f"{what}: {name} has values that are not finite")
    return v


def camera_table(K, R, t) -> np.ndarray:
    """The float64 camera table of rule 1, [N, RB_TRI_CAM] per image: P = K [R | t] (12, row-major), row 2 of R, t_z, C = -R^T t, and
    the exclusion flag 0 (triangulate_tracks sets it to 1 for the images not among `images`)."""
    N = K.shape[0]
    tab = np.zeros((N, cabi.RB_TRI_CAM))
    tab[:, :12] = (K @ np.concatenate((R, t[:, :, None]), 2)).reshape(N, 12)
    tab[:, 12:15] = R[:, 2]
    tab[:, 15] = t[:, 2]
    tab[:, 16:19] = -np.einsum("nji,nj->ni", R, t)
    return tab


def image_list(images, N, what):
    """`images`: distinct ints in [0, N), as a list, or ValueError."""
    images = images.tolist() if isinstance(images, (torch.Tensor, np.ndarray)) else list(images)
    try:
        if any(isinstance(i, (bool, np.bool_)) for i in images):
            raise TypeError
        out = [operator.index(i) for i in images]
    except TypeError:
        raise ValueError(f"{what}: images must hold ints, got {images!r}") from None
    if any(not 0 <= i < N for i in out):
        raise ValueError(f"{what}: images must lie in [0, {N}), got {out}")
    if len(set(out)) != len(out):
        raise ValueError(f"{what}: images must be distinct, got {out}")
    return out


def _check(graph, tracks, K, R, t, max_error, min_angle, max_hypotheses, seed, what="triangulate_tracks", device=True):
    """Argument rules, checked before any device work; `what` names the caller in the messages, and `device=False` leaves the
    device rule to the caller.  Returns (kp_offsets list, track_offsets list, camera table, max_error^2, min_angle in radians,
    max_hypotheses, seed)."""
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"{what}: graph must be a MatchGraph, got {type(graph).__name__}")
    if not isinstance(tracks, Tracks):
        raise ValueError(f"{what}: tracks must be Tracks, got {type(tracks).__name__}")
    kp_off = graph._kp_off
    for name, tv in (("graph.kp_offsets", graph.kp_offsets), ("tracks.track_offsets", tracks.track_offsets)):
        if not isinstance(tv, torch.Tensor) or tv.dtype != torch.int64 or tv.dim() != 1 or tv.numel() < 1:
            raise ValueError(f"{what}: {name} must be a 1-D int64 tensor of at least one entry, got "
                             f"{getattr(tv, 'dtype', type(tv).__name__)} {tuple(getattr(tv, 'shape', ()))}")
    tr_off = tracks.track_offsets.tolist()
    for name, off in (("graph.kp_offsets", kp_off), ("tracks.track_offsets", tr_off)):
        if off[0] != 0 or any(b < a for a, b in zip(off, off[1:])):
            raise ValueError(f"{what}: {name} must start at 0 and never decrease")
    N, Kr, T, E = len(kp_off) - 1, kp_off[-1], len(tr_off) - 1, tr_off[-1]
    if not isinstance(graph.keypoints, torch.Tensor) or graph.keypoints.dtype != torch.float32 or tuple(graph.keypoints.shape) != (Kr, 2):
        raise ValueError(f"{what}: graph.keypoints must be fp32 [{Kr}, 2], got {getattr(graph.keypoints, 'dtype', None)} "
                         f"{tuple(getattr(graph.keypoints, 'shape', ()))}")
    el = tracks.elements
    if not isinstance(el, torch.Tensor) or el.dtype != torch.int32 or tuple(el.shape) != (E, 2):
        raise ValueError(f"{what}: tracks.elements must be int32 [{E}, 2], got {getattr(el, 'dtype', None)} "
                         f"{tuple(getattr(el, 'shape', ()))}")
    if E >= 1 << 31:
        raise ValueError(f"{what}: {E} elements, at most 2^31 - 1 are supported")
    if T >= 1 << 31:
        raise ValueError(f"{what}: {T} tracks, at most 2^31 - 1 are supported")
    if N < 1:
        raise ValueError(f"{what}: the graph has no images")
    K = _float64("K", K, (N, 3, 3), what)
    R = _float64("R", R, (N, 3, 3), what)
    t = _float64("t", t, (N, 3), what)
    try:
        max_error, min_angle = float(max_error), float(min_angle)
    except (TypeError, ValueError):
        raise ValueError(f"{what}: max_error and min_angle must be numbers, got {max_error!r} and {min_angle!r}") from None
    if not (math.isfinite(max_error) and max_error > 0):
        raise ValueError(f"{what}: max_error must be finite and > 0, got {max_error!r}")
    if not 0 <= min_angle < 180:
        raise ValueError(f"{what}: min_angle must lie in [0, 180) degrees, got {min_angle!r}")
    bad = isinstance(max_hypotheses, bool)
    try:
        max_hypotheses = operator.index(max_hypotheses)
    except TypeError:
        bad = True
    if bad or not 1 <= max_hypotheses < 1 << 31:
        raise ValueError(f"{what}: max_hypotheses must be an int in [1, 2^31), got {max_hypotheses!r}")
    try:
        seed = operator.index(seed)
    except TypeError:
        raise ValueError(f"{what}: seed must be an int, got {seed!r}") from None
    if isinstance(seed, bool) or not 0 <= seed < 1 << 64:
        raise ValueError(f"{what}: seed must be an int in [0, 2^64), got {seed!r}")
    if Kr == 0 and E > 0:
        raise ValueError(f"{what}: the graph has no keypoints, so every element id is out of range")
    if device:
        _check_device([graph.kp_offsets, graph.keypoints, tracks.track_offsets, el], what)
    return kp_off, tr_off, camera_table(K, R, t), max_error * max_error, min_angle * (math.pi / 180.0), max_hypotheses, seed


def _check_device(tensors, what):
    dev = tensors[0].device
    if not all(tv.is_cuda and tv.device == dev for tv in tensors):
        raise ValueError(f"{what}: the graph's and tracks' tensors must be on one CUDA device, got {[tv.device for tv in tensors]}")


def triangulate_tracks(graph: MatchGraph, tracks: Tracks, K, R, t, *, max_error=4.0, min_angle=1.5, max_hypotheses=256,
                       seed=0, images=None) -> Points3D:
    """The 3-D point of every track of `tracks` (built from `graph`) seen by cameras x ~ K[i] (R[i] X + t[i]) in pixels of the
    image_sizes frame (x = (W / 2) (u + 1), `synthetic.planted_cameras`' convention).  K, R [N, 3, 3] and t [N, 3] are tensors or
    arrays of any float dtype, widened to float64 on the host.  Only graph.kp_offsets and graph.keypoints are read.

    Per track: a two-view DLT for every pair of its observations, or for `max_hypotheses` pairs drawn from the Philox stream of `seed`
    when it has more; the point with the most observations within `max_error` px (and in front of their cameras) wins, ties to the
    first; a multi-view DLT and at most RB_TRI_GN_ITERS Gauss-Newton steps over those inliers refine it; the inliers are recomputed
    once, and the track is ok when two of them, in distinct images, see the point under an angle of at least `min_angle` degrees.
    `images` (distinct ints in [0, N), or None for all) lists the registered cameras: an element of any other image is not an
    observation, a pair that contains it is skipped but keeps its index, and it is never an inlier, so the cameras of the other images
    are not used (they must still be finite).  With images=None the result is byte-identical to the call without the argument.
    The defaults of max_error (4 px) and min_angle (1.5 degrees) are COLMAP's triangulator.  With keypoints snapped to 1 px cells
    (`consolidate_matches`) and 0.5 px noise, the largest reprojection error of a true observation is about 2 px, so 4 px keeps them
    all; the cell's quantisation grows with cell_size, and at cell_size 4 it reaches about 4 px, so the default cuts a few true
    observations there and about 6 px keeps them.

    Bit-identical from run to run.  Arguments are checked before any device work; an element id outside its image's keypoints raises
    ValueError (the device checks every id before using it).  Host reads: the track offsets and the status word."""
    kp_off, tr_off, table, max_error2, min_angle, max_hypotheses, seed = _check(graph, tracks, K, R, t, max_error, min_angle,
                                                                                max_hypotheses, seed)
    N, T, E = len(kp_off) - 1, len(tr_off) - 1, tr_off[-1]
    if images is not None:
        registered = np.zeros(N, bool)
        registered[image_list(images, N, "triangulate_tracks")] = True
        table[:, 19] = np.where(registered, 0.0, 1.0)
    dev = graph.kp_offsets.device
    with torch.cuda.device(dev):
        X = torch.zeros(T, 3, dtype=torch.float64, device=dev)
        ok = torch.zeros(T, dtype=torch.uint8, device=dev)
        num_inliers = torch.zeros(T, dtype=torch.int32, device=dev)
        error = torch.zeros(T, dtype=torch.float64, device=dev)
        inlier = torch.zeros(E, dtype=torch.uint8, device=dev)
        if T > 0 and E > 0:
            # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
            info = torch.empty(1, dtype=torch.int64, device=dev)
            cabi.call("romab200_triangulate", "rb_tri_args", num_tracks=T, num_images=N,
                      track_offsets=torch.tensor(tr_off, dtype=torch.int64).to(dev, non_blocking=True), elements=tracks.elements.contiguous(),
                      num_elements=E, kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev, non_blocking=True),
                      keypoints=graph.keypoints.contiguous(), num_rows=kp_off[-1], cameras=torch.from_numpy(table).to(dev),
                      max_error2=max_error2, min_angle=min_angle, max_hypotheses=max_hypotheses, seed=seed, info=info, X=X, ok=ok,
                      num_inliers=num_inliers, error=error, inlier=inlier)
            if int(info[0].item()) & cabi.RB_TRI_BAD_ID:
                raise ValueError("triangulate_tracks: a track element lies outside its image's keypoints")
    return Points3D(X, ok.bool(), num_inliers, error, inlier.bool())
