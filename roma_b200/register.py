"""Image registration against triangulated tracks on the device (`register_images`): the absolute pose of listed images from their
keypoints that lie on ok tracks, COLMAP's EstimateAbsolutePose + RefineAbsolutePose, the step of its incremental mapper that adds a
camera to a reconstruction.  With `triangulate_tracks(..., images=...)` and `bundle_adjust` (the unregistered cameras in
fixed_poses) it grows a reconstruction from two known cameras to all of them without leaving the device.  The exact rules are in
include/romab200.h and INTEGRATION.md; `oracle/absolute_pose.py` restates them in numpy."""
from __future__ import annotations

import operator
from dataclasses import dataclass

import numpy as np
import torch

from . import cabi, geometry
from . import triangulate as _tri
from .match_graph import WORKSPACE_BYTES, MatchGraph
from .tracks import Tracks
from .triangulate import Points3D


@dataclass
class Registration:
    """Per listed image m: images[m] int64 (as given), R[m] float64 [3, 3] and t[m] [3] (x ~ K (R X + t); zero where not ok), ok[m]
    bool (a model was found), num_correspondences[m] and num_inliers[m] int64, accepted[m] bool (ok and num_inliers >= min_inliers).
    inlier [E] bool, aligned with tracks.elements, holds the inlier elements of the accepted images.  Tensors live on the graph's
    device."""
    images: torch.Tensor
    R: torch.Tensor
    t: torch.Tensor
    ok: torch.Tensor
    accepted: torch.Tensor
    num_correspondences: torch.Tensor
    num_inliers: torch.Tensor
    inlier: torch.Tensor


def chunk_bytes(ns) -> int:
    """Device bytes of one estimator chunk whose images have ns[m] correspondences (include/romab200.h): the buffers
    `geometry._abs_launch` allocates plus the gathered points, the image list and the packed offsets."""
    S = cabi.abspose_splits(max(ns))
    return (len(ns) * (cabi.RB_REG_ITEM_BYTES + cabi.RB_REG_SLICE_BYTES * S) + cabi.RB_REG_POINT_BYTES * max(sum(ns), 1)
            + cabi.RB_REG_CHUNK_BYTES)


def plan_chunks(ns, workspace_bytes) -> list:
    """Consecutive ranges [b, e) of the listed images covering all of them: each run is as long as `chunk_bytes` of its images stays
    within `workspace_bytes` and it holds at most RB_ABS_MAX_BATCH images; an image over the budget alone gets a chunk of its own."""
    chunks, b, M = [], 0, len(ns)
    while b < M:
        e = b + 1
        while e < M and e - b < cabi.RB_ABS_MAX_BATCH and chunk_bytes(ns[b:e + 1]) <= workspace_bytes:
            e += 1
        chunks.append((b, e))
        b = e
    return chunks


def _int(name, v, lo):
    if isinstance(v, bool):
        raise ValueError(f"register_images: {name} must be an int >= {lo}, got {v!r}")
    try:
        v = operator.index(v)
    except TypeError:
        raise ValueError(f"register_images: {name} must be an int >= {lo}, got {v!r}") from None
    if v < lo:
        raise ValueError(f"register_images: {name} must be an int >= {lo}, got {v!r}")
    return v


def _check(graph, tracks, points, K, images, max_error, confidence, max_iters, min_inliers, seed, workspace_bytes):
    """Argument rules, checked before any device work.  Returns (kp_offsets, track_offsets, K float64 [N, 3, 3], images, max_error^2,
    confidence, max_iters, min_inliers, seed, workspace_bytes)."""
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"register_images: graph must be a MatchGraph, got {type(graph).__name__}")
    N = len(graph._kp_off) - 1
    kp_off, tr_off, *_ = _tri._check(graph, tracks, K, np.tile(np.eye(3), (max(N, 0), 1, 1)), np.zeros((max(N, 0), 3)), 1.0, 0.0, 1, 0,
                                     what="register_images", device=False)
    T = len(tr_off) - 1
    K = _tri._float64("K", K, (N, 3, 3), "register_images")
    if not isinstance(points, Points3D):
        raise ValueError(f"register_images: points must be Points3D, got {type(points).__name__}")
    for name, v, dt, shape in (("points.X", points.X, torch.float64, (T, 3)), ("points.ok", points.ok, torch.bool, (T,))):
        if not isinstance(v, torch.Tensor) or v.dtype != dt or tuple(v.shape) != shape:
            raise ValueError(f"register_images: {name} must be {dt} {list(shape)} (aligned with tracks), got "
                             f"{getattr(v, 'dtype', type(v).__name__)} {tuple(getattr(v, 'shape', ()))}")
    images = _tri.image_list(images, N, "register_images")
    try:
        max_error2, confidence, max_iters, seed = geometry._abs_args(max_error, confidence, max_iters, seed)
    except ValueError as e:
        raise ValueError(f"register_images: {e}") from None
    min_inliers = _int("min_inliers", min_inliers, 0)
    workspace_bytes = _int("workspace_bytes", workspace_bytes, 1)
    _tri._check_device([graph.kp_offsets, graph.keypoints, tracks.track_offsets, tracks.elements, points.X, points.ok], "register_images")
    if not bool(torch.isfinite(points.X).all()):
        raise ValueError("register_images: points.X has values that are not finite")
    return kp_off, tr_off, K, images, max_error2, confidence, max_iters, min_inliers, seed, workspace_bytes


def register_images(graph: MatchGraph, tracks: Tracks, points: Points3D, K, images, *, max_error=12.0, confidence=0.9999, max_iters=10000,
                    min_inliers=30, seed=0, workspace_bytes=WORKSPACE_BYTES) -> Registration:
    """The pose of every image of `images` (distinct ints in [0, N)) from its correspondences with the ok tracks of `points` (from
    `triangulate_tracks` on the same graph and tracks): the elements (i, a) of ok tracks k, in element order, each pairing
    x = graph.keypoints[kp_offsets[i] + a] with X = points.X[k].  points.inlier is not consulted, since an unregistered image's
    elements are never triangulation inliers; a track with two elements in one image gives two correspondences.  K [N, 3, 3] is a
    tensor or array of any float dtype.  Image m's result is bit-identical to `estimate_absolute_pose_batched` on its correspondences
    alone (the same max_error px, confidence, max_iters and seed), whatever the other images, their order and workspace_bytes.  It
    is accepted when a model was found with at least `min_inliers` inliers.

    The defaults of max_error (12 px) and min_inliers (30) are COLMAP's mapper.  On `synthetic.planted_cameras` scenes (0.5 px noise,
    cells of 1 or 4 px, 20 % outlier samples through `verify_matches`, cameras 0 and 1 known) this accepts every image of the test
    scenes at N = 3 and 8 at either cell size, and at N = 30 with 300 points the 23 and 27 of 30 images that see 30 inlier tracks
    of the two known cameras; an incremental loop over N = 10 images then registers all of them.

    The gather runs on the device: every element id is checked (a bad one raises ValueError before any kernel indexes with it),
    radix_sort_hi32 orders the ok tracks' elements by image, and each chunk of images (at most `workspace_bytes` of estimator
    buffers, 1 GiB by default; an image over the budget runs alone) is packed for the estimator.  Bit-identical from run to run.
    Host reads: the status word, the per-image correspondence counts (N + 1 int64), and the estimator's `running` flag once per chunk
    and round of RB_ABS_ROUND hypotheses before the last."""
    kp_off, tr_off, K, images, max_error2, conf, max_iters, min_inliers, seed, workspace_bytes = _check(
        graph, tracks, points, K, images, max_error, confidence, max_iters, min_inliers, seed, workspace_bytes)
    N, T, E, M = len(kp_off) - 1, len(tr_off) - 1, tr_off[-1], len(images)
    dev = graph.kp_offsets.device
    with torch.cuda.device(dev):
        R = torch.zeros(M, 3, 3, dtype=torch.float64, device=dev)
        t = torch.zeros(M, 3, dtype=torch.float64, device=dev)
        ok = torch.zeros(M, dtype=torch.uint8, device=dev)
        num_inliers = torch.zeros(M, dtype=torch.int64, device=dev)
        inlier = torch.zeros(E, dtype=torch.bool, device=dev)
        counts = [0] * M
        if M and T and E:
            # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
            tiles = (E + cabi.RB_TRACKS_TILE - 1) // cabi.RB_TRACKS_TILE
            kw = dict(num_tracks=T, num_images=N, track_offsets=torch.tensor(tr_off, dtype=torch.int64).to(dev, non_blocking=True),
                      elements=tracks.elements.contiguous(), num_elements=E,
                      kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev, non_blocking=True), keypoints=graph.keypoints.contiguous(),
                      num_rows=kp_off[-1], track_ok=points.ok.to(torch.uint8).contiguous(), points=points.X.contiguous(),
                      info=torch.empty(1, dtype=torch.int64, device=dev), keys=torch.empty(E, dtype=torch.int64, device=dev),
                      keys_alt=torch.empty(E, dtype=torch.int64, device=dev),
                      hist=torch.empty(256 * tiles + 1, dtype=torch.int32, device=dev),
                      image_offsets=torch.empty(N + 1, dtype=torch.int64, device=dev), elem=torch.empty(E, dtype=torch.int32, device=dev),
                      track=torch.empty(E, dtype=torch.int32, device=dev))
            cabi.call("romab200_register_setup", "rb_register_args", **kw)
            if int(kw["info"][0].item()) & cabi.RB_REG_BAD_ID:
                raise ValueError("register_images: a track element lies outside its image's keypoints")
            img_off = kw["image_offsets"].tolist()
            counts = [img_off[i + 1] - img_off[i] for i in images]
            Kd = torch.from_numpy(K).to(dev)
            for b, e in plan_chunks(counts, workspace_bytes):
                ns = counts[b:e]
                total = sum(ns)
                x = torch.empty(max(total, 1), 2, dtype=torch.float64, device=dev)
                X = torch.empty(max(total, 1), 3, dtype=torch.float64, device=dev)
                off = torch.tensor(np.concatenate([[0], np.cumsum(ns)]), dtype=torch.int64).to(dev)
                if total:
                    cabi.call("romab200_register_gather", "rb_register_args", num_list=e - b,
                              images=torch.tensor(images[b:e], dtype=torch.int32).to(dev), out_offsets=off, x=x, X=X, **kw)
                buf = geometry._abs_launch(x, X, off, Kd[images[b:e]].contiguous(), max(ns), max_error2, conf, max_iters, seed)
                R[b:e], t[b:e], ok[b:e], num_inliers[b:e] = buf["R"], buf["t"], buf["ok"], buf["num_inliers"]
                if total:
                    # the accepted images' inlier elements: each image's segment of sorted element ids, in the packed order
                    seg = torch.cat([kw["elem"][img_off[i]:img_off[i + 1]] for i in images[b:e]]).long()
                    acc = buf["ok"].bool() & (buf["num_inliers"] >= min_inliers)
                    acc = torch.repeat_interleave(acc, torch.tensor(ns).to(dev), output_size=total)
                    inlier[seg] = buf["mask"][:total].bool() & acc
                del buf, x, X, off
    accepted = ok.bool() & (num_inliers >= min_inliers)
    return Registration(torch.tensor(images, dtype=torch.int64, device=dev), R, t, ok.bool(), accepted,
                        torch.tensor(counts, dtype=torch.int64, device=dev), num_inliers, inlier)
