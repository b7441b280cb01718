"""Dense reconstruction on the device: the dense warps of `match_pairs` triangulated against known cameras into one depth map per
image (`triangulate_warps`), the depth maps fused by multi-view consistency into a coloured point cloud (`fuse_depth_maps`), and a
binary PLY writer (`write_ply`).  `RegressionMatcher.dense_cloud` runs the whole chain chunk by chunk.  The exact rules are in
include/romab200.h and INTEGRATION.md; `oracle/dense.py` restates them in numpy.

    recon = reconstruct(pairs, graph, tracks, K)
    cloud = model.dense_cloud(images, pairs, K, recon.R, recon.t, registered=recon.registered)
    write_ply("scene.ply", cloud)
"""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass

import numpy as np
import torch

from . import cabi
from .camera import check_intrinsics, pinhole_K
from .matcher import pair_tensor
from .triangulate import _float64

# the columns of DepthMaps.pair_counts: accepted elements, then each rejection reason in the order the rules test them
REASONS = ("accepted", "certainty", "range", "unregistered", "clamped", "behind", "reprojection", "angle")


@dataclass
class DepthMaps:
    """One depth map per image on the warp grid [H, W], accumulated over pairs: depth [N, H, W] float32 (z in the image's camera
    frame, 0 where no element was accepted), score [N, H, W] float32 (the winning certainty), source [N, H, W] int64 (the winner's
    2 k + half, k the global pair index, or -1) and pair_counts [P, 8] int64 (per pair: accepted elements, then the rejections of
    each reason of `REASONS[1:]`).  Tensors live on the warps' device."""
    depth: torch.Tensor
    score: torch.Tensor
    source: torch.Tensor
    pair_counts: torch.Tensor


@dataclass
class DenseCloud:
    """Emitted points, ordered by image, then pixel: points [M, 3] float64 world coordinates, colors [M, 3] uint8, image [M] int32 (the
    view that emitted it), pixel [M] int64 (r W + c on its grid), num_views [M] int32 (agreeing views, the reference included) and
    score [M] float32 (the certainty behind its depth)."""
    points: torch.Tensor
    colors: torch.Tensor
    image: torch.Tensor
    pixel: torch.Tensor
    num_views: torch.Tensor
    score: torch.Tensor


def camera_table(K, R, t, intrinsics=None) -> np.ndarray:
    """The float64 camera table [N, RB_DENSE_CAM] of include/romab200.h: K, K^-1, R (row-major), t, (f, cx, cy, k), 2 unused.  With
    `intrinsics` [N, 4], K is `pinhole_K(intrinsics)`."""
    if intrinsics is not None:
        K = pinhole_K(np.asarray(intrinsics, np.float64))
    N = K.shape[0]
    tab = np.zeros((N, cabi.RB_DENSE_CAM))
    tab[:, 0:9] = K.reshape(N, 9)
    tab[:, 9:18] = np.linalg.inv(K).reshape(N, 9)
    tab[:, 18:27] = R.reshape(N, 9)
    tab[:, 27:30] = t
    if intrinsics is not None:
        tab[:, 30:34] = intrinsics
    return tab


def _number(what, name, v, lo, strict):
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"{what}: {name} must be a number, got {v!r}") from None
    if not math.isfinite(v) or v < lo or (strict and v == lo):
        raise ValueError(f"{what}: {name} must be finite and {'>' if strict else '>='} {lo}, got {v!r}")
    return v


def _int(what, name, v, lo):
    try:
        if isinstance(v, bool):
            raise TypeError
        v = operator.index(v)
    except TypeError:
        raise ValueError(f"{what}: {name} must be an int, got {v!r}") from None
    if v < lo:
        raise ValueError(f"{what}: {name} must be >= {lo}, got {v}")
    return v


def _pairs(what, pairs, N):
    try:
        return pair_tensor(pairs, N)
    except (ValueError, IndexError) as e:
        raise ValueError(f"{what}: {e}") from None


def _sizes(what, image_sizes):
    """image_sizes [N, 2] (H, W) positive integers as an int32 CPU tensor."""
    if isinstance(image_sizes, torch.Tensor):
        if image_sizes.dtype.is_floating_point or image_sizes.dtype.is_complex or image_sizes.dtype == torch.bool:
            raise ValueError(f"{what}: image_sizes must hold integers, got {image_sizes.dtype}")
        s = image_sizes.detach().to("cpu", torch.int64)
    else:
        try:
            s = torch.tensor([[operator.index(h), operator.index(w)] for h, w in image_sizes], dtype=torch.int64).reshape(-1, 2)
        except (TypeError, ValueError):
            raise ValueError(f"{what}: image_sizes must be [N, 2] integers (H, W), got {image_sizes!r}") from None
    if s.dim() != 2 or s.shape[1] != 2 or s.shape[0] < 1:
        raise ValueError(f"{what}: image_sizes must be [N, 2] (H, W) with N >= 1, got shape {tuple(s.shape)}")
    if int(s.min()) < 1 or int(s.max()) >= 1 << 24:
        raise ValueError(f"{what}: image sizes must lie in [1, 2^24), got {s.tolist()}")
    return s.to(torch.int32)


def _registered(what, registered, N):
    if registered is None:
        return np.ones(N, np.uint8)
    r = registered.detach().cpu().numpy() if isinstance(registered, torch.Tensor) else np.asarray(registered)
    if r.dtype != np.bool_ or r.shape != (N,):
        raise ValueError(f"{what}: registered must be a bool mask of shape [{N}], got {r.dtype} {list(r.shape)}")
    return r.astype(np.uint8)


def _cameras(what, N, K, R, t, intrinsics):
    """(camera table, radial flag) of the K / intrinsics alternative, all checked on the host."""
    R = _float64("R", R, (N, 3, 3), what)
    t = _float64("t", t, (N, 3), what)
    if intrinsics is not None:
        if K is not None:
            raise ValueError(f"{what}: give K or intrinsics, not both (with intrinsics, pass K=None)")
        c = check_intrinsics(intrinsics, N, what)
        return camera_table(None, R, t, c), 1
    if K is None:
        raise ValueError(f"{what}: K is required without intrinsics")
    K = _float64("K", K, (N, 3, 3), what)
    if not (np.abs(np.linalg.det(K)) > 0).all():
        raise ValueError(f"{what}: K must be invertible")
    return camera_table(K, R, t), 0


def _tri_options(what, min_certainty=0.05, max_error=4.0, min_angle=1.5):
    min_certainty = _number(what, "min_certainty", min_certainty, 0.0, False)
    max_error = _number(what, "max_error", max_error, 0.0, True)
    min_angle = _number(what, "min_angle", min_angle, 0.0, False)
    if min_angle >= 180:
        raise ValueError(f"{what}: min_angle must lie in [0, 180) degrees, got {min_angle!r}")
    return min_certainty, max_error, min_angle


def _fuse_options(what, max_reproj_error=2.0, max_depth_error=0.01, min_num_views=3):
    return (_number(what, "max_reproj_error", max_reproj_error, 0.0, True), _number(what, "max_depth_error", max_depth_error, 0.0, False),
            _int(what, "min_num_views", min_num_views, 1))


def check_cameras(what, pairs, K, R, t, image_sizes, registered=None, intrinsics=None, **options):
    """The host checks of `triangulate_warps` and `fuse_depth_maps` that do not need the warps (for callers that must refuse bad
    arguments before matching); options are those of either function."""
    tri = {k: options.pop(k) for k in ("min_certainty", "max_error", "min_angle") if k in options}
    fuse = {k: options.pop(k) for k in ("max_reproj_error", "max_depth_error", "min_num_views") if k in options}
    if options:
        raise ValueError(f"{what}: unknown options {sorted(options)}")
    N = _sizes(what, image_sizes).shape[0]
    _pairs(what, pairs, N)
    _cameras(what, N, K, R, t, intrinsics)
    _registered(what, registered, N)
    _tri_options(what, **tri)
    _fuse_options(what, **fuse)
    return tri, fuse


def _device_of(what, *tensors):
    dev = tensors[0].device
    if not all(isinstance(v, torch.Tensor) and v.is_cuda and v.device == dev for v in tensors):
        raise ValueError(f"{what}: the tensors must be on one CUDA device, got {[getattr(v, 'device', None) for v in tensors]}")
    return dev


def new_depth_maps(N: int, H: int, W: int, P: int, device) -> DepthMaps:
    """Empty maps for N images on an H x W grid and P pairs: 16 bytes per grid pixel per image."""
    return DepthMaps(torch.zeros(N, H, W, device=device), torch.zeros(N, H, W, device=device),
                     torch.full((N, H, W), -1, dtype=torch.int64, device=device),
                     torch.zeros(P, cabi.RB_DENSE_REASONS, dtype=torch.int64, device=device))


def triangulate_warps(pairs, warp, certainty, K, R, t, image_sizes, *, first_pair=0, depth_maps=None, registered=None,
                      intrinsics=None, min_certainty=0.05, max_error=4.0, min_angle=1.5) -> DepthMaps:
    """Triangulates the symmetric dense warps of the pairs `first_pair .. first_pair + P'` of `pairs` [P, 2] into per-image depth
    maps on the warp grid.

    warp [P', H, 2W, 4] and certainty [P', H, 2W] are fp32 on a CUDA device, as `match_pairs` returns them (or hands them to its
    `on_batch(k0, warp, certainty)` callback, which can call this with first_pair=k0).  The cameras are x ~ K (R X + t) in the pixel
    frame of image_sizes [N, 2] (H, W): K, R [N, 3, 3] and t [N, 3] as `reconstruct` returns them, or SIMPLE_RADIAL intrinsics [N, 4]
    with K=None.  registered [N] bool (default all) excludes the other images' elements.

    Every element (a grid pixel of one image and its match in the other) is triangulated by the two-view DLT at its canonical pixel
    centre and its fp32 match position, and rejected, in this order, for certainty <= min_certainty (RoMa's sample_thresh by
    default) or a non-finite value, a match outside [-1, 1], an unregistered image, an undistortion clamp, a point behind either
    camera, a reprojection error above max_error px, or a triangulation angle below min_angle degrees (the last two defaults are
    `triangulate_tracks`').  A grid pixel keeps the accepted element of largest certainty, ties to the smallest 2 k + half.

    depth_maps=None creates the maps; passing the previous result accumulates into it (in place, and returns it).  The result does
    not depend on how the pairs are chunked, in what order the chunks come, or on timing: it is bit-identical.  Memory: 16 bytes per
    grid pixel per image (2.4 GB for 200 images on the 864 x 864 grid) plus 4 bytes per warp element of scratch.  Arguments are
    checked before any device work; nothing is read back."""
    what = "triangulate_warps"
    sizes = _sizes(what, image_sizes)
    N = sizes.shape[0]
    pairs = _pairs(what, pairs, N)
    P = pairs.shape[0]
    if not isinstance(warp, torch.Tensor) or not isinstance(certainty, torch.Tensor):
        raise ValueError(f"{what}: warp and certainty must be tensors")
    if warp.dtype != torch.float32 or certainty.dtype != torch.float32:
        raise ValueError(f"{what}: fp32 warp and certainty expected, got {warp.dtype} and {certainty.dtype}")
    if warp.dim() != 4 or warp.shape[3] != 4 or tuple(certainty.shape) != tuple(warp.shape[:3]):
        raise ValueError(f"{what}: warp [P', H, 2W, 4] and certainty [P', H, 2W] expected, got {tuple(warp.shape)} and "
                         f"{tuple(certainty.shape)}")
    C, H, W2 = warp.shape[:3]
    if W2 % 2 or W2 == 0 or H == 0:
        raise ValueError(f"{what}: the warp must be symmetric, [P', H, 2W, 4] with an even width, got {tuple(warp.shape)}")
    W = W2 // 2
    first_pair = _int(what, "first_pair", first_pair, 0)
    if C < 1 or first_pair + C > P or 2 * C > 65535:
        raise ValueError(f"{what}: rows {first_pair} .. {first_pair + C} do not fit the {P} pairs (at most 32767 rows per call)")
    if P >= 1 << 31:
        raise ValueError(f"{what}: {P} pairs, at most 2^31 - 1 are supported")
    table, radial = _cameras(what, N, K, R, t, intrinsics)
    reg = _registered(what, registered, N)
    min_certainty, max_error, min_angle = _tri_options(what, min_certainty, max_error, min_angle)
    dev = _device_of(what, warp, certainty)
    if depth_maps is not None:
        if not isinstance(depth_maps, DepthMaps):
            raise ValueError(f"{what}: depth_maps must be DepthMaps, got {type(depth_maps).__name__}")
        want = {"depth": ((N, H, W), torch.float32), "score": ((N, H, W), torch.float32), "source": ((N, H, W), torch.int64),
                "pair_counts": ((P, cabi.RB_DENSE_REASONS), torch.int64)}
        for name, (shape, dt) in want.items():
            v = getattr(depth_maps, name)
            if not isinstance(v, torch.Tensor) or tuple(v.shape) != shape or v.dtype != dt or v.device != dev or not v.is_contiguous():
                raise ValueError(f"{what}: depth_maps.{name} must be a contiguous {dt} {list(shape)} tensor on {dev}, got "
                                 f"{getattr(v, 'dtype', None)} {tuple(getattr(v, 'shape', ()))}")
    rows = pairs[first_pair:first_pair + C]
    images = torch.unique(rows.flatten()).to(torch.int32)
    with torch.cuda.device(dev):
        dm = depth_maps if depth_maps is not None else new_depth_maps(N, H, W, P, dev)
        kw = dict(pairs=pairs.to(dev, non_blocking=True), num_pairs=P, num_images=N, first_pair=first_pair, chunk=C, H=H, W=W,
                  warp=warp.detach().contiguous(), certainty=certainty.detach().contiguous(), image_sizes=sizes.to(dev, non_blocking=True),
                  cameras=torch.from_numpy(table).to(dev, non_blocking=True), registered=torch.from_numpy(reg).to(dev, non_blocking=True),
                  radial=radial, min_certainty=min_certainty, max_error2=max_error * max_error, min_angle=min_angle * (math.pi / 180.0),
                  images=images.to(dev, non_blocking=True), num_list=images.numel(), depth=dm.depth, score=dm.score, source=dm.source,
                  elem_depth=torch.empty(C, 2, H, W, device=dev),
                  partial=torch.empty(2 * C, cabi.RB_DENSE_MAX_CTAS, cabi.RB_DENSE_REASONS, dtype=torch.int32, device=dev),
                  pair_counts=dm.pair_counts)
        cabi.call("romab200_dense_triangulate", "rb_dense_tri_args", **kw)
        cabi.call("romab200_dense_resolve", "rb_dense_tri_args", **kw)
    return dm


def neighbours(pairs, registered) -> list:
    """Per image, the registered images sharing a row of `pairs` with it, ascending (an image is not its own neighbour)."""
    N = len(registered)
    nb = [set() for _ in range(N)]
    for i, j in pairs.tolist():
        if i != j and registered[i] and registered[j]:
            nb[i].add(j)
            nb[j].add(i)
    return [sorted(s) for s in nb]


def fuse_depth_maps(dm: DepthMaps, pairs, K, R, t, image_sizes, *, registered=None, intrinsics=None, colors=None,
                    max_reproj_error=2.0, max_depth_error=0.01, min_num_views=3) -> DenseCloud:
    """Fuses the depth maps of `triangulate_warps` into one point per surface patch.

    The neighbours of image i are the registered images that share a row of `pairs` with it.  A pixel p of a registered image i with
    depth > 0 is back-projected to X; neighbour j agrees when X projects into j's grid at a pixel q whose depth is within
    max_depth_error (relative) of X's depth in j, and q back-projected lands within max_reproj_error px of p in i.  p is kept when at
    least min_num_views - 1 neighbours agree (min_num_views counts the reference view), and emitted only if no agreeing neighbour
    has a smaller index than i, so a patch several views agree on comes out once, from its lowest-index view.  The point is the float64
    mean of X and the agreeing back-projections, in neighbour order.

    max_reproj_error (2 px) and max_depth_error (0.01) are COLMAP's stereo-fusion defaults; min_num_views defaults to 3, lower than
    COLMAP's min_num_pixels = 5, because the scenes this serves have few images per point.  colors is None (128 grey) or a list of N
    uint8 [H_i, W_i, 3] tensors on the maps' device at any resolution (e.g. from `decode_jpeg`); a point takes the nearest pixel of
    its view's image.  Cameras as in `triangulate_warps`.  Bit-identical from run to run; one host read, the number of points."""
    what = "fuse_depth_maps"
    if not isinstance(dm, DepthMaps):
        raise ValueError(f"{what}: dm must be DepthMaps, got {type(dm).__name__}")
    sizes = _sizes(what, image_sizes)
    N = sizes.shape[0]
    pairs = _pairs(what, pairs, N)
    if not isinstance(dm.depth, torch.Tensor) or dm.depth.dim() != 3 or dm.depth.shape[0] != N or dm.depth.dtype != torch.float32:
        raise ValueError(f"{what}: dm.depth must be float32 [{N}, H, W], got {getattr(dm.depth, 'dtype', None)} "
                         f"{tuple(getattr(dm.depth, 'shape', ()))}")
    H, W = dm.depth.shape[1:]
    if not isinstance(dm.score, torch.Tensor) or tuple(dm.score.shape) != (N, H, W) or dm.score.dtype != torch.float32:
        raise ValueError(f"{what}: dm.score must be float32 [{N}, {H}, {W}]")
    table, radial = _cameras(what, N, K, R, t, intrinsics)
    reg = _registered(what, registered, N)
    max_reproj_error, max_depth_error, min_num_views = _fuse_options(what, max_reproj_error, max_depth_error, min_num_views)
    if colors is not None and len(colors) != N:
        raise ValueError(f"{what}: colors must hold {N} images, got {len(colors)}")
    dev = _device_of(what, dm.depth, dm.score)
    tiles = -(-H * W // cabi.RB_DENSE_TILE)
    if N * tiles >= (1 << 31) - 1:
        raise ValueError(f"{what}: {N * tiles} tiles of {cabi.RB_DENSE_TILE} pixels, at most 2^31 - 2 are supported")
    col = None
    if colors is not None:
        for i, c in enumerate(colors):
            if not isinstance(c, torch.Tensor) or c.dtype != torch.uint8 or c.dim() != 3 or c.shape[2] != 3 or c.shape[0] < 1 or \
                    c.shape[1] < 1 or c.device != dev:
                raise ValueError(f"{what}: colors[{i}] must be a uint8 [H, W, 3] tensor on {dev}, got {getattr(c, 'dtype', None)} "
                                 f"{tuple(getattr(c, 'shape', ()))} on {getattr(c, 'device', None)}")
        col_sizes = torch.tensor([list(c.shape[:2]) for c in colors], dtype=torch.int32)
        col_off = torch.zeros(N + 1, dtype=torch.int64)
        col_off[1:] = torch.cumsum(col_sizes[:, 0].long() * col_sizes[:, 1].long() * 3, 0)
    nb = neighbours(pairs, reg)
    nbr_off = np.zeros(N + 1, np.int64)
    nbr_off[1:] = np.cumsum([len(v) for v in nb])
    nbr = np.array([j for v in nb for j in v] or [0], np.int32)
    with torch.cuda.device(dev):
        if colors is not None:
            col = torch.cat([c.contiguous().reshape(-1) for c in colors])
        kw = dict(num_images=N, H=H, W=W, image_sizes=sizes.to(dev, non_blocking=True), cameras=torch.from_numpy(table).to(dev, non_blocking=True),
                  registered=torch.from_numpy(reg).to(dev, non_blocking=True), radial=radial,
                  nbr_offsets=torch.from_numpy(nbr_off).to(dev, non_blocking=True), nbrs=torch.from_numpy(nbr).to(dev, non_blocking=True),
                  depth=dm.depth.contiguous(), score=dm.score.contiguous(), max_reproj_error2=max_reproj_error * max_reproj_error,
                  max_depth_error=max_depth_error, min_num_views=min_num_views, colors=col,
                  color_offsets=None if col is None else col_off.to(dev, non_blocking=True),
                  color_sizes=None if col is None else col_sizes.to(dev, non_blocking=True), color_bytes=0 if col is None else col.numel(),
                  tile_scan=torch.empty(N * tiles + 1, dtype=torch.int64, device=dev))
        cabi.call("romab200_dense_fuse_count", "rb_dense_fuse_args", **kw)
        M = int(kw["tile_scan"][N * tiles].item())
        out = DenseCloud(torch.empty(M, 3, dtype=torch.float64, device=dev), torch.empty(M, 3, dtype=torch.uint8, device=dev),
                         torch.empty(M, dtype=torch.int32, device=dev), torch.empty(M, dtype=torch.int64, device=dev),
                         torch.empty(M, dtype=torch.int32, device=dev), torch.empty(M, device=dev))
        cabi.call("romab200_dense_fuse_emit", "rb_dense_fuse_args", **kw, num_points=M, points=out.points, rgb=out.colors, image=out.image,
                  pixel=out.pixel, num_views=out.num_views, point_score=out.score)
    return out


def write_ply(path, cloud: DenseCloud) -> None:
    """Writes the cloud as a binary little-endian PLY: `float x y z` and `uchar red green blue` per vertex (the positions rounded to
    float32), which Open3D, MeshLab and CloudCompare read."""
    if not isinstance(cloud, DenseCloud):
        raise ValueError(f"write_ply: cloud must be a DenseCloud, got {type(cloud).__name__}")
    p = cloud.points.detach().cpu().numpy()
    c = cloud.colors.detach().cpu().numpy()
    if p.ndim != 2 or p.shape[1] != 3 or c.shape != p.shape or c.dtype != np.uint8:
        raise ValueError(f"write_ply: points [M, 3] and uint8 colors [M, 3] expected, got {p.shape} and {c.dtype} {c.shape}")
    v = np.empty(p.shape[0], dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("red", "u1"), ("green", "u1"), ("blue", "u1")])
    v["x"], v["y"], v["z"] = p[:, 0], p[:, 1], p[:, 2]
    v["red"], v["green"], v["blue"] = c[:, 0], c[:, 1], c[:, 2]
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {p.shape[0]}\n"
              "property float x\nproperty float y\nproperty float z\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n")
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(v.tobytes())
