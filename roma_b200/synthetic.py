"""Seeded synthetic weights in the reference's state-dict layout.

The reference fetches `roma_outdoor.pth` / `dinov2_vitl14_pretrain.pth` from URLs
(`romatch/models/model_zoo/__init__.py:6-15,42-49`); neither this container nor the GPU box has
a network, so every parity test, golden vector and benchmark in this repository runs on weights
produced here.  The generator is pure torch-CPU with an explicit `torch.Generator`, so the same
seed gives bit-identical tensors on every machine with the same torch build, and the resulting
dicts load into the *unmodified* reference with `strict=True` (that is how `tests/golden` was
produced).

All BatchNorm running statistics, LayerScale gammas and biases are randomised so that BN folding,
LayerScale and bias epilogues are actually exercised by the parity tests (defaults of 0/1 would hide
bugs there).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

from . import arch


def _fan_in(shape):
    n = 1
    for d in shape[1:]:
        n *= d
    return max(n, 1)


def _fill(kind: str, shape, g: torch.Generator) -> torch.Tensor:
    def randn(std):
        return torch.randn(shape, generator=g, dtype=torch.float32) * std

    def uniform(lo, hi):
        return torch.rand(shape, generator=g, dtype=torch.float32) * (hi - lo) + lo

    if kind in ("conv", "linear", "pos_conv", "disp_emb"):
        return randn(1.0 / math.sqrt(_fan_in(shape)))
    if kind in ("conv_relu", "dwconv"):
        return randn(math.sqrt(2.0 / _fan_in(shape)))
    if kind == "to_out":                     # peaky (realistic) anchor distribution: logit std ~4
        return randn(4.0 / math.sqrt(_fan_in(shape)))
    if kind == "proj":                       # keeps projected features (and local correlations) O(1)
        return randn(0.35 / math.sqrt(_fan_in(shape)))
    if kind == "out_conv":                   # keeps per-scale flow/certainty updates moderate
        return randn(0.3 / math.sqrt(_fan_in(shape)))
    if kind == "bias":
        return randn(0.05)
    if kind in ("bn_w", "bn_var", "ln_w"):
        return uniform(0.8, 1.2)
    if kind in ("bn_b", "bn_mean", "ln_b"):
        return randn(0.1)
    if kind == "bn_count":
        return torch.zeros((), dtype=torch.int64)
    if kind == "ls":
        return uniform(0.5, 1.0)
    if kind == "token":
        return randn(0.02)
    if kind == "zeros":
        return torch.zeros(shape, dtype=torch.float32)
    raise KeyError(kind)


def make_matcher_weights(seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """State dict with the 603 tensors of `RegressionMatcher.state_dict()` (SURVEY §3.1-5)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(1000003 * (seed + 1))
    sd = OrderedDict((k, _fill(kind, shape, g)) for k, shape, kind in arch.matcher_param_specs())
    # the certainty logit shares `to_out` with the 4096 anchor logits; keep it O(1) so that the final
    # sigmoid is not saturated and certainty errors stay visible in parity tests
    sd["decoder.embedding_decoder.to_out.weight"][-1] *= 0.125
    for s in arch.SCALES:                    # centre the accumulated certainty logit near 0
        sd[f"decoder.conv_refiner.{s}.out_conv.bias"][2] += 0.6
    return sd


def make_dinov2_weights(seed: int = 0) -> "OrderedDict[str, torch.Tensor]":
    """State dict of DINOv2 ViT-L/14 as `vit_large(...).state_dict()` lays it out."""
    g = torch.Generator(device="cpu")
    g.manual_seed(7919 * (seed + 1) + 17)
    return OrderedDict((k, _fill(kind, shape, g)) for k, shape, kind in arch.dinov2_param_specs())


def make_weights(seed: int = 0):
    return make_matcher_weights(seed), make_dinov2_weights(seed)


def make_pair(batch: int, coarse, upsample, seed: int = 1):
    """Synthetic N(0,1) image tensors, the distribution the reference's own timing tests use
    (`tests/test_roma_upsample_inference_time.py:9-12`): (A, B, A_high, B_high).  Resolutions are ints (square) or (h, w)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    ch, cw = (coarse, coarse) if isinstance(coarse, int) else coarse
    a = torch.randn(batch, 3, ch, cw, generator=g)
    b = torch.randn(batch, 3, ch, cw, generator=g)
    if upsample is None:
        return a, b, None, None
    uh, uw = (upsample, upsample) if isinstance(upsample, int) else upsample
    ah = torch.randn(batch, 3, uh, uw, generator=g)
    bh = torch.randn(batch, 3, uh, uw, generator=g)
    return a, b, ah, bh


def make_pil_pair(seed: int = 3, size_a=(200, 150), size_b=(180, 220)):
    """Two seeded RGB PIL images of different sizes (width, height) for the PIL/path input route
    (`matcher.py:806-816`): smooth random blobs so that the bicubic resize is well exercised."""
    import numpy as np
    from PIL import Image

    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    out = []
    for (w, h) in (size_a, size_b):
        low = torch.rand(1, 3, 12, 16, generator=g)
        img = torch.nn.functional.interpolate(low, size=(h, w), mode="bicubic", align_corners=False)
        arr = (img[0].clamp(0, 1) * 255).round().to(torch.uint8).permute(1, 2, 0).numpy()
        out.append(Image.fromarray(np.ascontiguousarray(arr), "RGB"))
    return out[0], out[1]


# ---- TinyRoMa ----------------------------------------------------------------------------------------
class _ConvBN(torch.nn.Module):
    """Conv2d (no bias) -> BatchNorm2d(affine=False) -> ReLU, wrapped as `self.layer` (XFeat's basic layer as publicly described)."""

    def __init__(self, cin, cout, k=3, stride=1, relu=True):
        super().__init__()
        nn = torch.nn
        self.layer = nn.Sequential(nn.Conv2d(cin, cout, k, stride=stride, padding=k // 2, bias=False), nn.BatchNorm2d(cout, affine=False),
                                   nn.ReLU(inplace=True) if relu else nn.Identity())

    def forward(self, x):
        return self.layer(x)


class XFeatStandIn(torch.nn.Module):
    """A module with the XFeat backbone layout as publicly described (SURVEY §8f): InstanceNorm -> block1 (x4, two stride-2
    layers) + skip1 (AvgPool 4 + 1x1) -> block2 -> block3 (s2) -> block4 (s2) -> block5 (s2) -> fusion of x3 + up(x4) + up(x5).
    It is NOT verified against the real XFeat network (that source is not available offline); TinyRoMa reads the structure of
    whatever module it is given, so nothing depends on this one.  `heatmap_head` / `keypoint_head` / `fine_matcher` are dummies
    that TinyRoMa's constructor deletes."""

    def __init__(self, widths=(4, 8, 24, 64, 128), fusion_extra=True):
        super().__init__()
        nn = torch.nn
        w1, w2, w3, w4, w5 = widths
        self.norm = nn.InstanceNorm2d(1)
        self.skip1 = nn.Sequential(nn.AvgPool2d(4, stride=4), nn.Conv2d(1, w3, 1, stride=1, padding=0))
        self.block1 = nn.Sequential(_ConvBN(1, w1), _ConvBN(w1, w2, stride=2), _ConvBN(w2, w2), _ConvBN(w2, w3, stride=2))
        self.block2 = nn.Sequential(_ConvBN(w3, w3), _ConvBN(w3, w3))
        self.block3 = nn.Sequential(_ConvBN(w3, w4, stride=2), _ConvBN(w4, w4), _ConvBN(w4, w4, k=1))
        self.block4 = nn.Sequential(_ConvBN(w4, w4, stride=2), _ConvBN(w4, w4), _ConvBN(w4, w4))
        self.block5 = nn.Sequential(_ConvBN(w4, w5, stride=2), _ConvBN(w5, w5), _ConvBN(w5, w5), _ConvBN(w5, w4, k=1))
        fusion = [_ConvBN(w4, w4), _ConvBN(w4, w4)] if fusion_extra else [_ConvBN(w4, w4)]
        self.block_fusion = nn.Sequential(*fusion, nn.Conv2d(w4, w4, 1, padding=0))
        self.heatmap_head = nn.Conv2d(w4, 1, 1)
        self.keypoint_head = nn.Conv2d(w4, 65, 1)
        self.fine_matcher = nn.Linear(2 * w4, 64)


def xfeat_standin(**kw) -> torch.nn.Module:
    """The stand-in XFeat backbone used by the tests, goldens and benchmark (see XFeatStandIn), in eval mode."""
    return XFeatStandIn(**kw).eval()


def make_tiny_weights(seed: int, xfeat: torch.nn.Module) -> "OrderedDict[str, torch.Tensor]":
    """Seeded TinyRoMa checkpoint in the reference key layout for this `xfeat` (`xfeat.0.*`, `coarse_matcher.*`, `fine_matcher.*`):
    the keys and shapes `tiny_roma_v1_model(weights, xfeat=xfeat)` loads strictly.  BN statistics are randomised so that folding is
    exercised; the last 1x1 convs of the heads are kept small so that the flow updates stay moderate."""
    from .tiny import expected_state_dict_shapes
    g = torch.Generator(device="cpu")
    g.manual_seed(4099 * (seed + 1) + 11)
    sd = OrderedDict()
    for k, shape in expected_state_dict_shapes(xfeat).items():
        leaf = k.rsplit(".", 1)[1]
        if leaf == "num_batches_tracked":
            sd[k] = torch.zeros((), dtype=torch.int64)
        elif leaf == "running_var":
            sd[k] = _fill("bn_var", shape, g)
        elif leaf == "running_mean":
            sd[k] = _fill("bn_mean", shape, g)
        elif leaf == "bias":
            sd[k] = _fill("bias", shape, g)
        elif len(shape) == 4 and shape[0] == 3 and ("coarse_matcher" in k or "fine_matcher" in k):
            sd[k] = _fill("out_conv", shape, g)
        elif len(shape) == 4:
            sd[k] = _fill("conv_relu", shape, g)
        else:
            sd[k] = _fill("bn_w", shape, g)
    return sd


def _jpeg_image(rng, w: int, h: int, gray: bool):
    """Smooth gradients + sharp-edged rectangles + noise, so that long Huffman codes and large AC categories occur."""
    import numpy as np
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    c = 1 if gray else 3
    img = np.empty((h, w, c))
    for k in range(c):
        img[..., k] = 128 + 100 * np.sin(x / (7 + 13 * rng.rand()) + k) * np.cos(y / (5 + 11 * rng.rand()))
    for _ in range(6):
        x0, y0 = rng.randint(0, w), rng.randint(0, h)
        img[y0:y0 + rng.randint(1, h + 1), x0:x0 + rng.randint(1, w + 1)] = rng.randint(0, 256, size=c)
    img += rng.randn(h, w, c) * rng.choice([2.0, 20.0, 60.0])
    img = np.clip(img, 0, 255).astype(np.uint8)
    return img[..., 0] if gray else img


def jpeg_corpus(seed: int = 0, max_pixels: int = None):
    """Seeded JPEG test/benchmark corpus encoded with the installed Pillow: [(name, bytes, decline)], `decline` None for
    files the device decoder handles, else a substring of the reason it declines them.  Covers quality 50 / 90 / 100,
    subsampling 0 / 1 / 2, optimised Huffman tables, restart intervals (1 and 3 blocks, one row), "L" images, sizes from
    1 x 1 to 6000 x 4000 (entries above `max_pixels` are left out), and progressive, CMYK and 4:4:0 files to decline."""
    import io

    import numpy as np
    from PIL import Image

    rng = np.random.RandomState(seed)
    out = []

    def add(name, w, h, gray=False, decline=None, edit=None, **kw):
        if max_pixels is not None and w * h > max_pixels:
            return
        arr = _jpeg_image(rng, w, h, gray)
        im = Image.fromarray(arr, "L" if gray else "RGB")
        if kw.pop("cmyk", False):
            im = im.convert("CMYK")
        buf = io.BytesIO()
        im.save(buf, "JPEG", **kw)
        data = buf.getvalue()
        if edit is not None:
            data = edit(data)
        out.append((name, data, decline))

    for w, h in ((1, 1), (1, 17), (7, 9), (17, 33), (64, 48)):
        for q in (50, 90, 100):
            for ss in (0, 1, 2):
                add(f"rgb_{w}x{h}_q{q}_s{ss}", w, h, quality=q, subsampling=ss)
        add(f"gray_{w}x{h}_q90", w, h, gray=True, quality=90)
    add("rgb_17x33_opt", 17, 33, quality=90, subsampling=2, optimize=True)
    add("rgb_17x33_rst1", 17, 33, quality=90, subsampling=2, restart_marker_blocks=1)
    add("gray_64x48_rst3", 64, 48, gray=True, quality=90, restart_marker_blocks=3)
    add("rgb_640x480_q90_s2", 640, 480, quality=90, subsampling=2)
    add("rgb_640x480_q50_s0", 640, 480, quality=50, subsampling=0)
    add("rgb_640x480_q100_s1", 640, 480, quality=100, subsampling=1)
    add("rgb_640x480_opt", 640, 480, quality=90, subsampling=2, optimize=True)
    add("rgb_640x480_rst1", 640, 480, quality=90, subsampling=2, restart_marker_blocks=1)
    add("rgb_640x480_rst3", 640, 480, quality=75, subsampling=2, restart_marker_blocks=3)
    add("rgb_640x480_rstrow", 640, 480, quality=90, subsampling=1, restart_marker_rows=1)
    add("gray_640x480_q90", 640, 480, gray=True, quality=90)
    add("rgb_2040x1530_q90_s2", 2040, 1530, quality=90, subsampling=2)
    add("rgb_6000x4000_q90_s2", 6000, 4000, quality=90, subsampling=2)
    add("progressive_64x48", 64, 48, quality=90, progressive=True, decline="progressive")
    add("cmyk_64x48", 64, 48, quality=90, cmyk=True, decline="4 components")

    def to_440(data):
        i = data.index(b"\xff\xc0")             # SOF0 of a 4:4:4 file: luma sampling byte 0x11 -> 0x12 (h 1, v 2)
        b = bytearray(data)
        assert b[i + 11] == 0x11
        b[i + 11] = 0x12
        return bytes(b)

    add("rgb_64x48_440", 64, 48, quality=90, subsampling=0, edit=to_440, decline="sampling layout")
    return out


def jpeg_edits(seed: int = 0):
    """Deterministic edits of small corpus files for the tests of the JPEG decoders: [(name, bytes)].
      - 16 x 16 grayscale and 4:2:0 q100 files whose quantisation tables are all set to 1, 2, 8 or 32: from 8 up, the
        dequantised coefficients leave the range of the 16-bit IDCT Pillow runs;
      - single-bit flips at evenly spaced offsets of the entropy-coded data of every accepted 64 x 48 corpus file.
    Each edit either decodes to exactly Pillow's bytes or is declined."""
    import io

    import numpy as np
    from PIL import Image

    from .jpeg import parse

    out = []
    rng = np.random.RandomState(seed + 7)
    for gray in (True, False):
        im = Image.fromarray(_jpeg_image(rng, 16, 16, gray), "L" if gray else "RGB")
        buf = io.BytesIO()
        im.save(buf, "JPEG", quality=100, subsampling=2)
        base = buf.getvalue()
        for qv in (1, 2, 8, 32):
            b = bytearray(base)
            i = 0
            while True:                                 # every DQT segment: 8-bit tables, entries -> qv
                i = b.find(b"\xff\xdb", i)
                if i < 0:
                    break
                n = (b[i + 2] << 8 | b[i + 3]) - 2
                for t in range(n // 65):
                    b[i + 5 + 65 * t:i + 5 + 65 * t + 64] = bytes([qv]) * 64
                i += 2 + n
            out.append((f"dqt{qv}_{'gray' if gray else 'rgb'}_16x16", bytes(b)))
    for name, data, decline in jpeg_corpus(seed, max_pixels=64 * 48):
        if decline is not None or "64x48" not in name:
            continue
        s0 = parse(data).scan_data
        for off in range(s0, len(data) - 2, max(1, (len(data) - 2 - s0) // 12)):
            for bit in (0, 2, 5):
                b = bytearray(data)
                b[off] ^= 1 << bit
                out.append((f"{name}_flip{off}.{bit}", bytes(b)))
    return out


def _scene_intrinsics(rng, width, height):
    """Pinhole intrinsics of a width x height camera: focal length near 3/4 of the width (1100-1300 px at 1600), pixels within 2 %
    of square, the principal point within width / 80 of the centre."""
    import numpy as np

    s = width / 1600.0
    f = rng.uniform(1100.0 * s, 1300.0 * s)
    return np.array([[f, 0.0, width / 2 + rng.uniform(-20 * s, 20 * s)], [0.0, f * rng.uniform(0.98, 1.02), height / 2 + rng.uniform(-20 * s, 20 * s)],
                     [0.0, 0.0, 1.0]])


def _scene_rotation(rng, deg_lo, deg_hi):
    """A rotation by deg_lo .. deg_hi degrees about a random axis (Rodrigues)."""
    import numpy as np

    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = np.deg2rad(rng.uniform(deg_lo, deg_hi))
    S = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    return np.eye(3) + np.sin(ang) * S + (1 - np.cos(ang)) * S @ S


def two_view_scene(seed: int, n: int, outlier_frac: float, noise: float = 0.5, width: int = 1600, height: int = 1200):
    """A seeded calibrated two-view scene for the pose estimator: focal lengths near 1200 px, a 5-20 degree rotation about a
    random axis, a unit baseline in a random direction, `n` points seen by camera 0 at depths 6-14, Gaussian pixel noise of
    `noise` px in both images, and a fraction `outlier_frac` of correspondences whose second point is uniform in image 1.
    Returns float64 numpy arrays: kpts0, kpts1 [n, 2], K0, K1 [3, 3], R [3, 3], t [3] (x1 ~ K1 (R X + t)), and outlier bool [n]
    marking the replaced correspondences."""
    import numpy as np

    rng = np.random.default_rng(seed)
    K0, K1 = _scene_intrinsics(rng, width, height), _scene_intrinsics(rng, width, height)
    R = _scene_rotation(rng, 5.0, 20.0)
    t = rng.normal(size=3)
    t /= np.linalg.norm(t)
    px = np.c_[rng.uniform(0, width, n), rng.uniform(0, height, n), np.ones(n)]
    X = (np.linalg.inv(K0) @ px.T).T * rng.uniform(6.0, 14.0, n)[:, None]
    x1 = (K1 @ (X @ R.T + t).T).T
    kpts0 = px[:, :2] + rng.normal(scale=noise, size=(n, 2))
    kpts1 = x1[:, :2] / x1[:, 2:] + rng.normal(scale=noise, size=(n, 2))
    out = rng.random(n) < outlier_frac
    kpts1[out] = np.c_[rng.uniform(0, width, out.sum()), rng.uniform(0, height, out.sum())]
    return {"kpts0": kpts0, "kpts1": kpts1, "K0": K0, "K1": K1, "R": R, "t": t, "outlier": out}


def depth_scene(seed: int, batch: int, h0: int, w0: int, h1: int = None, w1: int = None):
    """Seeded piecewise-planar two-view scenes with exact depth maps, for the depth-based warps (`roma_b200.depth_warp`).  Each pair
    sees a tilted ground plane 8-13 units away and, in front of it, one occluding quad at 4-5 units; camera 1 is camera 0 moved by
    a unit baseline, mostly sideways, and rotated by 8-16 degrees (intrinsics and rotation as in `two_view_scene`, scaled to the
    image size).  The depth of a pixel is the z of the nearest ray-plane intersection through its centre (x + 0.5, y + 0.5) in
    that view's own camera frame, so the two maps are consistent to rounding; it is stored as float32, like MegaDepth's.  Seven
    random rectangles per view are holes of zero depth.  The motion is large enough that pixels of view 0 fall in all four classes of
    `warp_kpts` in quantity: zero depth, not covisible, depth-inconsistent (occluded by the quad, or landing on a hole), valid.
    h1, w1 default to h0, w0.  Returns torch CPU tensors: depth0 [B, h0, w0] and depth1 [B, h1, w1] float32, T_0to1 [B, 4, 4]
    (X1 = R X0 + t), K0, K1 [B, 3, 3] float64."""
    import numpy as np

    h1, w1 = h1 or h0, w1 or w0
    rng = np.random.default_rng(seed)

    def render(K, R, t, h, w, planes):
        # rays through the pixel centres of this view; a plane n . X0 = d of frame 0 is (R n) . X = d + (R n) . t in this frame
        ys, xs = np.meshgrid(np.arange(h) + 0.5, np.arange(w) + 0.5, indexing="ij")
        rays = np.stack((xs, ys, np.ones_like(xs)), -1) @ np.linalg.inv(K).T
        depth = np.full((h, w), np.inf)
        for n, d, centre, axes, half in planes:
            n1 = R @ n
            with np.errstate(divide="ignore", invalid="ignore"):
                z = (d + n1 @ t) / (rays @ n1)
            hit = np.isfinite(z) & (z > 0)
            if centre is not None:                   # the quad: bounded in its own plane, tested in frame 0
                X0 = ((rays * np.where(hit, z, 0.0)[..., None]) - t) @ R
                for e, a in zip(axes, half):
                    hit &= np.abs((X0 - centre) @ e) < a
            depth = np.where(hit & (z < depth), z, depth)
        depth[~np.isfinite(depth)] = 0.0
        for _ in range(7):
            hh, hw = int(h * rng.uniform(0.08, 0.2)), int(w * rng.uniform(0.08, 0.2))
            y, x = rng.integers(0, h - hh), rng.integers(0, w - hw)
            depth[y:y + hh, x:x + hw] = 0.0
        return depth.astype(np.float32)

    out = {k: [] for k in ("depth0", "depth1", "T", "K0", "K1")}
    for _ in range(batch):
        K0, K1 = _scene_intrinsics(rng, w0, h0), _scene_intrinsics(rng, w1, h1)
        R = _scene_rotation(rng, 8.0, 16.0)
        t = np.array([rng.choice([-1.0, 1.0]), rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3)])
        t /= np.linalg.norm(t)
        n = np.array([rng.uniform(-0.15, 0.15), rng.uniform(0.3, 0.5), 1.0])
        ground = (n / np.linalg.norm(n), rng.uniform(8.0, 11.0), None, None, None)
        qn = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0])
        qn /= np.linalg.norm(qn)
        centre = np.array([rng.uniform(-1.0, 1.0), rng.uniform(-0.7, 0.7), rng.uniform(4.0, 5.0)])
        e1 = np.cross(qn, [0.0, 1.0, 0.0])
        e1 /= np.linalg.norm(e1)
        quad = (qn, qn @ centre, centre, (e1, np.cross(qn, e1)), (rng.uniform(1.0, 1.4), rng.uniform(0.8, 1.2)))
        T = np.eye(4)
        T[:3, :3], T[:3, 3] = R, t
        out["depth0"].append(render(K0, np.eye(3), np.zeros(3), h0, w0, (ground, quad)))
        out["depth1"].append(render(K1, R, t, h1, w1, (ground, quad)))
        out["T"].append(T), out["K0"].append(K0), out["K1"].append(K1)
    return tuple(torch.from_numpy(np.stack(out[k])) for k in ("depth0", "depth1", "T", "K0", "K1"))


def planar_scene(seed: int, n: int, outlier_frac: float, noise: float = 0.5, width: int = 640, height: int = 480):
    """A seeded HPatches-like homography pair: H is a random perspective warp of the image that moves each corner by up to a
    fifth of the image size, `n` points uniform in image A, their images under H with Gaussian noise of `noise` px, and a
    fraction `outlier_frac` of correspondences whose second point is uniform in image B.  Returns float64 numpy arrays: src,
    dst [n, 2], H [3, 3] (dst ~ H src), inlier [n] bool, and the image size (w, h)."""
    import numpy as np

    rng = np.random.default_rng(seed)
    c = np.array([[0.0, 0.0], [0.0, height - 1.0], [width - 1.0, 0.0], [width - 1.0, height - 1.0]])
    moved = c + rng.uniform(-0.2, 0.2, size=(4, 2)) * np.array([width, height])
    A = []
    for (x, y), (u, v) in zip(c, moved):
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y, -u])
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y, -v])
    H = np.linalg.svd(np.array(A))[2][-1].reshape(3, 3)
    H = H / H[2, 2]
    src = np.c_[rng.uniform(0, width, n), rng.uniform(0, height, n)]
    p = np.c_[src, np.ones(n)] @ H.T
    dst = p[:, :2] / p[:, 2:] + rng.normal(scale=noise, size=(n, 2))
    out = rng.random(n) < outlier_frac
    dst[out] = np.c_[rng.uniform(0, width, out.sum()), rng.uniform(0, height, out.sum())]
    return {"src": src, "dst": dst, "H": H, "inlier": ~out, "size": (width, height)}


def homography_corner_error(H_pred, H_gt, width: int, height: int):
    """The HPatches harness's error (hpatches_sequences_homog_benchmark.py): the mean distance of the four image corners mapped by
    the predicted and the true homography, divided by min(w, h) / 480.  A missing prediction (None) counts as infinite."""
    import numpy as np

    if H_pred is None:
        return float("inf")
    c = np.array([[0, 0, 1], [0, height - 1, 1], [width - 1, 0, 1], [width - 1, height - 1, 1]], dtype=np.float64)
    a = c @ np.asarray(H_pred, dtype=np.float64).T
    b = c @ np.asarray(H_gt, dtype=np.float64).T
    d = np.linalg.norm(a[:, :2] / a[:, 2:] - b[:, :2] / b[:, 2:], axis=1).mean()
    return float(d / (min(width, height) / 480.0))


def homography_auc(errors, thresholds=(3, 5, 10)):
    """Area under the recall-error curve up to each threshold (px), normalised to [0, 1], as the harness reports AUC@3/5/10."""
    import numpy as np

    errors = np.sort(np.r_[0.0, np.asarray(errors, dtype=np.float64)])
    recall = np.r_[0.0, (np.arange(len(errors) - 1) + 1) / (len(errors) - 1)]
    out = []
    for th in thresholds:
        last = np.searchsorted(errors, th)
        r = np.r_[recall[:last], recall[last - 1]]
        e = np.r_[errors[:last], th]
        out.append(float(np.trapezoid(r, x=e) / th))
    return out


def planted_views(seed: int, n_images: int, n_points: int, *, size=(768, 1024), cell_size: int = 1, visibility: float = 0.5,
                  outlier_frac: float = 0.0, device="cpu"):
    """Seeded multi-view samples with planted tracks, for `consolidate_matches` and `build_tracks`.  Each of `n_images` images of
    `size` (H, W) sees each of `n_points` scene points with probability `visibility`, at a cell of `cell_size` px of its own (the
    points take distinct cells in every image).  Every pair (i, j), i < j, of the exhaustive graph gets one sample per point both
    images see: each side at its cell's centre plus uniform noise of up to a quarter cell, drawn per sample, with certainty in
    [0.5, 1).  On top of a pair's m such samples come round(m * outlier_frac / (1 - outlier_frac)) outliers, so that a fraction
    `outlier_frac` of its samples are outliers: both sides uniform in their images, certainty in [0.05, 0.5).  Pairs with fewer
    samples than the largest are padded with certainty 0, which consolidate_matches ignores.
    Returns, on `device`: pairs [P, 2] int64, matches [P, n, 4] fp32 (normalised (xA, yA, xB, yB), as sample_batched returns them),
    certainty [P, n] fp32, image_sizes [N, 2] int64, and views [n_points, N] int64, the cell cy * gw + cx of each point in each
    image (gw = ceil(W / cell_size)), -1 where the image does not see it."""
    H, W = size
    cs = int(cell_size)
    gh, gw = -(-H // cs), -(-W // cs)
    if n_points > gh * gw:
        raise ValueError(f"planted_views: {n_points} points do not fit in {gh * gw} cells")
    g = torch.Generator(device=device).manual_seed(seed)
    vis = torch.rand(n_images, n_points, generator=g, device=device) < visibility
    cells = torch.stack([torch.randperm(gh * gw, generator=g, device=device)[:n_points] for _ in range(n_images)])
    return _planted_samples(g, vis, cells, H, W, cs, outlier_frac, device)


def _planted_samples(g, vis, cells, H, W, cs, outlier_frac, device):
    """The samples of `planted_views` from g's stream for points seen where vis [N, n_points] is set, at cells [N, n_points] of cs px:
    returns (pairs, matches, certainty, image_sizes, views)."""
    n_images = vis.shape[0]
    gw = -(-W // cs)
    pairs = torch.triu_indices(n_images, n_images, 1, device=device).T.contiguous()
    P = pairs.shape[0]
    co = vis[pairs[:, 0]] & vis[pairs[:, 1]]
    n_in = co.sum(1)
    n_out = torch.round(n_in * (outlier_frac / (1.0 - outlier_frac))).long() if outlier_frac > 0 else torch.zeros_like(n_in)
    n = int((n_in + n_out).max()) if P else 0
    matches = torch.zeros(P, n, 4, device=device)
    certainty = torch.zeros(P, n, device=device)

    def start(counts):
        return torch.cumsum(counts, 0) - counts

    def side(cell, count):
        """Normalised (u, v) of `count` positions in the given cells: the centre of the cell's pixels plus uniform noise."""
        lo_x, lo_y = (cell % gw) * cs, (cell // gw) * cs
        hi_x, hi_y = torch.clamp(lo_x + cs, max=W), torch.clamp(lo_y + cs, max=H)
        noise = torch.rand(count, 2, generator=g, device=device, dtype=torch.float64) - 0.5
        x = (lo_x + hi_x) / 2 + (hi_x - lo_x) * noise[:, 0] / 2
        y = (lo_y + hi_y) / 2 + (hi_y - lo_y) * noise[:, 1] / 2
        return torch.stack((2 * x / W - 1, 2 * y / H - 1), 1).float()

    k, p = co.nonzero(as_tuple=True)
    slot = torch.arange(k.numel(), device=device) - start(n_in)[k]
    matches[k, slot, 0:2] = side(cells[pairs[k, 0], p], k.numel())
    matches[k, slot, 2:4] = side(cells[pairs[k, 1], p], k.numel())
    certainty[k, slot] = 0.5 + 0.5 * torch.rand(k.numel(), generator=g, device=device)
    k = torch.repeat_interleave(torch.arange(P, device=device), n_out)
    slot = n_in[k] + torch.arange(k.numel(), device=device) - start(n_out)[k]
    matches[k, slot] = torch.rand(k.numel(), 4, generator=g, device=device) * 2 - 1
    certainty[k, slot] = 0.05 + 0.45 * torch.rand(k.numel(), generator=g, device=device)
    sizes = torch.tensor([[H, W]] * n_images, dtype=torch.int64, device=device)
    return pairs, matches, certainty, sizes, torch.where(vis, cells, -1).T.contiguous()


def planted_cameras(seed: int, n_images: int, n_points: int, *, size=(768, 1024), cell_size: int = 1, noise: float = 0.5,
                    visibility: float = 0.5, outlier_frac: float = 0.0, device="cpu", radial=None, spread: bool = False, camera_ids=None):
    """Seeded multi-view samples of a real scene, for geometric verification (`verify_matches`): `planted_views` with geometry.  A
    cloud of `n_points` scene points fills a 8 x 6 x 6 box around the origin; `n_images` pinhole cameras of `size` (H, W) with the
    intrinsics of `_scene_intrinsics` stand 8-10 units from the origin at azimuths of -40..40 degrees and heights of -1..1 and look at
    a point near the origin, so depths vary from about 5 to 13 and no pair's F is degenerate.  A point's observed position in an
    image is its projection plus Gaussian noise of `noise` px, drawn once per (point, image), so every pair puts the point in the same
    cell.  The observation is dropped when it lies outside the image or behind the camera, when a draw with probability
    `visibility` fails, or when its cell (the fp32 rule of `consolidate_matches` applied to the normalised coordinates) is already
    taken by a lower-indexed point.  Samples, outliers, certainties and padding are those of `planted_views` for these cells.
    Returns, on `device`: what `planted_views` returns (pairs, matches, certainty, image_sizes, views), then K [N, 3, 3], R [N, 3, 3]
    and t [N, 3] float64 (x ~ K (R X + t)) and X [n_points, 3] float64.

    Options, drawn from a second generator so that the draws above are the same with and without them:
    - radial=(k_lo, k_hi): SIMPLE_RADIAL cameras (`roma_b200.camera`): each image keeps the f of its pinhole intrinsics, square pixels,
      the principal point at (W / 2, H / 2) and k uniform in [k_lo, k_hi], applied before the noise and the cell assignment.  K is
      then the [N, 4] (f, cx, cy, k) float64 intrinsics.
    - spread=True: look-at targets uniform in a 4 x 3 x 3 box, heights of -3..3 and rolls of -20..20 degrees about the optical
      axis, so that the optical axes do not all meet near one point (per-image focal lengths are then better determined).
    - camera_ids [n_images] (integers >= 0): shared cameras.  Every image of a group takes the intrinsics of the group's first image,
      and with `radial` the group draws one k (one draw per id in [0, max + 1)), so the rows of K within a group are equal."""
    import numpy as np

    H, W = size
    cs = int(cell_size)
    gw = -(-W // cs)
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.0, 1.0, (n_points, 3)) * np.array([4.0, 3.0, 3.0])
    K = np.stack([_scene_intrinsics(rng, W, H) for _ in range(n_images)])
    az = np.deg2rad(rng.uniform(-40.0, 40.0, n_images))
    r, h = rng.uniform(8.0, 10.0, n_images), rng.uniform(-1.0, 1.0, n_images)
    C = np.stack((r * np.sin(az), h, -r * np.cos(az)), 1)
    target = rng.uniform(-0.5, 0.5, (n_images, 3))
    extra = np.random.default_rng([seed, 1])
    roll = np.zeros(n_images)
    if spread:
        target = extra.uniform(-1.0, 1.0, (n_images, 3)) * np.array([2.0, 1.5, 1.5])
        C[:, 1] = extra.uniform(-3.0, 3.0, n_images)
        roll = np.deg2rad(extra.uniform(-20.0, 20.0, n_images))
    R = np.empty((n_images, 3, 3))
    for c in range(n_images):
        z = (target[c] - C[c]) / np.linalg.norm(target[c] - C[c])
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R[c] = np.stack((x, np.cross(z, x), z))
        if roll[c]:
            cr, sr = np.cos(roll[c]), np.sin(roll[c])
            R[c] = np.array([[cr, -sr, 0.0], [sr, cr, 0.0], [0.0, 0.0, 1.0]]) @ R[c]
    t = -np.einsum("cij,cj->ci", R, C)
    if camera_ids is not None:
        ids = np.asarray(camera_ids, np.int64)
        if ids.shape != (n_images,) or ids.min() < 0:
            raise ValueError(f"planted_cameras: camera_ids must be [{n_images}] integers >= 0")
        first = {}
        for i, g in enumerate(ids.tolist()):
            first.setdefault(g, i)
        K = K[[first[g] for g in ids.tolist()]]
    if radial is not None:
        k = extra.uniform(radial[0], radial[1], n_images if camera_ids is None else int(ids.max()) + 1)
        if camera_ids is not None:
            k = k[ids]
        K = np.stack((K[:, 0, 0], np.full(n_images, W / 2), np.full(n_images, H / 2), k), 1)
        pc = np.einsum("cij,pj->cpi", R, X) + t[:, None]
        depth = pc[..., 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            xn = pc[..., :2] / depth[..., None]
            d = 1.0 + K[:, 3, None] * (xn * xn).sum(-1)
            xy = K[:, None, 0, None] * d[..., None] * xn + K[:, None, 1:3] + rng.normal(scale=noise, size=(n_images, n_points, 2))
    else:
        p = np.einsum("cij,cjk,pk->cpi", K, R, X) + np.einsum("cij,cj->ci", K, t)[:, None]        # [N, n_points, 3]
        depth = p[..., 2]
        with np.errstate(divide="ignore", invalid="ignore"):
            xy = p[..., :2] / depth[..., None] + rng.normal(scale=noise, size=(n_images, n_points, 2))
    vis = (depth > 0) & (xy[..., 0] >= 0) & (xy[..., 0] < W) & (xy[..., 1] >= 0) & (xy[..., 1] < H)
    vis &= rng.random((n_images, n_points)) < visibility
    u = np.where(vis, 2 * xy[..., 0] / W - 1, 0.0).astype(np.float32)
    v = np.where(vis, 2 * xy[..., 1] / H - 1, 0.0).astype(np.float32)
    px = np.float32(W / 2) * (u + np.float32(1))
    py = np.float32(H / 2) * (v + np.float32(1))
    cx = np.clip(np.floor(px), 0, W - 1).astype(np.int64) // cs
    cy = np.clip(np.floor(py), 0, H - 1).astype(np.int64) // cs
    cells = cy * gw + cx
    for c in range(n_images):
        seen = np.flatnonzero(vis[c])
        first = np.zeros(n_points, bool)
        first[seen[np.unique(cells[c, seen], return_index=True)[1]]] = True
        vis[c] &= first
    g = torch.Generator(device=device).manual_seed(seed)
    out = _planted_samples(g, torch.from_numpy(vis).to(device), torch.from_numpy(cells).to(device), H, W, cs, outlier_frac, device)
    return out + tuple(torch.from_numpy(a).to(device) for a in (K, R, t, X))


def perturb_cameras(seed: int, R, t, rot_deg: float, centre: float):
    """Seeded noise on cameras x ~ K (R X + t): each rotation turned by `rot_deg` degrees about a uniformly random axis (R' = Q R)
    and each centre C = -R^T t moved by `centre` units in a uniformly random direction.  R [N, 3, 3] and t [N, 3] are tensors or
    arrays; returns float64 (R', t') of the same kind, on the same device."""
    import numpy as np

    dev = R.device if isinstance(R, torch.Tensor) else None
    Rn = R.detach().cpu().double().numpy() if dev is not None else np.asarray(R, np.float64)
    tn = t.detach().cpu().double().numpy() if dev is not None else np.asarray(t, np.float64)
    rng = np.random.default_rng(seed)
    N = Rn.shape[0]
    axis = rng.normal(size=(N, 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    step = rng.normal(size=(N, 3))
    step /= np.linalg.norm(step, axis=1, keepdims=True)
    th = np.deg2rad(rot_deg)
    Kx = np.zeros((N, 3, 3))
    Kx[:, 0, 1], Kx[:, 0, 2], Kx[:, 1, 2] = -axis[:, 2], axis[:, 1], -axis[:, 0]
    Kx -= Kx.transpose(0, 2, 1)
    Q = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    C = -np.einsum("nji,nj->ni", Rn, tn) + centre * step
    R2 = Q @ Rn
    t2 = -np.einsum("nij,nj->ni", R2, C)
    if dev is None:
        return R2, t2
    return torch.from_numpy(R2).to(dev), torch.from_numpy(t2).to(dev)


def planted_tracks(views, min_length: int = 2):
    """The planted tracks of `planted_views` with at least `min_length` views, as a set of tuples ((image, cell), ...) in image order."""
    v = views.cpu().numpy()
    return {tuple((i, int(c)) for i, c in enumerate(row) if c >= 0) for row in v if (row >= 0).sum() >= min_length}


def track_cells(track_offsets, elements, kp_offsets, keypoints, width: int, cell_size: int = 1):
    """Tracks (offsets and (image, keypoint id) elements) as the tuples of `planted_tracks`: each element's keypoint mapped to its
    cell, for images `width` px wide."""
    import numpy as np

    off, el = track_offsets.cpu().numpy(), elements.cpu().numpy().astype(np.int64)
    kp, kpo = keypoints.cpu().numpy(), kp_offsets.cpu().numpy()
    xy = kp[kpo[el[:, 0]] + el[:, 1]] if el.size else np.zeros((0, 2), np.float32)
    gw = -(-width // cell_size)
    cell = (np.floor(xy[:, 1]).astype(np.int64) // cell_size) * gw + np.floor(xy[:, 0]).astype(np.int64) // cell_size
    pairs = list(zip(el[:, 0].tolist(), cell.tolist()))
    return {tuple(pairs[off[t]:off[t + 1]]) for t in range(len(off) - 1)}


def track_points(track_offsets, elements, kp_offsets, keypoints, views, width: int, cell_size: int = 1):
    """The planted point of every track, int64 [T]: each element's keypoint mapped to its cell by the rule of `track_cells`, then to
    the point whose view in that image (`views` [n_points, N] of `planted_views` or `planted_cameras`) is that cell.  -1 for a track
    whose elements are not all views of one point."""
    import numpy as np

    off, el = track_offsets.cpu().numpy(), elements.cpu().numpy().astype(np.int64)
    kp, kpo, v = keypoints.cpu().numpy(), kp_offsets.cpu().numpy(), views.cpu().numpy()
    T = len(off) - 1
    if el.size == 0:
        return np.full(T, -1, np.int64)
    xy = kp[kpo[el[:, 0]] + el[:, 1]]
    gw = -(-width // cell_size)
    cell = (np.floor(xy[:, 1]).astype(np.int64) // cell_size) * gw + np.floor(xy[:, 0]).astype(np.int64) // cell_size
    span = int(max(v.max(), cell.max())) + 1
    p, i = np.nonzero(v >= 0)
    keys = i * span + v[p, i]                               # (image, cell) of every planted view
    order = np.argsort(keys)
    keys, p = np.r_[keys[order], -1], np.r_[p[order], -1]   # a sentinel, so that a miss finds a key that differs
    q = el[:, 0] * span + cell
    at = np.minimum(np.searchsorted(keys[:-1], q), keys.size - 1)
    point = np.where(keys[at] == q, p[at], -1)
    out = np.full(T, -1, np.int64)
    for k in range(T):
        pk = point[off[k]:off[k + 1]]
        if pk.size and pk[0] >= 0 and (pk == pk[0]).all():
            out[k] = pk[0]
    return out


def _radial_rays(intr, x, y):
    """Normalised undistorted coordinates of pixels (x, y) under SIMPLE_RADIAL (f, cx, cy, k): the Newton loop of the keypoint
    undistortion (include/romab200.h), which converges for the scenes here (no pixel reaches the turning radius)."""
    import numpy as np

    f, cx, cy, k = intr
    dx, dy = x - cx, y - cy
    rd = np.sqrt(dx * dx + dy * dy) / f
    rho = rd.copy()
    for _ in range(20):
        rho = rho - (rho * (1.0 + k * rho * rho) - rd) / (1.0 + 3.0 * k * rho * rho)
    with np.errstate(divide="ignore", invalid="ignore"):
        s = np.where(rd > 0, rho / rd, 1.0)
    return dx * s / f, dy * s / f


def depth_views(seed: int, n_images: int, size=(96, 128), radial=None):
    """Seeded multi-view scenes with exact per-view depth maps, for dense reconstruction (`roma_b200.dense`).  Cameras are laid out as
    in `planted_cameras` (pinhole intrinsics of `_scene_intrinsics`, 8-10 units from the origin at azimuths of -40..40 degrees and
    heights of -1..1, looking at a point near the origin).  The scene is `depth_scene`'s: a tilted ground plane n . X = d 1.5-3 units
    beyond the origin, and two occluding quads 0-2 units in front of it.  View i's depth at pixel (x, y) is the z in its camera frame of
    the nearest ray-plane intersection through the pixel centre (x + 0.5, y + 0.5), stored as float32; five random rectangles per view
    are holes of zero depth.  Each view also gets a uint8 colour image, a function of the world point it sees (black where it sees
    nothing), so the colours of one surface point agree across views.
    radial=(k_lo, k_hi): SIMPLE_RADIAL cameras with the pinhole f, the principal point at (W / 2, H / 2) and k uniform in the range
    (from a second generator, so the other draws do not change); the pixel centres are then distorted pixels.
    Returns a dict of CPU tensors: depth [N, H, W] float32, K [N, 3, 3] float64 (pinhole_K of the intrinsics when radial), intrinsics
    [N, 4] float64 or None, R [N, 3, 3], t [N, 3] float64 (x ~ K (R X + t)), colors [N, H, W, 3] uint8, image_sizes [N, 2] int64."""
    import numpy as np

    H, W = size
    rng = np.random.default_rng(seed)
    K = np.stack([_scene_intrinsics(rng, W, H) for _ in range(n_images)])
    az = np.deg2rad(rng.uniform(-40.0, 40.0, n_images))
    r, h = rng.uniform(8.0, 10.0, n_images), rng.uniform(-1.0, 1.0, n_images)
    C = np.stack((r * np.sin(az), h, -r * np.cos(az)), 1)
    target = rng.uniform(-0.5, 0.5, (n_images, 3))
    R = np.empty((n_images, 3, 3))
    for c in range(n_images):
        z = (target[c] - C[c]) / np.linalg.norm(target[c] - C[c])
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R[c] = np.stack((x, np.cross(z, x), z))
    t = -np.einsum("cij,cj->ci", R, C)
    n = np.array([rng.uniform(-0.15, 0.15), rng.uniform(-0.25, -0.1), -1.0])
    planes = [(n / np.linalg.norm(n), -rng.uniform(1.5, 3.0), None, None, None)]
    for _ in range(2):
        qn = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), -1.0])
        qn /= np.linalg.norm(qn)
        centre = np.array([rng.uniform(-1.5, 1.5), rng.uniform(-1.0, 1.0), rng.uniform(-2.0, 0.0)])
        e1 = np.cross(qn, [0.0, 1.0, 0.0])
        e1 /= np.linalg.norm(e1)
        planes.append((qn, qn @ centre, centre, (e1, np.cross(qn, e1)), (rng.uniform(0.8, 1.2), rng.uniform(0.6, 1.0))))
    intr = None
    if radial is not None:
        k = np.random.default_rng([seed, 1]).uniform(radial[0], radial[1], n_images)
        intr = np.stack((K[:, 0, 0], np.full(n_images, W / 2), np.full(n_images, H / 2), k), 1)
        K = np.zeros((n_images, 3, 3))
        K[:, 0, 0] = K[:, 1, 1] = intr[:, 0]
        K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = intr[:, 1], intr[:, 2], 1.0
    ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    depth = np.zeros((n_images, H, W), np.float32)
    colors = np.zeros((n_images, H, W, 3), np.uint8)
    for c in range(n_images):
        if intr is None:
            rays = np.stack((xs, ys, np.ones_like(xs)), -1) @ np.linalg.inv(K[c]).T
        else:
            a, b = _radial_rays(intr[c], xs, ys)
            rays = np.stack((a, b, np.ones_like(a)), -1)
        dirs = rays @ R[c]                                  # world directions whose camera-frame z is 1
        z = np.full((H, W), np.inf)
        for nrm, d, centre, axes, half in planes:
            with np.errstate(divide="ignore", invalid="ignore"):
                s = (d - nrm @ C[c]) / (dirs @ nrm)
            hit = np.isfinite(s) & (s > 0)
            if centre is not None:
                Xw = C[c] + dirs * np.where(hit, s, 0.0)[..., None]
                for e, a in zip(axes, half):
                    hit &= np.abs((Xw - centre) @ e) < a
            z = np.where(hit & (s < z), s, z)
        seen = np.isfinite(z)
        Xw = C[c] + dirs * np.where(seen, z, 0.0)[..., None]
        rgb = 128 + 100 * np.sin(np.stack((3.0 * Xw[..., 0], 3.0 * Xw[..., 1], 2.0 * Xw[..., 0] + 2.0 * Xw[..., 2]), -1))
        colors[c] = np.where(seen[..., None], rgb, 0).astype(np.uint8)
        z[~seen] = 0.0
        for _ in range(5):
            hh, hw = int(H * rng.uniform(0.05, 0.12)), int(W * rng.uniform(0.05, 0.12))
            y0, x0 = rng.integers(0, H - hh), rng.integers(0, W - hw)
            z[y0:y0 + hh, x0:x0 + hw] = 0.0
        depth[c] = z.astype(np.float32)
    f64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64))     # noqa: E731
    return {"depth": torch.from_numpy(depth), "K": f64(K), "intrinsics": None if intr is None else f64(intr), "R": f64(R), "t": f64(t),
            "colors": torch.from_numpy(colors), "image_sizes": torch.tensor([[H, W]] * n_images, dtype=torch.int64)}


def depth_view_warps(views, pairs, device="cuda"):
    """The symmetric ground-truth warps of `depth_views` for the pairs [P, 2], on the views' own grid: for pair (i, j) the left half
    is `get_gt_warp(depth_i, depth_j, T_i->j, K_i, K_j)` (grid pixel of i, its match in j), the right half the same from j to i with the
    two positions swapped, as match_pairs lays out a symmetric warp; certainty is `prob`.  Pinhole views only (get_gt_warp has no
    distortion): radial views take the same rule in numpy float64 (the match is the distorted projection, and prob is 1 where the
    point is covisible strictly inside the image less one pixel and within 5 % of the other view's nearest depth).  Returns
    (warp [P, H, 2W, 4], certainty [P, H, 2W]) fp32 on `device`."""
    import numpy as np
    from .depth_warp import get_gt_warp

    pairs = torch.as_tensor(pairs, dtype=torch.int64).reshape(-1, 2)
    depth, R, t = views["depth"], views["R"], views["t"]
    N, H, W = depth.shape
    i, j = pairs[:, 0], pairs[:, 1]
    halves = []
    for a, b in ((i, j), (j, i)):
        Rr = R[b] @ R[a].transpose(1, 2)
        T = torch.zeros(len(a), 4, 4, dtype=torch.float64)
        T[:, :3, :3], T[:, :3, 3], T[:, 3, 3] = Rr, t[b] - (Rr @ t[a][..., None])[..., 0], 1.0
        gy, gx = (torch.linspace(-1 + 1 / n, 1 - 1 / n, n, dtype=torch.float32) for n in (H, W))
        grid = torch.stack(torch.meshgrid(gy, gx, indexing="ij")[::-1], -1).expand(len(a), H, W, 2)
        if views["intrinsics"] is None:
            x2, prob = get_gt_warp(depth[a].to(device), depth[b].to(device), T.to(device), views["K"][a].to(device),
                                   views["K"][b].to(device))
            x2 = x2.float()
        else:
            x2, prob = _radial_gt_warp(views, a, b, T, H, W)
            x2, prob = x2.to(device), prob.to(device)
        halves.append((grid.to(device), x2, prob))
    (g0, m0, p0), (g1, m1, p1) = halves
    warp = torch.cat((torch.cat((g0, m0), -1), torch.cat((m1, g1), -1)), 2)
    return warp.contiguous(), torch.cat((p0, p1), 2).contiguous()


def _radial_gt_warp(views, a, b, T, H, W):
    import numpy as np

    intr, depth, sizes = views["intrinsics"].numpy(), views["depth"].numpy(), views["image_sizes"].numpy()
    ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
    x2 = np.zeros((len(a), H, W, 2), np.float32)
    prob = np.zeros((len(a), H, W), np.float32)
    for q, (ia, ib) in enumerate(zip(a.tolist(), b.tolist())):
        fa, ca = intr[ia], intr[ib]
        ra, rb = _radial_rays(fa, xs, ys)              # the views' images are the size of their grids
        d = depth[ia].astype(np.float64)
        P = np.stack((ra * d, rb * d, d), -1) @ T[q, :3, :3].numpy().T + T[q, :3, 3].numpy()
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = P[..., 0] / P[..., 2], P[..., 1] / P[..., 2]
            dd = 1.0 + ca[3] * (x * x + y * y)
            u, v = ca[0] * dd * x + ca[1], ca[0] * dd * y + ca[2]
            Hb, Wb = sizes[ib]
            cov = (u > 0) & (u < Wb - 1) & (v > 0) & (v < Hb - 1)
            col = np.clip(np.floor(u * W / Wb), 0, W - 1).astype(np.int64)
            row = np.clip(np.floor(v * H / Hb), 0, H - 1).astype(np.int64)
            db = depth[ib][np.where(cov, row, 0), np.where(cov, col, 0)].astype(np.float64)
            ok = (d > 0) & cov & (np.abs((db - P[..., 2]) / db) < 0.05)
        x2[q] = np.stack((2 * u / Wb - 1, 2 * v / Hb - 1), -1)
        prob[q] = ok
    return torch.from_numpy(np.nan_to_num(x2)), torch.from_numpy(prob)
