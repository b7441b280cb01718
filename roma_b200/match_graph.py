"""Structure-from-motion match graph on the device (`consolidate_matches`): sampled dense matches of many pairs over one image set ->
per-image keypoints with ids and one-to-one keypoint matches per pair, the two things an SfM back end (COLMAP, GLOMAP, any track
builder) takes.  Every sample side is snapped to a pixel cell of its image, so that one scene point sampled at slightly different
sub-pixel positions in different pairs becomes one keypoint and tracks close.  The exact rules are in include/romab200.h and
INTEGRATION.md; `oracle/match_graph.py` restates them in numpy."""
from __future__ import annotations

import operator
from dataclasses import dataclass

import torch

from . import cabi
from .matcher import pair_tensor

# Device workspace of one call beyond its inputs and outputs: the cell grids of a group of images (12 bytes per cell; an image whose
# grid alone is larger gets a group of its own) and, when n is too large for shared memory, the pair sorts of a chunk of pairs
WORKSPACE_BYTES = 1 << 30
_CELL_BYTES = 12
_MAX_SIDE = 1 << 24            # image sides up to 2^24 px keep W / 2 and W - 1 exact in fp32


@dataclass
class MatchGraph:
    """Keypoints of image i are keypoints[kp_offsets[i]:kp_offsets[i + 1]] (pixel (x, y) of the image_sizes frame, id = row within
    the image) with kp_scores; the matches of pair k are matches[match_offsets[k]:match_offsets[k + 1]] (int32 (a, b): a keypoint id
    in image pairs[k][0], b in pairs[k][1], ascending a) with match_scores.  All tensors live on the device of the input."""
    kp_offsets: torch.Tensor
    keypoints: torch.Tensor
    kp_scores: torch.Tensor
    match_offsets: torch.Tensor
    matches: torch.Tensor
    match_scores: torch.Tensor

    def __post_init__(self):
        self._kp_off = self.kp_offsets.tolist()
        self._m_off = self.match_offsets.tolist()

    def keypoints_of(self, i: int) -> torch.Tensor:
        """[K_i, 2] keypoints of image i (a view)."""
        return self.keypoints[self._kp_off[i]:self._kp_off[i + 1]]

    def matches_of(self, k: int) -> torch.Tensor:
        """[M_k, 2] int32 (a, b) keypoint ids of pair k (a view)."""
        return self.matches[self._m_off[k]:self._m_off[k + 1]]


def pair_bytes(n: int) -> int:
    """Bytes one pair's sorts take (include/romab200.h): shared memory up to RB_MG_PAIR_SMEM, otherwise scratch."""
    n2 = 1 << max(0, (n - 1).bit_length())
    return (8 * n2 + 5 * n + 15) // 16 * 16


def _check(pairs, matches, certainty, image_sizes, cell_size, min_certainty, workspace_bytes):
    """Argument rules, checked before any device work.  Returns (pairs [P, 2] int64 CPU, matches [P, n, 4], certainty [P, n],
    image_sizes [N, 2] int64 CPU)."""
    if not isinstance(matches, torch.Tensor) or not isinstance(certainty, torch.Tensor):
        raise ValueError("consolidate_matches: matches and certainty must be tensors")
    if matches.dtype != torch.float32 or certainty.dtype != torch.float32:
        raise ValueError(f"consolidate_matches: fp32 matches and certainty expected, got {matches.dtype} and {certainty.dtype}")
    if matches.dim() < 2 or matches.shape[-1] != 4 or tuple(matches.shape[:-1]) != tuple(certainty.shape):
        raise ValueError(f"consolidate_matches: matches [P, ..., 4] and certainty [P, ...] must share their leading shape, got "
                         f"{tuple(matches.shape)} and {tuple(certainty.shape)}")
    try:
        cell_size = operator.index(cell_size)
    except TypeError:
        raise ValueError(f"consolidate_matches: cell_size must be a positive int, got {cell_size!r}") from None
    if cell_size < 1:
        raise ValueError(f"consolidate_matches: cell_size must be a positive int, got {cell_size!r}")
    if not (float(min_certainty) >= 0.0):
        raise ValueError(f"consolidate_matches: min_certainty must be >= 0, got {min_certainty!r}")
    if int(workspace_bytes) < 1:
        raise ValueError(f"consolidate_matches: workspace_bytes must be positive, got {workspace_bytes!r}")
    if isinstance(image_sizes, torch.Tensor):
        if image_sizes.dtype.is_floating_point or image_sizes.dtype.is_complex or image_sizes.dtype == torch.bool:
            raise ValueError(f"consolidate_matches: image_sizes must hold integers, got {image_sizes.dtype}")
        sizes = image_sizes.detach().to("cpu", torch.int64)
    else:
        try:
            sizes = torch.tensor([[operator.index(h), operator.index(w)] for h, w in image_sizes], dtype=torch.int64).reshape(-1, 2)
        except (TypeError, ValueError):
            raise ValueError(f"consolidate_matches: image_sizes must be [N, 2] integers (H, W), got {image_sizes!r}") from None
    if sizes.dim() != 2 or sizes.shape[1] != 2:
        raise ValueError(f"consolidate_matches: image_sizes must be [N, 2] (H, W), got shape {tuple(sizes.shape)}")
    if sizes.numel() and (int(sizes.min()) < 1 or int(sizes.max()) > _MAX_SIDE):
        raise ValueError(f"consolidate_matches: image sizes must lie in [1, {_MAX_SIDE}], got {sizes.tolist()}")
    pairs = pair_tensor(pairs, sizes.shape[0])
    P = pairs.shape[0]
    if matches.shape[0] != P:
        raise ValueError(f"consolidate_matches: {P} pairs but matches for {matches.shape[0]}")
    n = certainty[0].numel() if P else 0
    if P * n * 2 >= 1 << 62 or n >= 1 << 31:
        raise ValueError(f"consolidate_matches: {n} samples per pair is too many")
    if not matches.is_cuda or matches.device != certainty.device:
        raise ValueError(f"consolidate_matches: matches ({matches.device}) and certainty ({certainty.device}) must be on one CUDA device")
    return pairs, matches.reshape(P, n, 4), certainty.reshape(P, n), sizes, cell_size


def _empty(N, P, dev):
    z = torch.zeros
    return MatchGraph(z(N + 1, dtype=torch.int64, device=dev), z(0, 2, device=dev), z(0, device=dev), z(P + 1, dtype=torch.int64, device=dev),
                      z(0, 2, dtype=torch.int32, device=dev), z(0, device=dev))


def consolidate_matches(pairs, matches, certainty, image_sizes, *, cell_size=1, min_certainty=0.0, workspace_bytes=WORKSPACE_BYTES) -> MatchGraph:
    """Keypoints and one-to-one matches of an image set from sampled matches of its pairs.

    pairs: [P, 2] integers or (i, j) sequence (the rules of `match_pairs`); matches [P, n, 4] fp32 normalised (xA, yA, xB, yB) and
    certainty [P, n] fp32 on a CUDA device, as `sample_batched` returns them ([P, R, n, 4] from repeats=R counts as n·R per pair);
    image_sizes [N, 2] integers (H, W) >= 1, the pixel frame keypoints are wanted in.  A sample side is snapped to the cell
    (floor(x), floor(y)) // cell_size of its image, clamped to the image; sides with certainty <= min_certainty or a non-finite value
    are ignored.  Each occupied cell becomes one keypoint at its most certain side's position (ties to the first sample), numbered in
    raster order per image; each pair keeps the mutual-best keypoint matches of its samples.  Bit-identical from run to run and for
    any `workspace_bytes`, the device memory the call may use beyond inputs and outputs (more groups of images and chunks of pairs when
    smaller).  Two host reads: the keypoint and the match count."""
    pairs, m, c, sizes, cell_size = _check(pairs, matches, certainty, image_sizes, cell_size, min_certainty, workspace_bytes)
    P, n, N, dev = pairs.shape[0], c.shape[1], sizes.shape[0], matches.device
    if P == 0 or n == 0:
        return _empty(N, P, dev)
    workspace_bytes = int(workspace_bytes)
    with torch.cuda.device(dev):
        m, c = m.contiguous(), c.contiguous()
        occ = torch.bincount(pairs.flatten(), minlength=N)
        H, W = sizes[:, 0], sizes[:, 1]
        cells = torch.where(occ > 0, ((H + cell_size - 1) // cell_size) * ((W + cell_size - 1) // cell_size), 0)
        tiles = (cells + cabi.RB_MG_TILE - 1) // cabi.RB_MG_TILE
        cell_start, tile_start = torch.zeros(N + 1, dtype=torch.int64), torch.zeros(N + 1, dtype=torch.int64)
        cell_start[1:], tile_start[1:] = cells.cumsum(0), tiles.cumsum(0)
        groups = _groups(cells.tolist(), max(1, workspace_bytes // _CELL_BYTES))
        kp_capacity = int(torch.minimum(cells, occ * n).sum())
        max_cells = max(int(cell_start[e] - cell_start[b]) for b, e in groups)
        max_tiles = max(int(tile_start[e] - tile_start[b]) for b, e in groups)

        d_pairs = pairs.to(dev, non_blocking=True)
        d_sizes = sizes.to(torch.int32).to(dev, non_blocking=True)
        d_cell_start, d_tile_start = cell_start.to(dev, non_blocking=True), tile_start.to(dev, non_blocking=True)
        grid_bits = torch.empty(max(max_cells, 1), dtype=torch.int32, device=dev)
        grid_g = torch.empty(max(max_cells, 1), dtype=torch.int64, device=dev)
        tile_scan = torch.empty(max_tiles + 1, dtype=torch.int64, device=dev)
        kp_offsets = torch.zeros(N + 1, dtype=torch.int64, device=dev)
        keypoints = torch.empty(max(kp_capacity, 1), 2, device=dev)
        kp_scores = torch.empty(max(kp_capacity, 1), device=dev)
        sid = torch.empty(P, n, 2, dtype=torch.int32, device=dev)
        for b, e in groups:
            cabi.call("romab200_match_graph_keypoints", "rb_match_graph_keypoints_args", pairs=d_pairs, num_pairs=P, n=n, matches=m,
                      certainty=c, image_sizes=d_sizes, num_images=N, cell_size=cell_size, min_certainty=float(min_certainty),
                      cell_start=d_cell_start, tile_start=d_tile_start, img_begin=b, img_end=e, grid_bits=grid_bits, grid_g=grid_g,
                      grid_cells=int(cell_start[e] - cell_start[b]), tile_scan=tile_scan, grid_tiles=int(tile_start[e] - tile_start[b]),
                      kp_offsets=kp_offsets, keypoints=keypoints, kp_scores=kp_scores, kp_capacity=kp_capacity, sid=sid)
        del grid_bits, grid_g, tile_scan
        K = int(kp_offsets[N].item())
        keypoints, kp_scores = keypoints[:K].clone(), kp_scores[:K].clone()

        pb = pair_bytes(n)
        chunk = P if pb <= cabi.RB_MG_PAIR_SMEM else max(1, min(P, workspace_bytes // pb))
        scratch = None if pb <= cabi.RB_MG_PAIR_SMEM else torch.empty(chunk * pb, dtype=torch.uint8, device=dev)
        match_offsets = torch.empty(P + 1, dtype=torch.int64, device=dev)
        kw = dict(sid=sid, certainty=c, num_pairs=P, n=n, scratch=scratch, scratch_bytes=0 if scratch is None else scratch.numel(),
                  match_offsets=match_offsets)
        for k0 in range(0, P, chunk):
            cabi.call("romab200_match_graph_count", "rb_match_graph_pairs_args", pair_begin=k0, pair_end=min(P, k0 + chunk), **kw)
        M = int(match_offsets[P].item())
        out = torch.empty(M, 2, dtype=torch.int32, device=dev)
        scores = torch.empty(M, device=dev)
        if M:
            for k0 in range(0, P, chunk):
                cabi.call("romab200_match_graph_emit", "rb_match_graph_pairs_args", pair_begin=k0, pair_end=min(P, k0 + chunk),
                          matches=out, match_scores=scores, match_capacity=M, **kw)
    return MatchGraph(kp_offsets, keypoints, kp_scores, match_offsets, out, scores)


def _groups(cells, cap):
    """Consecutive image ranges [b, e) covering all images, each with at most `cap` cells unless one image alone has more."""
    groups, b, acc = [], 0, 0
    for i, c in enumerate(cells):
        if c and acc and acc + c > cap:
            groups.append((b, i))
            b, acc = i, 0
        acc += c
    groups.append((b, len(cells)))
    return groups
