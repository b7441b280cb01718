"""Feature tracks on the device (`build_tracks`): the connected components of a match graph's keypoint matches, i.e. each scene
point followed through every image that sees it, as a global SfM back end, a triangulator or a bundle adjuster takes them (COLMAP
calls the elements `TrackElement`s).  Components that put two keypoints of one image together are counted and, by default,
dropped.  The exact rules are in include/romab200.h and INTEGRATION.md; `oracle/tracks.py` restates them in numpy."""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass, field

import torch

from . import cabi
from .match_graph import MatchGraph
from .matcher import pair_tensor


@dataclass
class Tracks:
    """Track k is elements[track_offsets[k]:track_offsets[k + 1]]: int32 (image, keypoint id) rows, image ascending, then id
    ascending; its keypoint's row in the graph's keypoints is kp_offsets[image] + id.  kp_track [K] int32 is the track of every row
    of the keypoints, -1 for none.  num_conflicting counts the components that had two keypoints in one image.  Tensors live on the
    graph's device."""
    track_offsets: torch.Tensor
    elements: torch.Tensor
    kp_track: torch.Tensor
    num_conflicting: int
    _off: list = field(default=None, init=False, repr=False, compare=False)

    def __len__(self) -> int:
        return self.track_offsets.numel() - 1

    def elements_of(self, k: int) -> torch.Tensor:
        """[L_k, 2] int32 (image, keypoint id) of track k (a view).  The first call reads track_offsets to the host."""
        if self._off is None:
            self._off = self.track_offsets.tolist()
        return self.elements[self._off[k]:self._off[k + 1]]


def _offsets(name, t, off):
    """Checks a MatchGraph offset tensor and its host copy `off`: 1-D int64, starting at 0, never decreasing."""
    if t.dtype != torch.int64 or t.dim() != 1 or t.numel() < 1:
        raise ValueError(f"build_tracks: graph.{name} must be a 1-D int64 tensor of at least one entry, got {t.dtype} {tuple(t.shape)}")
    if off[0] != 0 or any(b < a for a, b in zip(off, off[1:])):
        raise ValueError(f"build_tracks: graph.{name} must start at 0 and never decrease")


def _check(pairs, graph, min_length, min_score):
    """Argument rules, checked before any device work.  Returns (pairs [P, 2] int64 CPU, kp_offsets and match_offsets as lists,
    min_length, min_score)."""
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"build_tracks: graph must be a MatchGraph, got {type(graph).__name__}")
    kp_off, m_off = graph._kp_off, graph._m_off
    _offsets("kp_offsets", graph.kp_offsets, kp_off)
    _offsets("match_offsets", graph.match_offsets, m_off)
    N, P, K, M = len(kp_off) - 1, len(m_off) - 1, kp_off[-1], m_off[-1]
    if K >= 1 << 31:
        raise ValueError(f"build_tracks: {K} keypoints, at most 2^31 - 1 are supported")
    if graph.matches.dtype != torch.int32 or tuple(graph.matches.shape) != (M, 2):
        raise ValueError(f"build_tracks: graph.matches must be int32 [{M}, 2], got {graph.matches.dtype} {tuple(graph.matches.shape)}")
    if graph.match_scores.dtype != torch.float32 or tuple(graph.match_scores.shape) != (M,):
        raise ValueError(f"build_tracks: graph.match_scores must be fp32 [{M}], got {graph.match_scores.dtype} {tuple(graph.match_scores.shape)}")
    pairs = pair_tensor(pairs, N)
    if pairs.shape[0] != P:
        raise ValueError(f"build_tracks: {pairs.shape[0]} pairs, but the graph has matches for {P}")
    if isinstance(min_length, bool):
        raise ValueError(f"build_tracks: min_length must be an int >= 2, got {min_length!r}")
    try:
        min_length = operator.index(min_length)
    except TypeError:
        raise ValueError(f"build_tracks: min_length must be an int >= 2, got {min_length!r}") from None
    if min_length < 2:
        raise ValueError(f"build_tracks: min_length must be an int >= 2, got {min_length!r}")
    try:
        score = float(min_score)
    except (TypeError, ValueError):
        raise ValueError(f"build_tracks: min_score must be a finite number >= 0, got {min_score!r}") from None
    if not (math.isfinite(score) and 0 <= score <= torch.finfo(torch.float32).max):
        raise ValueError(f"build_tracks: min_score must be a finite number >= 0, got {min_score!r}")
    if K == 0 and M > 0:
        raise ValueError("build_tracks: the graph has matches but no keypoints, so every match id is out of range")
    tensors = [graph.kp_offsets, graph.keypoints, graph.kp_scores, graph.match_offsets, graph.matches, graph.match_scores]
    dev = graph.kp_offsets.device
    if not all(isinstance(t, torch.Tensor) and t.is_cuda and t.device == dev for t in tensors):
        raise ValueError(f"build_tracks: the graph's tensors must be on one CUDA device, got {[getattr(t, 'device', t) for t in tensors]}")
    return pairs, kp_off, m_off, min_length, score


def build_tracks(pairs, graph: MatchGraph, *, min_length=2, min_score=0.0, drop_conflicts=True) -> Tracks:
    """Feature tracks of `graph`, the MatchGraph built from `pairs` (MatchGraph does not store them; the rules of `match_pairs`).

    Row r of graph.keypoints is a vertex; each match (a, b) of pair k = (i, j) with score > min_score (fp32) joins rows
    kp_offsets[i] + a and kp_offsets[j] + b.  A connected component with at least `min_length` rows is a track unless it holds two
    rows of one image (a conflict) and `drop_conflicts` is set; tracks are numbered by their smallest row.  Bit-identical from run to
    run.  Arguments are checked before any device work; a match id outside its image's keypoints raises ValueError (the device checks
    every id before using it).  Two host reads: the rows in components of two or more, and the final counts."""
    pairs, kp_off, m_off, min_length, min_score = _check(pairs, graph, min_length, min_score)
    N, P, K, M = len(kp_off) - 1, len(m_off) - 1, kp_off[-1], m_off[-1]
    dev = graph.kp_offsets.device
    if K == 0:
        return Tracks(torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(0, 2, dtype=torch.int32, device=dev),
                      torch.zeros(0, dtype=torch.int32, device=dev), 0)
    tile = cabi.RB_TRACKS_TILE
    with torch.cuda.device(dev):
        # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
        kw = dict(pairs=pairs.to(dev, non_blocking=True), num_pairs=P, num_images=N,
                  kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev, non_blocking=True), num_rows=K,
                  match_offsets=torch.tensor(m_off, dtype=torch.int64).to(dev, non_blocking=True), matches=graph.matches.contiguous(),
                  match_scores=graph.match_scores.contiguous(), num_matches=M, min_score=min_score, min_length=min_length,
                  drop_conflicts=int(bool(drop_conflicts)), parent=torch.empty(K, dtype=torch.int32, device=dev),
                  size=torch.empty(K, dtype=torch.int32, device=dev), tile_scan=torch.empty((K + tile - 1) // tile + 1, dtype=torch.int64, device=dev),
                  info=torch.empty(5, dtype=torch.int64, device=dev), kp_track=torch.empty(K, dtype=torch.int32, device=dev))
        cabi.call("romab200_tracks_link", "rb_tracks_args", **kw)
        status, kept = kw["info"][:2].tolist()
        _raise_on(status)
        if kept == 0:
            return Tracks(torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(0, 2, dtype=torch.int32, device=dev), kw["kp_track"], 0)
        track_offsets = torch.empty(kept // 2 + 1, dtype=torch.int64, device=dev)
        elements = torch.empty(kept, 2, dtype=torch.int32, device=dev)
        cabi.call("romab200_tracks_build", "rb_tracks_args", num_kept=kept, keys=torch.empty(kept, dtype=torch.int64, device=dev),
                  keys_alt=torch.empty(kept, dtype=torch.int64, device=dev),
                  hist=torch.empty(256 * ((kept + tile - 1) // tile) + 1, dtype=torch.int32, device=dev), track_offsets=track_offsets,
                  elements=elements, **kw)
        status, _, T, E, conflicting = kw["info"].tolist()
        _raise_on(status)
    return Tracks(track_offsets[:T + 1].clone(), elements[:E].clone(), kw["kp_track"], conflicting)


def _raise_on(status):
    if status & cabi.RB_TRACKS_BAD_ID:
        raise ValueError("build_tracks: a match id lies outside its image's keypoints")
    if status & cabi.RB_TRACKS_WALK:        # a parent walk longer than K steps, which the union-find's invariant rules out
        raise RuntimeError(f"build_tracks: union-find walk bound exceeded (status {status})")
