"""Geometric verification of a match graph on the device (`verify_matches`): a MAGSAC++ fundamental matrix per pair, and only its
inlier matches kept, the stage COLMAP and GLOMAP run between matching and track building.  Its output is a `MatchGraph` that
`build_tracks` takes unchanged.  The exact rules are in include/romab200.h and INTEGRATION.md; `oracle/verify.py` restates them in
numpy around a given estimator."""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass

import torch

from . import cabi, geometry
from .match_graph import WORKSPACE_BYTES, MatchGraph
from .matcher import pair_tensor


@dataclass
class PairGeometry:
    """Per pair k of the graph: F[k] float64 [3, 3] (x1^T F x0 = 0, unit Frobenius norm; zero where there is no model), ok[k] bool (a
    model was found), num_inliers[k] int64 (the matches within `threshold` of F) and accepted[k] bool (ok and num_inliers >=
    min_inliers).  Tensors live on the graph's device."""
    F: torch.Tensor
    ok: torch.Tensor
    num_inliers: torch.Tensor
    accepted: torch.Tensor


def _bytes(B, total, top):
    S = max(1, -(-top // geometry.FUND_SLICE))
    return (B * (cabi.RB_VERIFY_PAIR_BYTES + cabi.RB_VERIFY_SLICE_BYTES * S) + cabi.RB_VERIFY_POINT_BYTES * max(total, 1)
            + cabi.RB_VERIFY_CHUNK_BYTES)


def chunk_bytes(ns) -> int:
    """Device bytes of one estimator chunk whose pairs have ns[k] matches (include/romab200.h): the buffers `geometry._fund_launch`
    allocates plus the gathered points and offsets.  The score slices of every pair follow the chunk's largest pair."""
    return _bytes(len(ns), sum(ns), max(ns))


def plan_chunks(ns, workspace_bytes) -> list:
    """Consecutive pair ranges [b, e) covering all pairs: each run is as long as `chunk_bytes` of its pairs stays within
    `workspace_bytes`; a pair over the budget alone gets a chunk of its own."""
    chunks, b, P = [], 0, len(ns)
    while b < P:
        e, total, top = b + 1, ns[b], ns[b]
        while e < P and _bytes(e + 1 - b, total + ns[e], max(top, ns[e])) <= workspace_bytes:
            e, total, top = e + 1, total + ns[e], max(top, ns[e])
        chunks.append((b, e))
        b = e
    return chunks


def _int(name, v, lo):
    if isinstance(v, bool):
        raise ValueError(f"verify_matches: {name} must be an int >= {lo}, got {v!r}")
    try:
        v = operator.index(v)
    except TypeError:
        raise ValueError(f"verify_matches: {name} must be an int >= {lo}, got {v!r}") from None
    if v < lo:
        raise ValueError(f"verify_matches: {name} must be an int >= {lo}, got {v!r}")
    return v


def _check(pairs, graph, threshold, confidence, max_iters, min_inliers, seed, workspace_bytes):
    """Argument rules, checked before any device work.  Returns (pairs [P, 2] int64 CPU, threshold, confidence, max_iters,
    min_inliers, seed, workspace_bytes)."""
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"verify_matches: graph must be a MatchGraph, got {type(graph).__name__}")
    kp_off, m_off = graph._kp_off, graph._m_off
    for name, t, off in (("kp_offsets", graph.kp_offsets, kp_off), ("match_offsets", graph.match_offsets, m_off)):
        if t.dtype != torch.int64 or t.dim() != 1 or t.numel() < 1:
            raise ValueError(f"verify_matches: graph.{name} must be a 1-D int64 tensor of at least one entry, got {t.dtype} {tuple(t.shape)}")
        if off[0] != 0 or any(b < a for a, b in zip(off, off[1:])):
            raise ValueError(f"verify_matches: graph.{name} must start at 0 and never decrease")
    N, P, K, M = len(kp_off) - 1, len(m_off) - 1, kp_off[-1], m_off[-1]
    if graph.keypoints.dtype != torch.float32 or tuple(graph.keypoints.shape) != (K, 2):
        raise ValueError(f"verify_matches: graph.keypoints must be fp32 [{K}, 2], got {graph.keypoints.dtype} {tuple(graph.keypoints.shape)}")
    if graph.matches.dtype != torch.int32 or tuple(graph.matches.shape) != (M, 2):
        raise ValueError(f"verify_matches: graph.matches must be int32 [{M}, 2], got {graph.matches.dtype} {tuple(graph.matches.shape)}")
    if graph.match_scores.dtype != torch.float32 or tuple(graph.match_scores.shape) != (M,):
        raise ValueError(f"verify_matches: graph.match_scores must be fp32 [{M}], got {graph.match_scores.dtype} {tuple(graph.match_scores.shape)}")
    pairs = pair_tensor(pairs, N)
    if pairs.shape[0] != P:
        raise ValueError(f"verify_matches: {pairs.shape[0]} pairs, but the graph has matches for {P}")
    if P >= 1 << 31:
        raise ValueError(f"verify_matches: {P} pairs, at most 2^31 - 1 are supported")
    try:
        threshold, confidence = float(threshold), float(confidence)
    except (TypeError, ValueError):
        raise ValueError(f"verify_matches: threshold and confidence must be numbers, got {threshold!r} and {confidence!r}") from None
    if not (math.isfinite(threshold) and threshold > 0):
        raise ValueError(f"verify_matches: threshold must be finite and > 0, got {threshold!r}")
    if not 0 < confidence < 1:
        raise ValueError(f"verify_matches: confidence must lie in (0, 1), got {confidence!r}")
    max_iters = _int("max_iters", max_iters, 1)
    if max_iters >= 1 << 31:
        raise ValueError(f"verify_matches: max_iters must be below 2^31, got {max_iters}")
    min_inliers = _int("min_inliers", min_inliers, 0)
    workspace_bytes = _int("workspace_bytes", workspace_bytes, 1)
    seed = operator.index(seed)
    if K == 0 and M > 0:
        raise ValueError("verify_matches: the graph has matches but no keypoints, so every match id is out of range")
    tensors = [graph.kp_offsets, graph.keypoints, graph.kp_scores, graph.match_offsets, graph.matches, graph.match_scores]
    dev = graph.kp_offsets.device
    if not all(isinstance(t, torch.Tensor) and t.is_cuda and t.device == dev for t in tensors):
        raise ValueError(f"verify_matches: the graph's tensors must be on one CUDA device, got {[getattr(t, 'device', t) for t in tensors]}")
    return pairs, threshold, confidence, max_iters, min_inliers, seed, workspace_bytes


def verify_matches(pairs, graph: MatchGraph, *, threshold=2.0, confidence=0.999, max_iters=10000, min_inliers=15, seed=0,
                   workspace_bytes=WORKSPACE_BYTES):
    """Geometric verification of `graph`, the MatchGraph built from `pairs` (the rules of `match_pairs`).  Returns (verified
    MatchGraph, PairGeometry).

    Pair k = (i, j) gets the fundamental matrix `find_fundamental_batched` estimates from its matches' keypoints (MAGSAC++ over
    seven-point samples, sigma_max = `threshold` px of the image_sizes frame, `confidence`, at most `max_iters` hypotheses, the sample
    stream of `seed`), bit-identical to that call on the pair alone.  It is accepted when a model was found and at least
    `min_inliers` matches have a Sampson distance below `threshold`; the verified graph keeps exactly those matches of accepted pairs,
    in order and with their scores, and no match of a rejected pair.  Its kp_offsets, keypoints and kp_scores are the input's own
    tensors, and match_offsets still has P + 1 entries, so keypoint ids and pair indices do not change.  The defaults of confidence,
    max_iters and min_inliers are COLMAP's two-view verification.  The default threshold, 2 px, suits keypoints snapped to pixel
    cells of 1 px (`consolidate_matches`): on `synthetic.planted_cameras` with 0.5 px noise the true residual of an inlier is about
    0.6 px per coordinate (noise plus the cell's quantisation), so 2 px keeps the inliers while an outlier rarely falls inside the
    band around its epipolar line.  The quantisation grows with cell_size: at cell_size 4 the same scenes keep about 88 % of their
    inliers at 2 px and 97-99 % at 3 px, so pass about 3 px there.

    Bit-identical from run to run, for any `workspace_bytes` (the device memory of one estimator chunk, 1 GiB by default; a pair
    larger than that runs alone) and under any pair order.  Arguments are checked before any device work; a match id outside its
    image's keypoints raises ValueError (the device checks every id before using it, and no estimate runs then).  Host reads: the
    status word, the estimator's `running` flag once per chunk and round of 1 024 hypotheses before the last, and the kept total
    (the returned MatchGraph then reads its offsets, as every MatchGraph does)."""
    pairs, thr, conf, max_iters, min_inliers, seed, workspace_bytes = _check(pairs, graph, threshold, confidence, max_iters, min_inliers,
                                                                            seed, workspace_bytes)
    kp_off, m_off = graph._kp_off, graph._m_off
    N, P, K, M = len(kp_off) - 1, len(m_off) - 1, kp_off[-1], m_off[-1]
    dev = graph.kp_offsets.device
    with torch.cuda.device(dev):
        F = torch.zeros(P, 9, dtype=torch.float64, device=dev)
        ok = torch.zeros(P, dtype=torch.uint8, device=dev)
        num_inliers = torch.zeros(P, dtype=torch.int64, device=dev)
        accepted = torch.zeros(P, dtype=torch.uint8, device=dev)
        if M == 0:
            out = MatchGraph(graph.kp_offsets, graph.keypoints, graph.kp_scores, torch.zeros(P + 1, dtype=torch.int64, device=dev),
                             torch.zeros(0, 2, dtype=torch.int32, device=dev), torch.zeros(0, device=dev))
            return out, PairGeometry(F.view(P, 3, 3), ok.bool(), num_inliers, accepted.bool())
        # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
        d_m_off = torch.tensor(m_off, dtype=torch.int64).to(dev, non_blocking=True)
        kw = dict(pairs=pairs.to(dev, non_blocking=True), num_pairs=P, num_images=N,
                  kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev, non_blocking=True), keypoints=graph.keypoints.contiguous(),
                  num_rows=K, match_offsets=d_m_off, matches=graph.matches.contiguous(), match_scores=graph.match_scores.contiguous(),
                  num_matches=M, info=torch.empty(2, dtype=torch.int64, device=dev))
        cabi.call("romab200_verify_check", "rb_verify_args", **kw)
        if int(kw["info"][0].item()) & cabi.RB_VERIFY_BAD_ID:
            raise ValueError("verify_matches: a match id lies outside its image's keypoints")

        mask = torch.empty(M, dtype=torch.uint8, device=dev)
        ns = [e - b for b, e in zip(m_off, m_off[1:])]
        for b, e in plan_chunks(ns, workspace_bytes):
            m0, m1 = m_off[b], m_off[e]
            x0 = torch.empty(max(m1 - m0, 1), 2, dtype=torch.float64, device=dev)
            x1 = torch.empty_like(x0)
            off = torch.empty(e - b + 1, dtype=torch.int64, device=dev)
            cabi.call("romab200_verify_gather", "rb_verify_args", pair_begin=b, pair_end=e, x0=x0, x1=x1, chunk_offsets=off, **kw)
            buf = geometry._fund_launch(x0, x1, off, max(ns[b:e]), thr, conf, max_iters, seed)
            F[b:e] = buf["out_F"]
            ok[b:e] = buf["ok"]
            mask[m0:m1] = buf["mask"][:m1 - m0]
            del buf, x0, x1, off

        tiles = (M + cabi.RB_VERIFY_TILE - 1) // cabi.RB_VERIFY_TILE
        out_offsets = torch.empty(P + 1, dtype=torch.int64, device=dev)
        kw.update(ok=ok, mask=mask, min_inliers=min_inliers, num_inliers=num_inliers, accepted=accepted,
                  tile_scan=torch.empty(tiles + 1, dtype=torch.int64, device=dev), out_offsets=out_offsets)
        cabi.call("romab200_verify_count", "rb_verify_args", **kw)
        kept = int(kw["info"][1].item())
        out_matches = torch.empty(kept, 2, dtype=torch.int32, device=dev)
        out_scores = torch.empty(kept, device=dev)
        if kept:
            cabi.call("romab200_verify_emit", "rb_verify_args", num_kept=kept, out_matches=out_matches, out_scores=out_scores, **kw)
    out = MatchGraph(graph.kp_offsets, graph.keypoints, graph.kp_scores, out_offsets, out_matches, out_scores)
    return out, PairGeometry(F.view(P, 3, 3), ok.bool(), num_inliers, accepted.bool())
