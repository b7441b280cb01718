"""Pair selection for structure from motion (`select_pairs`): each image's nearest neighbours under the dot product of global
descriptors (`RegressionMatcher.global_descriptors`, or any others), as the deduplicated pair list that `match_pairs` and
`match_graph` take.  Scores come from romab200_gemm in blocks of rows that fit `workspace_bytes`, the neighbours from
`romab200_retrieval_select` and the pairs from `romab200_retrieval_pairs_*`.  The exact rules are in include/romab200.h and
INTEGRATION.md; `oracle/retrieval.py` restates them in numpy.  With synthetic weights the retrieval quality (recall of
overlapping pairs) is not measured, and it has not been measured on real DINOv2 weights either."""
from __future__ import annotations

import operator
from dataclasses import dataclass

import torch

from . import cabi
from .match_graph import WORKSPACE_BYTES


@dataclass
class RetrievalPairs:
    """neighbors [N, k] int64: row i's k nearest images j != i, score descending, then j ascending; scores [N, k] fp32 their dot
    products; pairs [P, 2] int64: {(min(i, j), max(i, j)) : j in neighbors[i]}, unique, sorted by (i, j).  On the descriptors' device."""
    neighbors: torch.Tensor
    scores: torch.Tensor
    pairs: torch.Tensor


def _check(descriptors, num_neighbors, workspace_bytes):
    """Argument rules, checked before any device work.  Returns (N, D, k, rows per score block)."""
    if not isinstance(descriptors, torch.Tensor) or not descriptors.dtype.is_floating_point:
        what = type(descriptors).__name__ if not isinstance(descriptors, torch.Tensor) else str(descriptors.dtype)
        raise ValueError(f"select_pairs: descriptors must be a floating-point CUDA tensor, got {what}")
    if descriptors.dim() != 2:
        raise ValueError(f"select_pairs: descriptors must be [N, D], got shape {tuple(descriptors.shape)}")
    N, D = descriptors.shape
    if not 2 <= N <= cabi.RB_RETRIEVAL_MAX_IMAGES:
        raise ValueError(f"select_pairs: {N} images, 2 to {cabi.RB_RETRIEVAL_MAX_IMAGES} are supported")
    if D < 1:
        raise ValueError("select_pairs: descriptors must have at least one component")
    try:
        if isinstance(num_neighbors, bool):
            raise TypeError
        num_neighbors = operator.index(num_neighbors)
    except TypeError:
        raise ValueError(f"select_pairs: num_neighbors must be an int in [1, {cabi.RB_RETRIEVAL_MAX_K}], got {num_neighbors!r}") from None
    if not 1 <= num_neighbors <= cabi.RB_RETRIEVAL_MAX_K:
        raise ValueError(f"select_pairs: num_neighbors must be an int in [1, {cabi.RB_RETRIEVAL_MAX_K}], got {num_neighbors!r}")
    rows = min(N, int(workspace_bytes) // (4 * N))
    if rows < 1:
        raise ValueError(f"select_pairs: workspace_bytes={workspace_bytes} holds no row of {N} fp32 scores ({4 * N} bytes)")
    if not descriptors.is_cuda:
        raise ValueError(f"select_pairs: descriptors must be a floating-point CUDA tensor, got one on {descriptors.device}")
    return N, D, min(num_neighbors, N - 1), rows


def select_pairs(descriptors, num_neighbors=20, *, workspace_bytes=WORKSPACE_BYTES) -> RetrievalPairs:
    """The pairs to match for an image set: each image with its min(num_neighbors, N - 1) nearest images by the dot product of the
    rows of `descriptors` [N, D] (a floating-point CUDA tensor, taken as contiguous fp32).

    The scores of `rows` rows against all N are made at a time in one block of at most `workspace_bytes` (there is no N x N buffer
    unless it fits), and the results are the same bytes for every `workspace_bytes`.  ValueError for arguments outside the rules
    (2 <= N <= 65535, 1 <= num_neighbors <= 128, D >= 1) before any device work, and for a non-finite descriptor or score after
    the selection (one host read, with the pair count)."""
    N, D, k, rows = _check(descriptors, num_neighbors, workspace_bytes)
    dev = descriptors.device
    with torch.cuda.device(dev):
        x = descriptors.detach().to(torch.float32).contiguous()
        block = torch.empty(rows * N, dtype=torch.float32, device=dev)
        neighbors = torch.empty(N, k, dtype=torch.int64, device=dev)
        scores = torch.empty(N, k, dtype=torch.float32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        for r0 in range(0, N, rows):
            r1 = min(N, r0 + rows)
            cabi.call("romab200_gemm", "rb_gemm_args", A=x[r0:r1], B=x, C=block, M=r1 - r0, N=N, K=D, lda=D, ldb=D, ldc=N, batch0=1, batch1=1,
                      ntaps=1, alpha=1.0, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32)
            cabi.call("romab200_retrieval_select", "rb_retrieval_args", num_images=N, k=k, scores=block, ld_scores=N, row_begin=r0, row_end=r1,
                      neighbors=neighbors, neighbor_scores=scores, status=status)
        total = N * k
        keys = torch.empty(total, dtype=torch.int64, device=dev)
        keys_alt = torch.empty(total, dtype=torch.int64, device=dev)
        hist = torch.empty(256 * (-(-total // cabi.RB_RETRIEVAL_TILE)) + 1, dtype=torch.int32, device=dev)
        offsets = torch.empty(total + 1, dtype=torch.int64, device=dev)
        kw = dict(num_images=N, k=k, neighbors=neighbors, keys=keys, keys_alt=keys_alt, hist=hist, offsets=offsets)
        cabi.call("romab200_retrieval_pairs_count", "rb_retrieval_args", **kw)
        bad, P = torch.cat((status.to(torch.int64), offsets[total:])).tolist()
        if bad:
            raise ValueError("select_pairs: a descriptor or a score is not finite")
        pairs = torch.empty(P, 2, dtype=torch.int64, device=dev)
        cabi.call("romab200_retrieval_pairs_emit", "rb_retrieval_args", num_pairs=P, pairs=pairs, **kw)
    return RetrievalPairs(neighbors, scores, pairs)
