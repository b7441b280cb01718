"""numpy restatement of the retrieval rules (include/romab200.h, "Retrieval"): the global descriptor from the full final-norm DINOv2
token array, the neighbour order and the pair list.  Scores are taken as given (`neighbors`) or, in `select_pairs`, as the float64
dot product rounded to fp32, which equals the device's fp32 FMA chain wherever every partial sum is exact (small dyadic entries)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

SQRT2 = np.float32(np.sqrt(2.0))


def _half(v):
    """v [E, C] fp32 -> v / (fp32(sqrt 2) * |v|) per row, |v| = sqrt of the squares summed in ascending channel order; 0 rows stay 0."""
    sq = np.cumsum(v * v, axis=1, dtype=np.float32)[:, -1]          # float32 cumsum is sequential
    norm = np.sqrt(sq).astype(np.float32)
    den = (SQRT2 * norm).astype(np.float32)
    out = np.zeros_like(v)
    nz = norm != 0
    out[nz] = v[nz] / den[nz, None]
    return out


def descriptor(tokens) -> np.ndarray:
    """tokens [E, 1 + n, C] (class token first) -> descriptors [E, 2C] fp32: [c / (sqrt2 |c|), m / (sqrt2 |m|)] with c the class
    token and m the patch tokens summed in ascending token order, then divided by n, every operation in fp32."""
    t = np.asarray(tokens, dtype=np.float32)
    n = t.shape[1] - 1
    m = (np.cumsum(t[:, 1:], axis=1, dtype=np.float32)[:, -1] / np.float32(n)).astype(np.float32)
    return np.concatenate((_half(t[:, 0].copy()), _half(m)), axis=1)


def neighbors(S, k):
    """S [N, N] fp32 scores -> (neighbors [N, k] int64, scores [N, k] fp32): per row the k largest S[i, j], j != i, score descending
    then j ascending (-0 counts as +0)."""
    S = np.asarray(S, dtype=np.float32)
    N = S.shape[0]
    nb = np.empty((N, k), dtype=np.int64)
    for i in range(N):
        j = np.array([c for c in range(N) if c != i], dtype=np.int64)
        s = S[i, j].astype(np.float64) + 0.0
        order = np.lexsort((j, -s))[:k]
        nb[i] = j[order]
    sc = np.take_along_axis(S, nb, axis=1) + np.float32(0)
    return nb, sc.astype(np.float32)


def pairs(nb, N) -> np.ndarray:
    """{(min(i, j), max(i, j)) : j in nb[i]}, unique, sorted by (i, j): [P, 2] int64."""
    i = np.repeat(np.arange(N, dtype=np.int64), nb.shape[1])
    j = nb.reshape(-1)
    keys = np.unique(np.minimum(i, j) * N + np.maximum(i, j))
    return np.stack((keys // N, keys % N), axis=1).astype(np.int64).reshape(-1, 2)


def select_pairs(X, num_neighbors=20):
    """(neighbors, scores, pairs) of descriptors X [N, D] with fp32(float64 X X^T) as the scores."""
    X = np.asarray(X, dtype=np.float64)
    N = X.shape[0]
    k = min(num_neighbors, N - 1)
    nb, sc = neighbors((X @ X.T).astype(np.float32), k)
    return nb, sc, pairs(nb, N)


def reference_tokens(oracle, x) -> torch.Tensor:
    """The final-norm DINOv2 tokens [B, 1 + n, 1024] (class token first) of images x [B, 3, H, W] from `roma_oracle.RomaOracle`'s
    ViT blocks: the token array whose patch rows `RomaOracle.dinov2` returns as a map."""
    d = oracle.d
    b = x.shape[0]
    t = F.conv2d(x, d["patch_embed.proj.weight"], d["patch_embed.proj.bias"], stride=14)
    hp, wp = t.shape[-2:]
    t = torch.cat((d["cls_token"].expand(b, -1, -1), t.flatten(2).transpose(1, 2)), dim=1) + oracle.dinov2_pos_embed(hp, wp)
    for i in range(24):
        t = oracle._vit_block(t, f"blocks.{i}", d, 16, 1e-6, True)
    return F.layer_norm(t, (1024,), d["norm.weight"], d["norm.bias"], 1e-6)
