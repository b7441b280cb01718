"""numpy statement of `roma_b200.build_tracks` (include/romab200.h, INTEGRATION.md): the feature tracks of a match graph.  The
components come from `scipy.sparse.csgraph.connected_components`, an algorithm independent of the device's union-find; each label is
mapped to its smallest row, then lexsort, head flags and unique runs apply rules 3-5.  The device result is pinned to this bit for
bit."""
from __future__ import annotations

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def _arr(graph, name, dtype):
    v = graph[name] if isinstance(graph, dict) else getattr(graph, name)
    if hasattr(v, "detach"):
        v = v.detach().cpu().numpy()
    return np.asarray(v, dtype)


def tracks(pairs, graph, min_length=2, min_score=0.0, drop_conflicts=True):
    """pairs [P, 2] and a match graph (a dict or object with kp_offsets [N + 1], match_offsets [P + 1], matches [M, 2] and
    match_scores [M], as `oracle.match_graph.consolidate` or `consolidate_matches` return it).  Returns a dict of numpy arrays:
    track_offsets int64 [T + 1], elements int32 [E, 2] (image, keypoint id), kp_track int32 [K], num_conflicting (an int), and root
    int64 [K] (the smallest row of every row's component).  ValueError for a match id outside its image's keypoints."""
    kp = _arr(graph, "kp_offsets", np.int64)
    mo = _arr(graph, "match_offsets", np.int64)
    m = _arr(graph, "matches", np.int64).reshape(-1, 2)
    s = _arr(graph, "match_scores", np.float32).reshape(-1)
    pairs = np.asarray(pairs, np.int64).reshape(-1, 2)
    N, K = kp.size - 1, int(kp[-1])
    pair_of = np.repeat(np.arange(mo.size - 1), np.diff(mo))
    i, j = pairs[pair_of, 0], pairs[pair_of, 1]
    a, b = m[:, 0], m[:, 1]
    if ((a < 0) | (a >= kp[i + 1] - kp[i]) | (b < 0) | (b >= kp[j + 1] - kp[j])).any():
        raise ValueError("tracks: a match id lies outside its image's keypoints")
    edge = s > np.float32(min_score)                                       # fp32; NaN is never an edge
    u, v = kp[i[edge]] + a[edge], kp[j[edge]] + b[edge]

    rows = np.arange(K, dtype=np.int64)
    if K:
        _, label = connected_components(coo_matrix((np.ones(u.size, np.int8), (u, v)), shape=(K, K)), directed=False)
        first = np.full(label.max() + 1, K, np.int64)
        np.minimum.at(first, label, rows)
        root = first[label]
    else:
        root = rows
    image = np.repeat(np.arange(N), np.diff(kp))

    order = np.lexsort((rows, root))                                       # (root, row): rule 5
    sr, si = root[order], image[order]
    head = np.ones(K, bool)
    head[1:] = sr[1:] != sr[:-1]
    start = np.flatnonzero(head)
    size = np.diff(np.r_[start, K])
    clash = np.zeros(K, bool)
    clash[1:] = ~head[1:] & (si[1:] == si[:-1])                            # same component, same image as the predecessor
    conflict = np.add.reduceat(clash, start) > 0 if K else np.zeros(0, bool)
    keep = (size >= int(min_length)) & ~(conflict & bool(drop_conflicts))

    T = int(keep.sum())
    kept = np.repeat(keep, size)                                           # per sorted element
    el_rows = order[kept]
    track_offsets = np.zeros(T + 1, np.int64)
    track_offsets[1:] = np.cumsum(size[keep])
    kp_track = np.full(K, -1, np.int32)
    kp_track[el_rows] = np.repeat(np.arange(T, dtype=np.int32), size[keep])
    el_img = image[el_rows]
    elements = np.stack((el_img, el_rows - kp[el_img]), 1).astype(np.int32).reshape(-1, 2)
    return dict(track_offsets=track_offsets, elements=elements, kp_track=kp_track, num_conflicting=int(conflict.sum()), root=root)
