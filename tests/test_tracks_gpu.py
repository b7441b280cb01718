"""`build_tracks` on the GPU: every output is bit-equal to the numpy oracle (oracle/tracks.py) on planted multi-view scenes, on match
graphs of uniform random samples (which hold a giant conflicting component), on a two-image zig-zag of 2^21 rows, a star, and
hand-built edge cases; two runs are byte-identical; the result does not change when pairs are reordered or reversed; planted tracks
come back exactly; and an out-of-range match id raises ValueError."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.tracks import tracks  # noqa: E402
from roma_b200 import MatchGraph, build_tracks, consolidate_matches, synthetic  # noqa: E402

DEV = "cuda"


def _assert_equal(res, ref):
    for name in ("track_offsets", "elements", "kp_track"):
        got, want = getattr(res, name).cpu(), torch.from_numpy(np.ascontiguousarray(ref[name]))
        assert got.dtype == want.dtype and got.shape == want.shape and torch.equal(got, want), name
    assert res.num_conflicting == ref["num_conflicting"]


def _check(pairs, g, **kw):
    res = build_tracks(pairs, g, **kw)
    ref = tracks(pairs.cpu().numpy() if isinstance(pairs, torch.Tensor) else pairs, g, **kw)
    _assert_equal(res, ref)
    return res, ref


def _planted(seed, N, outlier_frac, cs):
    pairs, m, c, sizes, views = synthetic.planted_views(seed, N, 600, size=(96, 128), cell_size=cs, outlier_frac=outlier_frac, device=DEV)
    return pairs, consolidate_matches(pairs, m, c, sizes, cell_size=cs), views


@pytest.mark.parametrize("seed, N, outlier_frac, cs", [(0, 3, 0.0, 1), (1, 3, 0.2, 4), (2, 8, 0.0, 4), (3, 8, 0.2, 1), (4, 30, 0.0, 1),
                                                       (5, 30, 0.2, 4), (6, 30, 0.2, 1)])
def test_planted_scenes_equal_the_oracle(seed, N, outlier_frac, cs):
    pairs, g, views = _planted(seed, N, outlier_frac, cs)
    scores = g.match_scores.cpu()
    at = float(scores.sort().values[len(scores) // 2])                  # a score present in the graph
    for min_length, drop, min_score in ((2, True, 0.0), (2, False, 0.0), (3, True, at), (3, False, 0.0), (2, True, at)):
        res, ref = _check(pairs, g, min_length=min_length, drop_conflicts=drop, min_score=min_score)
        assert len(res) > 0
    if outlier_frac == 0:
        for min_length in (2, 3):
            res = build_tracks(pairs, g, min_length=min_length)
            got = synthetic.track_cells(res.track_offsets, res.elements, g.kp_offsets, g.keypoints, 128, cs)
            assert got == synthetic.planted_tracks(views, min_length) and res.num_conflicting == 0


def _uniform(seed, N, P, n):
    """The uniform samples of tests/test_match_graph_gpu.py::_case, through consolidate_matches."""
    gen = torch.Generator().manual_seed(seed)
    sizes = torch.randint(8, 120, (N, 2), generator=gen)
    pairs = torch.randint(0, N, (P, 2), generator=gen)
    pairs[0] = pairs[0, 0]
    m = torch.rand(P, n, 4, generator=gen) * 2.2 - 1.1
    c = torch.rand(P, n, generator=gen)
    return pairs, consolidate_matches(pairs, m.to(DEV), c.to(DEV), sizes)


@pytest.mark.parametrize("seed, N, P, n", [(1, 5, 12, 3000), (2, 8, 30, 1000), (3, 4, 6, 10000)])
def test_uniform_samples_equal_the_oracle_with_a_giant_conflicting_component(seed, N, P, n):
    pairs, g = _uniform(seed, N, P, n)
    K = int(g.kp_offsets[-1])
    for drop in (True, False):
        res, ref = _check(pairs, g, drop_conflicts=drop)
    _check(pairs, g, min_length=3, min_score=0.5)
    giant = np.bincount(ref["root"]).max()
    assert giant > K // 4 and ref["num_conflicting"] >= 1
    assert int(torch.diff(res.track_offsets).max()) == giant                    # kept with drop_conflicts=False
    dropped = build_tracks(pairs, g)
    assert len(dropped) == 0 or int(torch.diff(dropped.track_offsets).max()) < giant


def _graph(kp_counts, pair_matches, scores=None):
    kp = torch.zeros(len(kp_counts) + 1, dtype=torch.int64)
    kp[1:] = torch.tensor(kp_counts).cumsum(0)
    mo = torch.zeros(len(pair_matches) + 1, dtype=torch.int64)
    mo[1:] = torch.tensor([len(x) for x in pair_matches]).cumsum(0)
    m = torch.cat([torch.as_tensor(x, dtype=torch.int32).reshape(-1, 2) for x in pair_matches]) if pair_matches else torch.zeros(0, 2, dtype=torch.int32)
    s = torch.ones(m.shape[0]) if scores is None else torch.as_tensor(scores, dtype=torch.float32)
    K = int(kp[-1])
    return MatchGraph(kp.to(DEV), torch.zeros(K, 2, device=DEV), torch.zeros(K, device=DEV), mo.to(DEV), m.to(DEV), s.to(DEV))


def test_zigzag_of_two_million_rows():
    """Pair (0, 1) matches a -> a, pair (1, 0) matches a -> a + 1: one component of 2^21 rows through deep unions."""
    n = 1 << 20
    a = torch.arange(n, dtype=torch.int32)
    g = _graph([n, n], [torch.stack((a, a), 1), torch.stack((a[:-1], a[1:]), 1)])
    pairs = [(0, 1), (1, 0)]
    res, _ = _check(pairs, g, drop_conflicts=False)
    assert len(res) == 1 and res.elements_of(0).shape == (2 * n, 2) and res.num_conflicting == 1
    assert bool((res.kp_track == 0).all())
    res, _ = _check(pairs, g)
    assert len(res) == 0 and res.num_conflicting == 1 and bool((res.kp_track == -1).all())


def test_star():
    """Keypoint 0 of image 0 matched to keypoint 1 of image j in pair (0, j), j = 1 .. 200."""
    pairs = [(0, j) for j in range(1, 201)]
    g = _graph([1] + [3] * 200, [[(0, 1)] for _ in pairs])
    res, _ = _check(pairs, g)
    assert len(res) == 1 and res.elements_of(0).tolist() == [[0, 0]] + [[j, 1] for j in range(1, 201)]


def test_id_ends_empty_images_and_empty_graphs():
    pairs = [(1, 3), (3, 1), (0, 4), (1, 1)]
    g = _graph([0, 5, 0, 3, 0], [[(0, 2), (4, 0)], [(2, 0), (0, 4)], [], [(4, 4)]])
    res, _ = _check(pairs, g)
    assert res.elements.tolist() == [[1, 0], [3, 2], [1, 4], [3, 0]]
    _check(pairs, g, drop_conflicts=False, min_length=3)
    res, _ = _check([(0, 1)], _graph([3, 2], [[]]))                           # M = 0
    assert len(res) == 0 and res.kp_track.tolist() == [-1] * 5
    res = build_tracks(torch.zeros(0, 2, dtype=torch.int64), _graph([0, 0, 0], []))   # K = 0
    assert res.track_offsets.tolist() == [0] and res.elements.shape == (0, 2) and res.kp_track.shape == (0,)


def test_two_runs_are_byte_identical():
    pairs, g, _ = _planted(7, 30, 0.2, 1)
    a, b = build_tracks(pairs, g, drop_conflicts=False), build_tracks(pairs, g, drop_conflicts=False)
    for name in ("track_offsets", "elements", "kp_track"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert a.num_conflicting == b.num_conflicting


def test_invariant_under_pair_order_and_reversal():
    pairs, g, _ = _planted(8, 8, 0.2, 1)
    P = pairs.shape[0]
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(0))
    flip = torch.rand(P, generator=torch.Generator().manual_seed(1)) < 0.5
    new_pairs, parts, scores = [], [], []
    for k in perm.tolist():
        m, s = g.matches_of(k), g.match_scores[g._m_off[k]:g._m_off[k + 1]]
        i, j = pairs[k].tolist()
        new_pairs.append((j, i) if flip[k] else (i, j))
        parts.append(m.flip(1) if flip[k] else m)
        scores.append(s)
    mo = torch.zeros(P + 1, dtype=torch.int64)
    mo[1:] = torch.tensor([p.shape[0] for p in parts]).cumsum(0)
    h = MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, mo.to(DEV), torch.cat(parts).contiguous(), torch.cat(scores))
    for kw in (dict(), dict(drop_conflicts=False, min_length=3)):
        a, b = build_tracks(pairs, g, **kw), build_tracks(new_pairs, h, **kw)
        for name in ("track_offsets", "elements", "kp_track"):
            assert torch.equal(getattr(a, name), getattr(b, name)), name
        assert a.num_conflicting == b.num_conflicting


@pytest.mark.parametrize("which, value", [(0, -1), (0, 5), (1, 3), (1, -(1 << 31))])
def test_out_of_range_match_id_raises(which, value):
    pairs = [(0, 1), (1, 2)]
    bad = [[(0, 0), (4, 2)], [(2, 0)]]
    bad[0][1] = tuple(value if c == which else x for c, x in enumerate(bad[0][1]))
    with pytest.raises(ValueError, match="outside"):
        build_tracks(pairs, _graph([5, 3, 1], bad))
    _check(pairs, _graph([5, 3, 1], [[(0, 0), (4, 2)], [(2, 0)]]))               # the device is fine afterwards
