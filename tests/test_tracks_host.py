"""CPU tests of feature tracks (`build_tracks`): the numpy oracle on hand-built match graphs (a closed triangle, a chain, a cycle that
puts two keypoints of one image together, i == j pairs and self-matches, repeated and reversed pairs, a score equal to min_score,
min_length 3, numbering by the smallest row, empty images, M = 0 and K = 0), the oracle against a plain union-find on seeded random
graphs, the planted generator's tracks through the match graph oracle, and the argument rules, all raised before any device work."""
import numpy as np
import pytest
import torch

from oracle.match_graph import consolidate
from oracle.tracks import tracks
from roma_b200 import cabi, synthetic, tracks as rb_tracks
from roma_b200.match_graph import MatchGraph


def graph(kp_counts, pair_matches):
    """A MatchGraph-like dict: kp_counts[i] keypoints in image i; pair_matches[k] = [(a, b) or (a, b, score), ...] of pair k."""
    kp = np.zeros(len(kp_counts) + 1, np.int64)
    kp[1:] = np.cumsum(kp_counts)
    mo = np.zeros(len(pair_matches) + 1, np.int64)
    mo[1:] = np.cumsum([len(m) for m in pair_matches])
    rows = [m for ms in pair_matches for m in ms]
    return dict(kp_offsets=kp, match_offsets=mo, matches=np.array([m[:2] for m in rows], np.int32).reshape(-1, 2),
                match_scores=np.array([m[2] if len(m) > 2 else 1.0 for m in rows], np.float32))


def as_lists(r):
    off = r["track_offsets"]
    return [r["elements"][off[t]:off[t + 1]].tolist() for t in range(len(off) - 1)]


def test_triangle_closes_into_one_track():
    g = graph([2, 2, 2], [[(0, 1)], [(1, 0)], [(0, 0)]])
    r = tracks([(0, 1), (1, 2), (0, 2)], g)
    assert as_lists(r) == [[[0, 0], [1, 1], [2, 0]]]
    assert r["kp_track"].tolist() == [0, -1, -1, 0, 0, -1] and r["num_conflicting"] == 0
    assert r["track_offsets"].tolist() == [0, 3]


def test_chain_over_four_images():
    g = graph([1, 3, 2, 1], [[(0, 2)], [(2, 1)], [(1, 0)]])
    r = tracks([(0, 1), (1, 2), (2, 3)], g)
    assert as_lists(r) == [[[0, 0], [1, 2], [2, 1], [3, 0]]]


def test_cycle_through_a_third_image_is_a_conflict():
    # 0:0 - 1:0 - 2:0 - 0:1: two keypoints of image 0 in one component
    g = graph([2, 1, 1], [[(0, 0)], [(0, 0)], [(0, 1)]])
    pairs = [(0, 1), (1, 2), (2, 0)]
    r = tracks(pairs, g)
    assert as_lists(r) == [] and r["num_conflicting"] == 1 and (r["kp_track"] == -1).all()
    r = tracks(pairs, g, drop_conflicts=False)
    assert as_lists(r) == [[[0, 0], [0, 1], [1, 0], [2, 0]]] and r["num_conflicting"] == 1


def test_self_pairs_conflict_and_self_matches_form_no_track():
    r = tracks([(0, 0)], graph([3], [[(0, 1), (2, 2)]]))
    assert as_lists(r) == [] and r["num_conflicting"] == 1
    r = tracks([(0, 0)], graph([3], [[(0, 1), (2, 2)]]), drop_conflicts=False)
    assert as_lists(r) == [[[0, 0], [0, 1]]] and r["kp_track"].tolist() == [0, 0, -1]
    r = tracks([(0, 0), (0, 1)], graph([3, 1], [[(2, 2)], [(1, 0)]]))
    assert as_lists(r) == [[[0, 1], [1, 0]]] and r["num_conflicting"] == 0


def test_repeated_and_reversed_pairs_just_add_edges():
    once = tracks([(0, 1), (1, 2)], graph([2, 2, 2], [[(0, 1), (1, 0)], [(1, 1)]]))
    again = tracks([(0, 1), (1, 0), (2, 1), (0, 1)], graph([2, 2, 2], [[(0, 1)], [(0, 1), (1, 0)], [(1, 1)], [(1, 0), (0, 1)]]))
    assert as_lists(once) == as_lists(again) == [[[0, 0], [1, 1], [2, 1]], [[0, 1], [1, 0]]]


def test_a_score_equal_to_min_score_is_not_an_edge():
    g = graph([1, 1, 1], [[(0, 0, 0.5)], [(0, 0, np.nextafter(np.float32(0.5), np.float32(1)))], [(0, 0, np.nan)]])
    r = tracks([(0, 1), (1, 2), (0, 2)], g, min_score=0.5)
    assert as_lists(r) == [[[1, 0], [2, 0]]]
    assert as_lists(tracks([(0, 1), (1, 2), (0, 2)], g)) == [[[0, 0], [1, 0], [2, 0]]]
    # min_score is rounded to fp32: 0.5 + 1e-12 is 0.5
    assert as_lists(tracks([(0, 1), (1, 2), (0, 2)], g, min_score=0.5 + 1e-12)) == [[[1, 0], [2, 0]]]


def test_min_length_three():
    g = graph([2, 2, 2], [[(0, 0), (1, 1)], [(0, 0)]])
    pairs = [(0, 1), (1, 2)]
    assert as_lists(tracks(pairs, g)) == [[[0, 0], [1, 0], [2, 0]], [[0, 1], [1, 1]]]
    r = tracks(pairs, g, min_length=3)
    assert as_lists(r) == [[[0, 0], [1, 0], [2, 0]]] and r["kp_track"].tolist() == [0, -1, 0, -1, 0, -1]


def test_tracks_are_numbered_by_their_smallest_row():
    # rows: image 0 = 0, 1; image 1 = 2, 3; image 2 = 4, 5.  Track {1, 2} comes after track {0, 5}, though 2 < 5.
    g = graph([2, 2, 2], [[(1, 0)], [(0, 1)]])
    r = tracks([(0, 1), (0, 2)], g)
    assert as_lists(r) == [[[0, 0], [2, 1]], [[0, 1], [1, 0]]] and r["kp_track"].tolist() == [0, 1, 1, -1, -1, 0]


def test_empty_images_no_matches_and_no_keypoints():
    g = graph([0, 2, 0, 1, 0], [[(1, 0)], []])
    r = tracks([(1, 3), (0, 4)], g)
    assert as_lists(r) == [[[1, 1], [3, 0]]] and r["kp_track"].tolist() == [-1, 0, 0]
    r = tracks([(0, 1)], graph([3, 2], [[]]))
    assert r["track_offsets"].tolist() == [0] and r["elements"].shape == (0, 2) and r["kp_track"].tolist() == [-1] * 5
    r = tracks(np.zeros((0, 2)), graph([0, 0], []))
    assert r["track_offsets"].tolist() == [0] and r["kp_track"].shape == (0,) and r["num_conflicting"] == 0
    with pytest.raises(ValueError):
        tracks([(0, 1)], graph([2, 2], [[(0, 2)]]))


def union_find_tracks(pairs, g, min_length, min_score, drop_conflicts):
    kp, mo = g["kp_offsets"], g["match_offsets"]
    parent = list(range(int(kp[-1])))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    for k, (i, j) in enumerate(pairs):
        for m in range(mo[k], mo[k + 1]):
            if g["match_scores"][m] > np.float32(min_score):
                a, b = find(kp[i] + g["matches"][m, 0]), find(kp[j] + g["matches"][m, 1])
                parent[max(a, b)] = min(a, b)
    comps = {}
    for r in range(len(parent)):
        comps.setdefault(find(r), []).append(r)
    image = np.repeat(np.arange(len(kp) - 1), np.diff(kp))
    out, conflicts = [], 0
    for root in sorted(comps):
        rows = comps[root]
        clash = len({image[r] for r in rows}) < len(rows)
        conflicts += clash
        if len(rows) >= min_length and not (clash and drop_conflicts):
            out.append([[int(image[r]), int(r - kp[image[r]])] for r in rows])
    return out, conflicts


@pytest.mark.parametrize("seed", range(6))
def test_oracle_equals_a_plain_union_find(seed):
    rng = np.random.default_rng(seed)
    N = int(rng.integers(2, 7))
    counts = rng.integers(0, 6, N)
    pairs = [tuple(rng.integers(0, N, 2)) for _ in range(int(rng.integers(1, 12)))]
    pm = [[(int(rng.integers(0, counts[i])), int(rng.integers(0, counts[j])), float(rng.integers(0, 4) / 4))
           for _ in range(int(rng.integers(0, 4)) if counts[i] and counts[j] else 0)] for i, j in pairs]
    g = graph(counts, pm)
    for min_length, min_score, drop in ((2, 0.0, True), (3, 0.25, False), (2, 0.5, False)):
        r = tracks(pairs, g, min_length, min_score, drop)
        want, conflicts = union_find_tracks(pairs, g, min_length, min_score, drop)
        assert as_lists(r) == want and r["num_conflicting"] == conflicts
        for t, els in enumerate(want):
            assert all(r["kp_track"][g["kp_offsets"][i] + a] == t for i, a in els)
        assert (r["kp_track"] >= 0).sum() == sum(len(e) for e in want)


@pytest.mark.parametrize("cell_size, min_length", [(1, 2), (4, 3)])
def test_planted_tracks_through_the_match_graph_oracle(cell_size, min_length):
    pairs, m, c, sizes, views = synthetic.planted_views(3, 6, 150, size=(48, 80), cell_size=cell_size, visibility=0.6)
    g = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy(), cell_size=cell_size)
    r = tracks(pairs.numpy(), g, min_length=min_length)
    got = synthetic.track_cells(torch.from_numpy(r["track_offsets"]), torch.from_numpy(r["elements"]), torch.from_numpy(g["kp_offsets"]),
                                torch.from_numpy(g["keypoints"]), 80, cell_size)
    want = synthetic.planted_tracks(views, min_length)
    assert len(want) > 50 and got == want and r["num_conflicting"] == 0


def test_planted_generator_shapes_and_outliers():
    pairs, m, c, sizes, views = synthetic.planted_views(1, 4, 60, size=(30, 40), outlier_frac=0.2)
    assert pairs.tolist() == [[0, 1], [0, 2], [0, 3], [1, 2], [1, 3], [2, 3]] and sizes.tolist() == [[30, 40]] * 4
    assert m.shape[:2] == c.shape and views.shape == (60, 4)
    inl = ((views[:, pairs[:, 0]] >= 0) & (views[:, pairs[:, 1]] >= 0)).sum(0)
    assert torch.equal((c >= 0.5).sum(1), inl)
    assert torch.equal(((c > 0) & (c < 0.5)).sum(1), torch.round(inl * 0.25).long())
    assert (m.abs() <= 1).all()


def mg(kp_offsets=(0, 2, 4, 6), match_offsets=(0, 1, 2), matches=((0, 1), (1, 0)), scores=(1.0, 1.0)):
    def t(x, dtype):
        return x if isinstance(x, torch.Tensor) else torch.tensor(x, dtype=dtype)

    return MatchGraph(t(kp_offsets, torch.int64), torch.zeros(1, 2), torch.zeros(1), t(match_offsets, torch.int64),
                      t(matches, torch.int32).reshape(-1, 2), t(scores, torch.float32))


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case, exc", [
    (dict(graph={"kp_offsets": torch.zeros(1, dtype=torch.int64)}), ValueError),   # not a MatchGraph
    (dict(pairs=[(0, 3)]), IndexError),
    (dict(pairs=[(0, 1.5), (1, 2)]), ValueError),
    (dict(pairs=torch.zeros(2, 3, dtype=torch.int64)), ValueError),
    (dict(pairs=[(0, 1)]), ValueError),                                             # two pairs of matches
    (dict(pairs=[(0, 1), (1, 2), (0, 2)]), ValueError),
    (dict(graph=mg(kp_offsets=(0, 2, 1, 6))), ValueError),                          # decreasing
    (dict(graph=mg(kp_offsets=(1, 2, 4, 6))), ValueError),
    (dict(graph=mg(match_offsets=(0, 2, 1))), ValueError),
    (dict(graph=mg(kp_offsets=torch.tensor([0, 2, 4, 6], dtype=torch.int32))), ValueError),
    (dict(graph=mg(kp_offsets=(0, 2, 1 << 30, 1 << 31))), ValueError),             # K = 2^31
    (dict(graph=mg(matches=((0, 1), (1, 0), (1, 1)))), ValueError),                 # more matches than match_offsets[P]
    (dict(graph=mg(matches=torch.zeros(2, 2, dtype=torch.int64))), ValueError),
    (dict(graph=mg(scores=(1.0,))), ValueError),
    (dict(graph=mg(kp_offsets=(0, 0, 0, 0))), ValueError),                          # matches but no keypoints
    (dict(min_length=1), ValueError),
    (dict(min_length=2.0), ValueError),
    (dict(min_length=True), ValueError),
    (dict(min_score=-0.5), ValueError),
    (dict(min_score=float("nan")), ValueError),
    (dict(min_score=float("inf")), ValueError),
    (dict(min_score=1e39), ValueError),                                             # infinite in fp32
    (dict(min_score="0.5x"), ValueError),
    ({}, ValueError),                                                               # CPU tensors: the call runs on a CUDA device only
])
def test_argument_errors_before_device_work(no_device, case, exc):
    kw = dict(pairs=[(0, 1), (1, 2)], graph=mg())
    kw.update(case)
    pairs, g = kw.pop("pairs"), kw.pop("graph")
    with pytest.raises(exc) as e:
        rb_tracks.build_tracks(pairs, g, **kw)
    assert ("CUDA device" in str(e.value)) == (not case)          # each case fails its own rule, not the device rule


def test_tracks_view_and_entry_points():
    t = rb_tracks.Tracks(torch.tensor([0, 2, 5]), torch.arange(10, dtype=torch.int32).reshape(5, 2), torch.zeros(3, dtype=torch.int32), 0)
    assert len(t) == 2 and t.elements_of(1).tolist() == [[4, 5], [6, 7], [8, 9]] and t.elements_of(0).shape == (2, 2)
    assert {"romab200_tracks_link", "romab200_tracks_build"} <= set(cabi.FUNCTIONS) and cabi.RB_TRACKS_TILE == 4096
