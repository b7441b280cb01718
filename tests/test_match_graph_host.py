"""CPU tests of the match graph (`consolidate_matches`): the numpy oracle on hand-built cases (cell boundaries, clamping of x = W,
certainty ties broken by g and by s, non-finite values and min_certainty, i == j and repeated pairs, unreferenced images,
cell_size > 1), a planted track that must get one id per image in every pair that sees it, the argument rules (all raised before any
device work), the image grouping and the header's constants."""
import numpy as np
import pytest
import torch

from oracle.match_graph import consolidate
from roma_b200 import cabi, match_graph


def norm(px, size):
    """Normalised coordinate of pixel position px in an image side of `size` px (the inverse of x = size / 2 * (u + 1))."""
    return np.float32(2 * px / size - 1)


def sample(pairs, rows, sizes):
    """matches / certainty [P, n, 4] / [P, n] from rows[k] = [(xA, yA, xB, yB, certainty) in pixels]."""
    P, n = len(rows), max(len(r) for r in rows)
    m, c = np.zeros((P, n, 4), np.float32), np.zeros((P, n), np.float32)
    for k, (i, j) in enumerate(pairs):
        (hi, wi), (hj, wj) = sizes[i], sizes[j]
        for s, (xa, ya, xb, yb, w) in enumerate(rows[k]):
            m[k, s] = (norm(xa, wi), norm(ya, hi), norm(xb, wj), norm(yb, hj))
            c[k, s] = w
    return m, c


def test_pixel_position_and_cell_boundaries():
    # W = 8: u = -0.25 gives x = 4 * 0.75 = 3.0 exactly (cell 3); u + 1 one float below 0.75 gives x < 3 (cell 2)
    sizes = [(4, 8), (4, 8)]
    m = np.zeros((1, 2, 4), np.float32)
    m[0, 0] = (-0.25, 0.0, 0.0, 0.0)
    m[0, 1] = (np.nextafter(np.float32(0.75), np.float32(0)) - np.float32(1), 0.0, 0.5, 0.0)
    r = consolidate([(0, 1)], m, np.ones((1, 2), np.float32), sizes)
    assert r["keypoints"][0].tolist() == [np.float32(4) * np.nextafter(np.float32(0.75), np.float32(0)), 2.0]
    assert r["keypoints"][1].tolist() == [3.0, 2.0]                 # raster order: cell 2 before cell 3
    assert r["sid"][0, :, 0].tolist() == [1, 0]


def test_x_equal_to_w_clamps_into_the_last_cell():
    sizes = [(6, 10), (6, 10)]
    m = np.array([[[1.0, 1.0, -1.0, -1.0], [1.5, -3.0, 0.9, 0.9]]], np.float32)
    r = consolidate([(0, 1)], m, np.array([[0.5, 0.25]], np.float32), sizes)
    # image 0: (10, 6) -> cell (9, 5); (12.5, -6) -> cell (9, 0); image 1: (0, 0) -> (0, 0); (9.5, 5.7) -> (9, 5)
    assert r["kp_offsets"].tolist() == [0, 2, 4]
    assert r["keypoints"][:2].tolist() == [[12.5, -6.0], [10.0, 6.0]]
    assert r["keypoints"][2:].tolist() == [[0.0, 0.0], [np.float32(5) * np.float32(1.9), np.float32(3) * np.float32(1.9)]]


def test_certainty_ties_go_to_the_smallest_g():
    # image 1, pixel (2, 2): side B of pair 0 (g = 1) and side A of pair 1 (g = (1 * 1 + 0) * 2 = 2) tie; side B of pair 0 wins
    sizes = [(8, 8)] * 3
    m, c = sample([(0, 1), (1, 2)], [[(1.5, 1.5, 2.25, 2.25, 0.5)], [(2.75, 2.75, 5.5, 5.5, 0.5)]], sizes)
    r = consolidate([(0, 1), (1, 2)], m, c, sizes)
    assert r["kp_offsets"].tolist() == [0, 1, 2, 3]
    assert r["keypoints"][1].tolist() == [2.25, 2.25]
    # a higher certainty beats a smaller g
    c[1, 0] = 0.75
    r = consolidate([(0, 1), (1, 2)], m, c, sizes)
    assert r["keypoints"][1].tolist() == [2.75, 2.75] and r["kp_scores"][1] == np.float32(0.75)


def test_pair_ties_go_to_the_smallest_s_and_matches_are_mutual():
    sizes = [(8, 8), (8, 8)]
    rows = [(1.5, 1.5, 3.5, 3.5, 0.5),         # s = 0: a = (1, 1), b = (3, 3)
            (1.5, 1.5, 5.5, 5.5, 0.5),         # s = 1: same a, same certainty: best_b(a) stays s = 0
            (6.5, 6.5, 3.5, 3.5, 0.25),        # s = 2: b = (3, 3) again at lower certainty: best_a(b) is a = (1, 1), not kept
            (6.5, 0.5, 6.5, 0.5, 0.125)]       # s = 3: a lone mutual pair
    m, c = sample([(0, 1)], [rows], sizes)
    r = consolidate([(0, 1)], m, c, sizes)
    ids_a, ids_b = r["sid"][0, :, 0].tolist(), r["sid"][0, :, 1].tolist()
    assert ids_a == [1, 1, 2, 0] and ids_b == [1, 2, 1, 0]         # raster order: (6, 0) < (1, 1) < (6, 6); (6, 0) < (3, 3) < (5, 5)
    assert r["matches"].tolist() == [[0, 0], [1, 1]]
    assert r["match_scores"].tolist() == [0.125, 0.5]
    assert r["match_offsets"].tolist() == [0, 2]


def test_non_finite_values_and_min_certainty_are_ignored():
    sizes = [(8, 8), (8, 8)]
    m, c = sample([(0, 1)], [[(1.5, 1.5, 1.5, 1.5, 0.5), (2.5, 2.5, 2.5, 2.5, 0.5), (3.5, 3.5, 3.5, 3.5, 0.5),
                               (4.5, 4.5, 4.5, 4.5, 0.1), (5.5, 5.5, 5.5, 5.5, 0.0)]], sizes)
    m[0, 0, 0] = np.nan                       # side A of s = 0 ignored, its side B kept
    m[0, 1, 3] = np.inf
    c[0, 2] = np.inf                          # both sides ignored
    r = consolidate([(0, 1)], m, c, sizes, min_certainty=0.1)
    assert r["sid"][0].tolist() == [[-1, 0], [0, -1], [-1, -1], [-1, -1], [-1, -1]]
    assert r["kp_offsets"].tolist() == [0, 1, 2]
    assert len(r["matches"]) == 0 and r["match_offsets"].tolist() == [0, 0]
    assert consolidate([(0, 1)], m, c, sizes)["kp_offsets"].tolist() == [0, 2, 4]     # 0.1 > 0 counts at the default


def test_self_pairs_repeated_pairs_unreferenced_images_and_cell_size():
    sizes = [(8, 8), (16, 16), (8, 8), (8, 8)]
    pairs = [(0, 0), (0, 3), (0, 3)]
    m, c = sample(pairs, [[(1.5, 1.5, 2.5, 2.5, 0.5)], [(1.25, 1.25, 7.5, 7.5, 0.75)], [(2.5, 2.5, 7.75, 7.25, 0.5)]], sizes)
    r = consolidate(pairs, m, c, sizes)
    assert r["kp_offsets"].tolist() == [0, 2, 2, 2, 3]            # images 1 and 2 have no pair
    assert r["keypoints"][:2].tolist() == [[1.25, 1.25], [2.5, 2.5]]
    assert r["sid"][:, 0].tolist() == [[0, 1], [0, 0], [1, 0]]
    assert r["matches"].tolist() == [[0, 1], [0, 0], [1, 0]]
    r = consolidate(pairs, m, c, sizes, cell_size=4)             # everything of image 0 in cell (0, 0)
    assert r["kp_offsets"].tolist() == [0, 1, 1, 1, 2]
    assert r["keypoints"][0].tolist() == [1.25, 1.25] and r["matches"].tolist() == [[0, 0], [0, 0], [0, 0]]


def test_planted_track_gets_one_id_per_image():
    """One scene point seen by pairs (0, 1), (1, 2), (0, 2) at slightly different sub-pixel positions: one keypoint per image, and
    the three pair matches close a track."""
    sizes = [(40, 60), (50, 30), (20, 20)]
    pairs = [(0, 1), (1, 2), (0, 2)]
    track = {0: (10.5, 20.5), 1: (5.5, 33.5), 2: (17.5, 3.5)}
    rng = np.random.default_rng(0)
    rows = []
    for i, j in pairs:
        r = [(track[i][0] + rng.uniform(-0.2, 0.2), track[i][1] + rng.uniform(-0.2, 0.2), track[j][0] + rng.uniform(-0.05, 0.05),
              track[j][1] + rng.uniform(-0.05, 0.05), 0.9)]
        for _ in range(30):                   # background points elsewhere, lower certainty
            r.append((rng.uniform(0, sizes[i][1]), rng.uniform(0, sizes[i][0]), rng.uniform(0, sizes[j][1]), rng.uniform(0, sizes[j][0]), 0.3))
        rows.append(r)
    m, c = sample(pairs, rows, sizes)
    r = consolidate(pairs, m, c, sizes)
    ids = {}
    for k, (i, j) in enumerate(pairs):
        a, b = r["sid"][k, 0]
        assert ids.setdefault(i, a) == a and ids.setdefault(j, b) == b
        mk = r["matches"][r["match_offsets"][k]:r["match_offsets"][k + 1]].tolist()
        assert [a, b] in mk
    for i, (x, y) in track.items():
        kp = r["keypoints"][r["kp_offsets"][i] + ids[i]]
        assert (int(kp[0]), int(kp[1])) == (int(x), int(y))


def test_oracle_is_one_to_one_on_random_samples():
    rng = np.random.default_rng(1)
    sizes = [(12, 9), (7, 15), (10, 10)]
    pairs = [(0, 1), (1, 2), (2, 0), (1, 1), (0, 1)]
    m = rng.uniform(-1.1, 1.1, (5, 400, 4)).astype(np.float32)
    c = (rng.integers(0, 4, (5, 400)) / 4).astype(np.float32)
    r = consolidate(pairs, m, c, sizes, cell_size=2)
    for k in range(5):
        mk = r["matches"][r["match_offsets"][k]:r["match_offsets"][k + 1]]
        assert len(set(mk[:, 0])) == len(mk) and len(set(mk[:, 1])) == len(mk) and (np.diff(mk[:, 0]) > 0).all()
    for i, (h, w) in enumerate(sizes):
        kp = r["keypoints"][r["kp_offsets"][i]:r["kp_offsets"][i + 1]]
        cell = (np.clip(np.floor(kp[:, 1]), 0, h - 1) // 2) * ((w + 1) // 2) + np.clip(np.floor(kp[:, 0]), 0, w - 1) // 2
        assert (np.diff(cell) > 0).all()                            # one keypoint per cell, raster order


def test_empty_inputs():
    r = consolidate(np.zeros((0, 2)), np.zeros((0, 5, 4)), np.zeros((0, 5)), [(4, 4)])
    assert r["kp_offsets"].tolist() == [0, 0] and r["match_offsets"].tolist() == [0]
    r = consolidate([(0, 0)], np.zeros((1, 0, 4)), np.zeros((1, 0)), [(4, 4)])
    assert r["kp_offsets"].tolist() == [0, 0] and r["match_offsets"].tolist() == [0, 0]


@pytest.fixture
def no_device(monkeypatch):
    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))


@pytest.mark.parametrize("case, exc", [
    (dict(matches=torch.zeros(2, 5, 4, dtype=torch.float64)), ValueError),
    (dict(matches=torch.zeros(2, 5, 3)), ValueError),
    (dict(certainty=torch.zeros(2, 6)), ValueError),
    (dict(matches=torch.zeros(3, 5, 4), certainty=torch.zeros(3, 5)), ValueError),
    (dict(pairs=[(0, 3)]), IndexError),
    (dict(pairs=[(0, 1.5)]), ValueError),
    (dict(pairs=torch.zeros(2, 3, dtype=torch.int64)), ValueError),
    (dict(image_sizes=[(4, 0), (4, 4), (4, 4)]), ValueError),
    (dict(image_sizes=[(4, 4.0), (4, 4), (4, 4)]), ValueError),
    (dict(image_sizes=torch.ones(3, 2)), ValueError),
    (dict(image_sizes=torch.ones(3, 3, dtype=torch.int64)), ValueError),
    (dict(cell_size=0), ValueError),
    (dict(cell_size=2.0), ValueError),
    (dict(min_certainty=-0.5), ValueError),
    (dict(min_certainty=float("nan")), ValueError),
    (dict(workspace_bytes=0), ValueError),
    ({}, ValueError),                         # CPU tensors: the call runs on a CUDA device only
])
def test_argument_errors_before_device_work(no_device, case, exc):
    kw = dict(pairs=[(0, 1), (2, 2)], matches=torch.zeros(2, 5, 4), certainty=torch.zeros(2, 5), image_sizes=[(4, 4)] * 3)
    kw.update(case)
    extra = {k: kw.pop(k) for k in ("cell_size", "min_certainty", "workspace_bytes") if k in kw}
    with pytest.raises(exc):
        match_graph.consolidate_matches(kw["pairs"], kw["matches"], kw["certainty"], kw["image_sizes"], **extra)


def test_match_graph_needs_sizes_of_tensor_images(no_device):
    from roma_b200.matcher import RegressionMatcher
    with pytest.raises(ValueError, match="image_sizes"):
        RegressionMatcher.match_graph(None, torch.zeros(2, 3, 8, 8), [(0, 1)])
    with pytest.raises(ValueError, match="2 images"):
        RegressionMatcher.match_graph(None, torch.zeros(2, 3, 8, 8), [(0, 1)], image_sizes=[(8, 8)])
    with pytest.raises(ValueError, match="num"):
        RegressionMatcher.match_graph(None, torch.zeros(2, 3, 8, 8), [(0, 1)], num=0, image_sizes=[(8, 8)] * 2)


def test_image_sizes_default_to_the_file_header(tmp_path):
    from PIL import Image
    from roma_b200.matcher import _image_size
    p = tmp_path / "a.png"
    Image.new("RGB", (37, 21)).save(p)
    assert _image_size(str(p)) == (21, 37) and _image_size(Image.new("RGB", (5, 9))) == (9, 5)


def test_groups_cover_every_image_under_the_cap():
    assert match_graph._groups([0, 10, 0, 10, 10, 0], 20) == [(0, 4), (4, 6)]
    assert match_graph._groups([30, 5, 0], 20) == [(0, 1), (1, 3)]                 # an image over the cap stands alone
    assert match_graph._groups([5, 5, 5], 1) == [(0, 1), (1, 2), (2, 3)]
    assert match_graph._groups([0, 0], 1) == [(0, 2)]


def test_header_constants_and_pair_bytes():
    assert cabi.RB_MG_TILE == 2048 and "romab200_match_graph_keypoints" in cabi.FUNCTIONS
    assert {"romab200_match_graph_count", "romab200_match_graph_emit"} <= set(cabi.FUNCTIONS)
    assert match_graph.pair_bytes(10000) == 8 * 16384 + 50000 <= cabi.RB_MG_PAIR_SMEM      # num = 10 000 sorts in shared memory
    assert match_graph.pair_bytes(20000) > cabi.RB_MG_PAIR_SMEM and match_graph.pair_bytes(1) == 16
