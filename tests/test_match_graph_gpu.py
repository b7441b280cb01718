"""`consolidate_matches` and `match_graph` on the GPU: the device result is bit-equal to the numpy oracle (oracle/match_graph.py) on
seeded uniform and clustered samples (several N, P and n, n above the shared-memory sort, cell_size 1 and 4, images of different
sizes, ties, non-finite values), the same under a tiny workspace (many image groups and pair chunks), byte-identical across runs,
and `match_graph` equals the hand-written match_pairs -> sample_batched -> consolidate_matches loop after the same seed."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

from conftest import ROOT  # noqa: E402
from oracle.match_graph import consolidate  # noqa: E402
from roma_b200 import consolidate_matches, roma_outdoor, synthetic  # noqa: E402

DEV = "cuda"


def _case(seed, N, P, n, clustered):
    g = torch.Generator().manual_seed(seed)
    sizes = torch.randint(8, 120, (N, 2), generator=g)
    pairs = torch.randint(0, N, (P, 2), generator=g)
    pairs[0] = pairs[0, 0]                                             # an (i, i) pair
    if clustered:
        # few centres, tiny spread and four certainty levels: many samples share a cell and a certainty, so the ties decide
        centres = torch.rand(6, 4, generator=g) * 2 - 1
        m = centres[torch.randint(0, 6, (P, n), generator=g)] + 0.01 * torch.randn(P, n, 4, generator=g)
        c = torch.randint(0, 5, (P, n), generator=g).float() / 4
    else:
        m = torch.rand(P, n, 4, generator=g) * 2.2 - 1.1                # some outside the image: clamped to its border
        c = torch.rand(P, n, generator=g)
    m[0, :3, 1] = float("nan")
    m[-1, :2, 2] = float("inf")
    c[-1, 5:7] = float("nan")
    m[:, -1] = 1.0                                                     # x = W, y = H
    return pairs, m.contiguous(), c.contiguous(), sizes


def _bits(t):
    t = t.detach().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def _assert_equal(res, ref):
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        got = _bits(getattr(res, name))
        want = _bits(torch.from_numpy(np.ascontiguousarray(ref[name])))
        assert got.shape == want.shape and torch.equal(got, want.to(got.dtype)), name


CASES = [  # (seed, N, P, n, clustered, cell_size)
    (0, 3, 4, 257, False, 1),
    (1, 5, 12, 3000, True, 1),
    (2, 8, 30, 1000, False, 4),
    (3, 4, 6, 10000, True, 4),
    (4, 6, 5, 20000, False, 1),                # 8 * 32768 + 5 * 20000 bytes: the sorts run in global scratch
    (5, 50, 40, 64, True, 1),
]


@pytest.mark.parametrize("seed, N, P, n, clustered, cs", CASES)
def test_bit_equal_to_the_oracle(seed, N, P, n, clustered, cs):
    pairs, m, c, sizes = _case(seed, N, P, n, clustered)
    ref = consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy(), cell_size=cs, min_certainty=0.0 if clustered else 0.05)
    res = consolidate_matches(pairs, m.to(DEV), c.to(DEV), sizes, cell_size=cs, min_certainty=0.0 if clustered else 0.05)
    _assert_equal(res, ref)
    assert ref["matches"].shape[0] > 0 and ref["keypoints"].shape[0] > 0
    for k in (0, P - 1):
        assert torch.equal(res.matches_of(k).cpu(), torch.from_numpy(ref["matches"][ref["match_offsets"][k]:ref["match_offsets"][k + 1]]))
    i = int(pairs[0, 0])
    assert torch.equal(res.keypoints_of(i).cpu(), torch.from_numpy(ref["keypoints"][ref["kp_offsets"][i]:ref["kp_offsets"][i + 1]]))


@pytest.mark.parametrize("seed, N, P, n, clustered, cs", [CASES[1], CASES[4], CASES[5]])
def test_tiny_workspace_gives_the_same_result(seed, N, P, n, clustered, cs):
    """4 KB: a group per image (each grid is larger than the cap) and, at n = 20 000, a pair chunk per pair."""
    pairs, m, c, sizes = _case(seed, N, P, n, clustered)
    m, c = m.to(DEV), c.to(DEV)
    big = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
    small = consolidate_matches(pairs, m, c, sizes, cell_size=cs, workspace_bytes=4096)
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        assert torch.equal(_bits(getattr(big, name)), _bits(getattr(small, name))), name


def test_two_runs_are_byte_identical():
    pairs, m, c, sizes = _case(7, 6, 20, 5000, True)
    m, c = m.to(DEV), c.to(DEV)
    a = consolidate_matches(pairs, m, c, sizes, cell_size=1)
    b = consolidate_matches(pairs, m, c, sizes, cell_size=1)
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        assert torch.equal(_bits(getattr(a, name)), _bits(getattr(b, name))), name


def test_repeats_and_empty_inputs():
    """[P, R, n, 4] from sample_batched(repeats=R) counts as n * R samples per pair; P = 0 and n = 0 give empty graphs."""
    pairs, m, c, sizes = _case(8, 4, 5, 600, False)
    res = consolidate_matches(pairs, m.view(5, 2, 300, 4).to(DEV), c.view(5, 2, 300).to(DEV), sizes)
    _assert_equal(res, consolidate(pairs.numpy(), m.numpy(), c.numpy(), sizes.numpy()))
    e = consolidate_matches(torch.zeros(0, 2, dtype=torch.int64), torch.zeros(0, 10, 4, device=DEV), torch.zeros(0, 10, device=DEV), sizes)
    assert e.kp_offsets.tolist() == [0] * 5 and e.match_offsets.tolist() == [0] and e.matches.shape == (0, 2)
    e = consolidate_matches(pairs, torch.zeros(5, 0, 4, device=DEV), torch.zeros(5, 0, device=DEV), sizes)
    assert e.kp_offsets.tolist() == [0] * 5 and e.match_offsets.tolist() == [0] * 6 and e.keypoints.shape == (0, 2)


PAIRS = [(i, j) for i in range(4) for j in range(i + 1, 4)] + [(2, 2), (1, 0)]


@pytest.fixture(scope="module")
def model(weights):
    return roma_outdoor(DEV, weights=weights[0], dinov2_weights=weights[1], coarse_res=112, upsample_res=168, amp_dtype=torch.float32)


def _by_hand(model, images, his, pairs, num, sizes, max_batch):
    buf = {}

    def on_batch(k0, warp, cert):
        mm, cc = model.sample_batched(warp, cert, num)
        if not buf:
            buf["m"], buf["c"] = torch.empty(len(pairs), mm.shape[2], 4, device=DEV), torch.empty(len(pairs), mm.shape[2], device=DEV)
        buf["m"][k0:k0 + mm.shape[0]] = mm[:, 0]
        buf["c"][k0:k0 + mm.shape[0]] = cc[:, 0]

    model.match_pairs(images, pairs, his, max_batch=max_batch, on_batch=on_batch)
    return consolidate_matches(pairs, buf["m"], buf["c"], sizes)


def test_match_graph_equals_the_hand_written_loop(model):
    A, B, Ah, Bh = synthetic.make_pair(2, 112, 168, seed=5)
    ims, his = torch.cat((A, B)).cuda(), torch.cat((Ah, Bh)).cuda()
    sizes = [(480, 640), (600, 800), (168, 168), (1000, 700)]
    torch.manual_seed(0)
    got = model.match_graph(ims, PAIRS, his, num=800, image_sizes=sizes, max_batch=3)
    torch.manual_seed(0)
    want = _by_hand(model, ims, his, PAIRS, 800, sizes, 3)
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        assert torch.equal(_bits(getattr(got, name)), _bits(getattr(want, name))), name
    assert got.matches.shape[0] > 100


def test_match_graph_defaults_to_the_file_sizes(model):
    paths = [os.path.join(ROOT, "tests", "golden", "jpeg", f) for f in ("sacre_coeur_A.jpg", "sacre_coeur_B.jpg", "toronto_A.jpg")]
    sizes = [Image.open(p).size[::-1] for p in paths]
    pairs = [(0, 1), (1, 2), (0, 2)]
    torch.manual_seed(1)
    got = model.match_graph(paths, pairs, num=500)
    torch.manual_seed(1)
    want = _by_hand(model, paths, None, pairs, 500, sizes, 8)
    for name in ("kp_offsets", "keypoints", "match_offsets", "matches"):
        assert torch.equal(_bits(getattr(got, name)), _bits(getattr(want, name))), name
    for i, (h, w) in enumerate(sizes):
        kp = got.keypoints_of(i)
        assert kp.shape[0] > 0 and float(kp[:, 0].max()) <= w and float(kp[:, 1].max()) <= h
