"""`verify_matches` on the GPU: on `planted_cameras` scenes every pair's F, ok, num_inliers and kept matches equal
`find_fundamental_batched` of that pair's gathered points alone, and the whole result equals `oracle/verify.py` fed those per-pair
results; the result does not depend on `workspace_bytes` or the pair order and two runs are byte-identical; an out-of-range match id
raises ValueError; and on a 16-image scene with 20 % outliers the verification keeps the planted inliers, removes the outliers and
improves `build_tracks`."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle.tracks import tracks as oracle_tracks  # noqa: E402
from oracle.verify import pair_points, verify  # noqa: E402
from roma_b200 import MatchGraph, USAC_MAGSAC, build_tracks, consolidate_matches, find_fundamental_batched, synthetic, verify_matches  # noqa: E402

DEV = "cuda"
THR = {1: 2.0, 4: 3.0}


def _scene(seed, N, outlier_frac, cs, points=400, size=(192, 256)):
    pairs, m, c, sizes, views = synthetic.planted_cameras(seed, N, points, size=size, cell_size=cs, outlier_frac=outlier_frac, device=DEV)[:5]
    return pairs, consolidate_matches(pairs, m, c, sizes, cell_size=cs), views


def _single(x0, x1, thr, seed=0):
    """find_fundamental_batched of one pair alone: (F [3, 3], ok, mask bool [n])."""
    F, ok, masks = find_fundamental_batched([torch.from_numpy(x0).to(DEV)], [torch.from_numpy(x1).to(DEV)], USAC_MAGSAC, thr, 0.999, 10000,
                                            seed=seed)
    return F[0].cpu().numpy(), bool(ok[0]), masks[0].view(-1).bool().cpu().numpy()


def _bytes_equal(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.cpu(), b.cpu())


def _same(r1, r2):
    (g1, p1), (g2, p2) = r1, r2
    return all(_bytes_equal(getattr(g1, n), getattr(g2, n)) for n in ("match_offsets", "matches", "match_scores")) and \
        all(_bytes_equal(getattr(p1, n), getattr(p2, n)) for n in ("F", "ok", "num_inliers", "accepted"))


@pytest.mark.parametrize("seed, N, outlier_frac, cs", [(0, 3, 0.0, 1), (1, 3, 0.2, 4), (2, 8, 0.2, 1), (3, 8, 0.0, 4), (4, 30, 0.2, 1),
                                                       (5, 30, 0.0, 1)])
def test_every_pair_equals_its_own_estimate_and_the_oracle(seed, N, outlier_frac, cs):
    pairs, g, _ = _scene(seed, N, outlier_frac, cs, points=250 if N == 30 else 400)
    thr = THR[cs]
    out, geom = verify_matches(pairs, g, threshold=thr)
    assert out.kp_offsets is g.kp_offsets and out.keypoints is g.keypoints and out.kp_scores is g.kp_scores
    assert out.match_offsets.numel() == pairs.shape[0] + 1
    pts = pair_points(pairs.cpu().numpy(), g)
    single = {}
    for k, (x0, x1) in enumerate(pts):
        if len(x0) >= 7:
            single[k] = _single(x0, x1, thr)
        else:
            assert not bool(geom.ok[k]) and bool((geom.F[k] == 0).all())
    for k, (F, ok, mask) in single.items():
        assert np.array_equal(geom.F[k].cpu().numpy(), F) and bool(geom.ok[k]) == ok and int(geom.num_inliers[k]) == int(mask.sum()), k
    ref = verify(pairs.cpu().numpy(), g, lambda k, x0, x1: (single[k][0] if single[k][1] else None, single[k][2]), min_inliers=15)
    for name in ("match_offsets", "matches", "match_scores"):
        got, want = getattr(out, name).cpu(), torch.from_numpy(np.ascontiguousarray(ref[name]))
        assert got.dtype == want.dtype and torch.equal(got, want), name
    for name in ("F", "ok", "num_inliers", "accepted"):
        assert torch.equal(getattr(geom, name).cpu(), torch.from_numpy(ref[name])), name
    assert bool(geom.accepted.any())


def test_workspace_pair_order_and_reruns():
    pairs, g, _ = _scene(6, 8, 0.2, 1)
    base = verify_matches(pairs, g)
    assert _same(base, verify_matches(pairs, g))                                   # byte-identical reruns
    assert _same(base, verify_matches(pairs, g, workspace_bytes=1))               # every pair its own chunk
    assert _same(base, verify_matches(pairs, g, workspace_bytes=3 << 20))
    P = pairs.shape[0]
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(0))
    parts = [g.matches_of(k) for k in perm.tolist()]
    scores = [g.match_scores[g._m_off[k]:g._m_off[k + 1]] for k in perm.tolist()]
    mo = torch.zeros(P + 1, dtype=torch.int64)
    mo[1:] = torch.tensor([p.shape[0] for p in parts]).cumsum(0)
    h = MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, mo.to(DEV), torch.cat(parts).contiguous(), torch.cat(scores))
    out, geom = verify_matches(pairs[perm.to(pairs.device)], h)
    (bo, bg) = base
    for name in ("F", "ok", "num_inliers", "accepted"):
        assert torch.equal(getattr(geom, name), getattr(bg, name)[perm.to(DEV)]), name
    for n, k in enumerate(perm.tolist()):
        assert torch.equal(out.matches_of(n), bo.matches_of(k))
        assert torch.equal(out.match_scores[out._m_off[n]:out._m_off[n + 1]], bo.match_scores[bo._m_off[k]:bo._m_off[k + 1]])


def test_repeated_self_and_tiny_pairs():
    pairs, g, _ = _scene(7, 3, 0.2, 1)
    P = pairs.shape[0]
    # pair 0 again, pair 1 reversed with its matches flipped, an i == j pair of identity matches, and a pair of 5 matches
    parts = [g.matches_of(0), g.matches_of(1).flip(1), torch.arange(40, dtype=torch.int32, device=DEV).repeat(2, 1).T.contiguous(),
             g.matches_of(2)[:5]]
    new_pairs = torch.cat([pairs, torch.tensor([pairs[0].tolist(), pairs[1].flip(0).tolist(), [0, 0], pairs[2].tolist()], device=pairs.device)])
    allm = [g.matches_of(k) for k in range(P)] + parts
    mo = torch.zeros(len(allm) + 1, dtype=torch.int64)
    mo[1:] = torch.tensor([p.shape[0] for p in allm]).cumsum(0)
    scores = torch.rand(int(mo[-1]), generator=torch.Generator().manual_seed(1)).to(DEV)
    h = MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, mo.to(DEV), torch.cat(allm).contiguous(), scores)
    out, geom = verify_matches(new_pairs, h)
    assert torch.equal(geom.F[P], geom.F[0]) and int(geom.num_inliers[P]) == int(geom.num_inliers[0])
    assert torch.equal(out.matches_of(P), out.matches_of(0)) and not bool(geom.ok[P + 3]) and out.matches_of(P + 3).shape[0] == 0
    pts = pair_points(new_pairs.cpu().numpy(), h)
    for k in (P + 1, P + 2):
        F, ok, mask = _single(*pts[k], 2.0)
        assert np.array_equal(geom.F[k].cpu().numpy(), F) and bool(geom.ok[k]) == ok and int(geom.num_inliers[k]) == int(mask.sum())


def test_no_matches():
    pairs, g, _ = _scene(8, 3, 0.0, 1)
    e = MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, torch.zeros(4, dtype=torch.int64, device=DEV),
                   torch.zeros(0, 2, dtype=torch.int32, device=DEV), torch.zeros(0, device=DEV))
    out, geom = verify_matches(pairs, e)
    assert out.match_offsets.tolist() == [0] * 4 and out.matches.shape == (0, 2) and not bool(geom.ok.any())
    assert geom.F.shape == (3, 3, 3) and geom.num_inliers.dtype == torch.int64 and geom.accepted.dtype == torch.bool


@pytest.mark.parametrize("which, value", [(0, -1), (0, 1 << 20), (1, -(1 << 31))])
def test_out_of_range_match_id_raises(which, value):
    pairs, g, _ = _scene(9, 3, 0.0, 1)
    m = g.matches.clone()
    m[g._m_off[1] + 3, which] = value
    bad = MatchGraph(g.kp_offsets, g.keypoints, g.kp_scores, g.match_offsets, m, g.match_scores)
    with pytest.raises(ValueError, match="outside"):
        verify_matches(pairs, bad)
    verify_matches(pairs, g)                                                           # the device is fine afterwards


def _labels(pairs, g, views, width):
    """Per match: True when its two keypoints are one planted point's views (cell_size 1)."""
    kp, xy = g.kp_offsets.cpu().numpy(), g.keypoints.cpu().numpy()
    mo, m = g.match_offsets.cpu().numpy(), g.matches.cpu().numpy().astype(np.int64)
    v = views.cpu().numpy()
    cell = np.floor(xy[:, 1]).astype(np.int64) * width + np.floor(xy[:, 0]).astype(np.int64)
    N = v.shape[1]
    lut = [np.full(int(v[:, i].max()) + 2, -1, np.int64) for i in range(N)]
    for i in range(N):
        seen = v[:, i] >= 0
        lut[i][v[seen, i]] = np.flatnonzero(seen)
    out = np.zeros(m.shape[0], bool)
    pr = pairs.cpu().numpy()
    for k, (i, j) in enumerate(pr):
        ci, cj = cell[kp[i] + m[mo[k]:mo[k + 1], 0]], cell[kp[j] + m[mo[k]:mo[k + 1], 1]]
        pi = np.where(ci < lut[i].size - 1, lut[i][np.minimum(ci, lut[i].size - 1)], -1)
        pj = np.where(cj < lut[j].size - 1, lut[j][np.minimum(cj, lut[j].size - 1)], -1)
        out[mo[k]:mo[k + 1]] = (pi >= 0) & (pi == pj)
    return out


def test_quality_on_a_planted_scene_with_outliers():
    H, W = 768, 1024
    pairs, m, c, sizes, views = synthetic.planted_cameras(11, 16, 20000, size=(H, W), outlier_frac=0.2, device=DEV)[:5]
    g = consolidate_matches(pairs, m, c, sizes)
    out, geom = verify_matches(pairs, g)
    inl = _labels(pairs, g, views, W)
    mo = g.match_offsets.cpu().numpy()
    kept = np.zeros(inl.size, bool)
    om, oo = out.matches.cpu().numpy(), out.match_offsets.cpu().numpy()
    gm = g.matches.cpu().numpy()
    for k in range(pairs.shape[0]):
        keys = gm[mo[k]:mo[k + 1], 0].astype(np.int64) << 32 | gm[mo[k]:mo[k + 1], 1]
        got = om[oo[k]:oo[k + 1], 0].astype(np.int64) << 32 | om[oo[k]:oo[k + 1], 1]
        kept[mo[k]:mo[k + 1]] = np.isin(keys, got)
    inlier_kept, outlier_removed = kept[inl].mean(), (~kept[~inl]).mean()
    before, after = build_tracks(pairs, g), build_tracks(pairs, out)
    planted = synthetic.planted_tracks(views)
    recall = [len(planted & synthetic.track_cells(t.track_offsets, t.elements, g.kp_offsets, g.keypoints, W)) / len(planted)
              for t in (before, after)]
    print(f"inliers kept {inlier_kept:.4f}, outliers removed {outlier_removed:.4f}, recall {recall[0]:.3f} -> {recall[1]:.3f}, "
          f"conflicting {before.num_conflicting} -> {after.num_conflicting}, accepted {int(geom.accepted.sum())} of {pairs.shape[0]}")
    assert inlier_kept >= 0.95 and outlier_removed >= 0.95
    assert recall[1] > recall[0] and after.num_conflicting < before.num_conflicting
    host = {k: getattr(out, k).cpu().numpy() for k in ("kp_offsets", "match_offsets", "matches", "match_scores")}
    ref = oracle_tracks(pairs.cpu().numpy(), host)
    assert torch.equal(after.track_offsets.cpu(), torch.from_numpy(ref["track_offsets"]))
