"""Retrieval on the GPU: `global_descriptors` bit for bit against the oracle fed the engine's own DINOv2 tokens in every precision mode
(and end to end against the CPU fp32 oracle in the parity mode), its batch and input-route invariance, and `select_pairs` exactly
against the oracle on dyadic descriptors, against float64 on random unit descriptors, for every workspace size, and composed with
`match_graph`."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import retrieval as oracle  # noqa: E402
from oracle.roma_oracle import RomaOracle  # noqa: E402
from roma_b200 import model_zoo, roma_outdoor, select_pairs, synthetic  # noqa: E402

MODES = {"fp32": (torch.float32, "tcgen05"), "fp32_simt": (torch.float32, "simt"), "fp16": (torch.float16, None), "bf16": (torch.bfloat16, None)}


def _model(weights, mode, coarse=112, up=168, **kw):
    amp, backend = MODES[mode]
    model_zoo.fp32_backend = backend
    try:
        return roma_outdoor("cuda", weights=weights[0], dinov2_weights=weights[1], coarse_res=coarse, upsample_res=up, amp_dtype=amp, **kw)
    finally:
        model_zoo.fp32_backend = None


@pytest.fixture(scope="module")
def images():
    A, B, _, _ = synthetic.make_pair(4, 112, 168, seed=9)
    return torch.cat((A, B))[:7].cuda()


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("mode", list(MODES))
def test_descriptor_equals_the_oracle_on_the_engines_tokens(weights, images, mode):
    model = _model(weights, mode)
    model.engine.debug = {}
    d = model.global_descriptors(images[:5])
    tokens = model.engine.debug["vit.out"]
    model.engine.debug = None
    assert tokens.shape == (5, 64 + 1, 1024)
    ref = torch.from_numpy(oracle.descriptor(tokens.cpu().numpy()))
    assert d.shape == (5, 2048) and d.dtype == torch.float32
    assert _bits_equal(d.cpu(), ref)
    assert _bits_equal(model.global_descriptors(images[:5]), d)          # the CUDA-graph replays compute the same bytes
    assert _bits_equal(model.global_descriptors(images[:5]), d)
    if mode == "fp32":
        ref = oracle.descriptor(oracle.reference_tokens(RomaOracle(*weights, coarse_res=112), images[:5].cpu()).numpy())
        err = np.abs(d.cpu().numpy() - ref).max()
        print(f"parity-mode descriptor vs CPU fp32 oracle: max abs err {err:.2e}")
        assert err <= 1e-4, err


def test_descriptor_batch_and_route_invariance(weights, images, tmp_path):
    model = _model(weights, "fp16")
    ref = model.global_descriptors(images, max_batch=1)
    for mb in (3, 8):
        assert _bits_equal(model.global_descriptors(images, max_batch=mb), ref), mb
    pils = synthetic.make_pil_pair(5) + synthetic.make_pil_pair(6)
    paths = []
    for i, im in enumerate(pils):
        paths.append(str(tmp_path / f"im{i}.png"))
        im.save(paths[-1])
    d_pil = model.global_descriptors(pils, max_batch=3)
    d_path = model.global_descriptors(paths, max_batch=2)
    d_tensor = model.global_descriptors(torch.cat(model._coarse_inputs(pils, ["pil"] * 4)[0]), max_batch=4)
    assert _bits_equal(d_pil, d_path) and _bits_equal(d_pil, d_tensor)
    assert model.global_descriptors(images[:0]).shape == (0, 2048)


def test_identical_images_have_identical_descriptors(weights, images):
    ims = images.clone()
    ims[5] = ims[1]
    model = _model(weights, "fp32")
    d = model.global_descriptors(ims, max_batch=4)
    assert _bits_equal(d[5], d[1]) and not torch.equal(d[0], d[1])
    res = select_pairs(d, 6)
    s = {(i, int(j)): float(v) for i in range(7) for j, v in zip(res.neighbors[i].tolist(), res.scores[i].tolist())}
    assert s[(1, 5)] == s[(5, 1)]
    assert (d.norm(dim=1) - 1).abs().max() < 1e-5


def _dyadic(N, D, seed):
    g = torch.Generator().manual_seed(seed)
    X = torch.randint(-4, 5, (N, D), generator=g).float() / 8
    X[17] = X[5]
    X[30] = X[2]
    X[31] = X[2]
    X[12] = 0
    return X


@pytest.mark.parametrize("N,D,k", [(40, 12, 5), (40, 7, 39), (40, 3, 1), (2, 5, 20), (300, 9, 128)])
def test_selection_equals_the_oracle_on_dyadic_descriptors(N, D, k):
    """Entries are multiples of 1/8 of at most 1/2, so every fp32 score is exact and ties are planted: duplicate rows, a zero row,
    and few distinct values at D = 3."""
    X = _dyadic(N, D, N + D) if N > 32 else torch.randint(-4, 5, (N, D), generator=torch.Generator().manual_seed(1)).float() / 8
    res = select_pairs(X.cuda(), k)
    nb, sc, pairs = oracle.select_pairs(X.numpy(), k)
    assert np.array_equal(res.neighbors.cpu().numpy(), nb)
    assert np.array_equal(res.scores.cpu().numpy().view(np.int32), sc.view(np.int32))
    assert np.array_equal(res.pairs.cpu().numpy(), pairs)
    assert res.neighbors.dtype == torch.int64 and res.pairs.dtype == torch.int64 and res.scores.dtype == torch.float32
    for ws in (4 * N, 4 * N * 3 + 5):
        again = select_pairs(X.cuda(), k, workspace_bytes=ws)
        assert torch.equal(again.neighbors, res.neighbors) and _bits_equal(again.scores, res.scores) and torch.equal(again.pairs, res.pairs)


@pytest.mark.parametrize("N", [1000, 5000])
def test_selection_on_random_unit_descriptors(N):
    D, k = 2048, 20
    g = torch.Generator(device="cuda").manual_seed(N)
    X = torch.randn(N, D, device="cuda", generator=g)
    X = X / X.norm(dim=1, keepdim=True)
    res = select_pairs(X, k)
    S = X.double() @ X.double().T
    assert (res.scores.double() - S.gather(1, res.neighbors)).abs().max().item() <= 1e-6
    S.fill_diagonal_(-float("inf"))
    S.scatter_(1, res.neighbors, -float("inf"))
    assert (S.max(dim=1).values - res.scores[:, -1].double()).max().item() <= 1e-6
    assert (res.neighbors != torch.arange(N, device="cuda")[:, None]).all()
    assert (res.scores[:, :-1] >= res.scores[:, 1:]).all()
    s = {}
    for i, (js, vs) in enumerate(zip(res.neighbors.tolist(), res.scores.view(torch.int32).tolist())):
        for j, v in zip(js, vs):
            s[(i, j)] = v
    both = [(i, j) for (i, j) in s if (j, i) in s]
    assert both and all(s[(i, j)] == s[(j, i)] for i, j in both)
    pairs = res.pairs.cpu()
    assert torch.equal(pairs, torch.unique(pairs, dim=0)) and (pairs[:, 0] < pairs[:, 1]).all() and pairs.shape[0] <= N * k
    assert (torch.bincount(pairs.flatten(), minlength=N) >= k).all()
    small = select_pairs(X, k, workspace_bytes=4 * N * (N // 5 - 3))
    assert torch.equal(small.neighbors, res.neighbors) and _bits_equal(small.scores, res.scores) and torch.equal(small.pairs, res.pairs)


def test_non_finite_descriptors_raise():
    X = torch.randn(50, 16, device="cuda")
    for bad in (float("nan"), float("inf")):
        Y = X.clone()
        Y[7, 3] = bad
        with pytest.raises(ValueError, match="not finite"):
            select_pairs(Y, 4)
    with pytest.raises(ValueError, match="not finite"):
        select_pairs(torch.full((4, 2), 3e38, device="cuda"), 2)


def test_selected_pairs_feed_match_graph(weights, images):
    model = _model(weights, "fp16", upsample_preds=False)
    d = model.global_descriptors(images)
    res = select_pairs(d, 2)
    sizes = [(112, 112)] * images.shape[0]
    torch.manual_seed(3)
    auto = model.match_graph(images, res.pairs, image_sizes=sizes, num=500)
    torch.manual_seed(3)
    hand = model.match_graph(images, [tuple(p) for p in res.pairs.tolist()], image_sizes=sizes, num=500)
    for name in ("kp_offsets", "keypoints", "kp_scores", "match_offsets", "matches", "match_scores"):
        assert torch.equal(getattr(auto, name), getattr(hand, name)), name
