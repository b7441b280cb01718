"""`match_pairs` on the GPU: every pair of a graph over one image set equals what `match()` returns for that pair, in every precision
mode, with and without symmetry and upsampling, through tensors, paths and PIL images, chunk callbacks, CUDA-graph replays and a
freed arena.  Bar 1e-6 like test_sharding_gpu.py (per-pair arithmetic does not depend on the batch a pair travels in)."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu

from conftest import ROOT, load_golden  # noqa: E402
from roma_b200 import model_zoo, roma_outdoor, synthetic  # noqa: E402

TOL = 1e-6
JPEGS = [os.path.join(ROOT, "tests", "golden", "jpeg", f) for f in ("sacre_coeur_A.jpg", "sacre_coeur_B.jpg", "toronto_A.jpg")]
# all 10 unordered pairs of 5 images, one reversed pair, one repeated pair and one (i, i)
PAIRS = [(i, j) for i in range(5) for j in range(i + 1, 5)] + [(3, 1), (0, 1), (2, 2)]
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
    A, B, Ah, Bh = synthetic.make_pair(3, 112, 168, seed=7)
    return torch.cat((A, B))[:5].cuda(), torch.cat((Ah, Bh))[:5].cuda()


def _match_each(model, ims, his, pairs):
    outs = [model.match(ims[i:i + 1], ims[j:j + 1], im_A_high_res=his[i:i + 1] if model.upsample_preds else None,
                        im_B_high_res=his[j:j + 1] if model.upsample_preds else None) for i, j in pairs]
    return torch.cat([w for w, _ in outs]), torch.cat([c for _, c in outs])


def _err(a, b):
    return max((a[0] - b[0]).abs().max().item(), (a[1] - b[1]).abs().max().item())


@pytest.mark.parametrize("mode", list(MODES))
def test_match_pairs_equals_match(weights, images, mode):
    _check_equals_match(_model(weights, mode), *images, mode)


@pytest.mark.parametrize("mode", list(MODES))
def test_match_pairs_equals_match_odd_grid(weights, mode):
    """126 x 182 -> 182 x 238: a coarse grid of 9 x 13 = 117 tokens, an odd size for the per-image GP solve."""
    A, B, Ah, Bh = synthetic.make_pair(3, (126, 182), (182, 238), seed=7)
    model = _model(weights, mode, (126, 182), (182, 238))
    _check_equals_match(model, torch.cat((A, B))[:5].cuda(), torch.cat((Ah, Bh))[:5].cuda(), mode)


def _check_equals_match(model, ims, his, mode):
    model.use_cuda_graph = False          # eager on both sides; graph replays are covered below
    for symmetric in (True, False):
        for upsample in (True, False):
            model.symmetric, model.upsample_preds = symmetric, upsample
            ref = _match_each(model, ims, his, PAIRS)
            for max_batch in (2, 3):
                got = model.match_pairs(ims, PAIRS, his if upsample else None, max_batch=max_batch)
                assert got[0].shape == ref[0].shape and got[1].shape == ref[1].shape
                err = _err(got, ref)
                print(f"[{mode} sym={symmetric} up={upsample} max_batch={max_batch}] max-abs difference to match(): {err:.3e}")
                assert err <= TOL, (mode, symmetric, upsample, max_batch, err)


def test_match_pairs_golden_inside_larger_graph(weights):
    """The small_sym_up golden (made from the unmodified reference) as pair (1, 3) of a 4-image graph, in the parity mode."""
    g = load_golden("small_sym_up")
    coarse, up, sym, upp, batch, seed, step = (int(v) for v in g["meta"])
    A, B, Ah, Bh = synthetic.make_pair(batch, coarse, up, seed)
    X, Y, Xh, Yh = synthetic.make_pair(1, coarse, up, seed + 100)
    ims = torch.cat((X, A[:1], Y, B[:1])).cuda()
    his = torch.cat((Xh, Ah[:1], Yh, Bh[:1])).cuda()
    model = _model(weights, "fp32", coarse, up, symmetric=bool(sym), upsample_preds=bool(upp))
    warp, cert = model.match_pairs(ims, [(0, 2), (1, 3), (3, 1), (2, 1)], his, max_batch=3)
    w = warp[1:2, ::step, ::step].cpu().numpy()
    c = cert[1:2, ::step, ::step].cpu().numpy()
    assert w.shape == g["warp"][:1].shape
    assert np.abs(w - g["warp"][:1]).max() <= 1e-4 and np.abs(c - g["certainty"][:1]).max() <= 1e-4


@pytest.mark.parametrize("route", ["path", "pil"])
def test_match_pairs_path_and_pil_routes(weights, route):
    model = _model(weights, "fp32", symmetric=True, upsample_preds=True)
    inputs = JPEGS if route == "path" else [Image.open(p).convert("RGB") for p in JPEGS]
    pairs = [(0, 1), (1, 2), (2, 0), (1, 1)]
    got = model.match_pairs(inputs, pairs, max_batch=2)
    outs = [model.match(inputs[i], inputs[j]) for i, j in pairs]
    ref = torch.cat([w for w, _ in outs]), torch.cat([c for _, c in outs])
    assert got[0].shape == ref[0].shape == (4, 168, 336, 4)
    assert _err(got, ref) <= TOL


def test_match_pairs_on_batch(weights, images):
    model = _model(weights, "fp32", symmetric=True, upsample_preds=True)
    ims, his = images
    full = model.match_pairs(ims, PAIRS, his, max_batch=3)
    seen = []
    ret = model.match_pairs(ims, torch.tensor(PAIRS), his, max_batch=3, on_batch=lambda k, w, c: seen.append((k, w.clone(), c.clone())))
    assert ret is None
    assert [k for k, _, _ in seen] == list(range(0, len(PAIRS), 3)) and all(w.shape[0] <= 3 for _, w, _ in seen)
    assert torch.equal(torch.cat([w for _, w, _ in seen]), full[0]) and torch.equal(torch.cat([c for _, _, c in seen]), full[1])


def test_match_pairs_graph_replay_and_free_buffers(weights):
    model = _model(weights, "fp32", symmetric=True, upsample_preds=True)
    eager = _model(weights, "fp32", symmetric=True, upsample_preds=True)
    eager.use_cuda_graph = False
    calls = [(seed, pairs) for seed, pairs in ((11, PAIRS), (12, [(4, 0), (1, 2), (3, 3), (0, 4), (2, 1)]), (13, PAIRS[::-1]))]
    for k, (seed, pairs) in enumerate(calls):
        A, B, Ah, Bh = synthetic.make_pair(3, 112, 168, seed=seed)
        ims, his = torch.cat((A, B))[:5].cuda(), torch.cat((Ah, Bh))[:5].cuda()
        replays0 = sum(e["calls"] > 2 for e in model._pair_graphs.values())
        got = model.match_pairs(ims, pairs, his, max_batch=2)
        if k == 2:
            assert all(e["graph"] is not None for e in model._pair_graphs.values())
            assert sum(e["calls"] > 2 for e in model._pair_graphs.values()) > replays0      # this call replayed
        assert _err(got, eager.match_pairs(ims, pairs, his, max_batch=2)) <= TOL
    model.engine.free_buffers()
    gen = model.engine.generation
    got = model.match_pairs(ims, pairs, his, max_batch=2)
    assert model._pair_graphs and all(e["generation"] == gen for e in model._pair_graphs.values())      # recorded again
    assert _err(got, eager.match_pairs(ims, pairs, his, max_batch=2)) <= TOL


def test_match_pairs_errors(weights, images):
    model = _model(weights, "fp32", symmetric=True, upsample_preds=True)
    ims, his = images
    with pytest.raises(IndexError):
        model.match_pairs(ims, [(0, 5)], his)
    with pytest.raises(ValueError):
        model.match_pairs(ims, torch.zeros(2, 3, dtype=torch.long), his)
    with pytest.raises(ValueError):
        model.match_pairs([JPEGS[0], ims[0:1]], [(0, 1)])
    with pytest.raises(AssertionError):          # as match(): tensors with upsample_preds need their high-res partners
        model.match_pairs(ims, [(0, 1)])
    with pytest.raises(AssertionError):
        model.match(ims[0:1], ims[1:2])
    warp, cert = model.match_pairs(ims, [], his)
    assert warp.shape == (0, 168, 336, 4) and cert.shape == (0, 168, 336)
