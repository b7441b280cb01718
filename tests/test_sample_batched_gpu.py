"""`sample_batched` on the GPU: bit-equality with the `sample()` loop it replaces, for RoMa and TinyRoMa, in every sample mode, on
both KDE schedules, with more draws than pixels, with fewer positive certainties than draws and under any chunk budget; and the
batched kernels against their per-item calls (`kde_density` with `batch`, `weighted_sample` with `seed_stride` / `repeats`,
`sample_gather`)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from roma_b200 import cabi, roma_outdoor, sampling, synthetic  # noqa: E402
from roma_b200.packing import at  # noqa: E402

DEV = "cuda"
MODES = ["threshold_balanced", "threshold", "balanced", "plain"]


@pytest.fixture(scope="module")
def roma(weights):
    return roma_outdoor(DEV, weights=weights[0], dinov2_weights=weights[1], coarse_res=112, upsample_res=168, amp_dtype=torch.float32)


@pytest.fixture(scope="module")
def tiny():
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    return tiny_roma_v1_outdoor("cuda:0", weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)


@pytest.fixture(scope="module")
def warps():
    """Seeded smooth warps [3, 96, 256, 4] (n = 24576 >= 4 * 5000, so num = 5000 runs the symmetric 16-split KDE) with a certainty
    map that is high in some regions, low in others and zero on a lattice."""
    g = torch.Generator().manual_seed(3)
    B, H, W = 3, 96, 256
    ys, xs = torch.linspace(-1 + 1 / H, 1 - 1 / H, H), torch.linspace(-1 + 1 / W, 1 - 1 / W, W)
    grid = torch.stack((xs[None].expand(H, W), ys[:, None].expand(H, W)), -1)[None].expand(B, -1, -1, -1)
    shift = 0.1 * torch.sin(3 * grid + torch.rand(B, 1, 1, 2, generator=g) * 6) + 0.01 * torch.randn(B, H, W, 2, generator=g)
    warp = torch.cat((grid, (grid + shift).clamp(-1, 1)), -1).contiguous()
    cert = torch.sigmoid(4 * torch.randn(B, H, W, generator=g) + 3 * grid[..., 0])
    cert[:, ::5, ::7] = 0.0
    return warp.to(DEV), cert.to(DEV)


def _loop(model, M, C, num, R, seed):
    torch.manual_seed(seed)
    outs = [model.sample(M[b], C[b], num) for b in range(M.shape[0]) for _ in range(R)]
    k = outs[0][0].shape[0]
    return torch.stack([m for m, _ in outs]).view(M.shape[0], R, k, 4), torch.stack([c for _, c in outs]).view(M.shape[0], R, k)


def _batched(model, M, C, num, R, seed, **kw):
    torch.manual_seed(seed)
    return model.sample_batched(M, C, num, repeats=R, **kw)


def _same(a, b):
    assert a[0].shape == b[0].shape and a[1].shape == b[1].shape, (a[0].shape, b[0].shape)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.fixture(params=["roma", "tiny"])
def model(request, roma, tiny):
    m = roma if request.param == "roma" else tiny
    mode = m.sample_mode
    yield m
    m.sample_mode = mode


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("B,R", [(1, 1), (1, 2), (3, 1), (3, 2)])
@pytest.mark.parametrize("num", [500, 5000])
def test_batched_equals_sample_loop(model, warps, mode, B, R, num):
    """num = 500: k1 <= 2000 < 8192, one-pass KDE; num = 5000: k1 = 20000, symmetric 16-split KDE (balanced modes)."""
    model.sample_mode = mode
    M, C = warps[0][:B], warps[1][:B]
    for seed in (0, 1):
        ref = _loop(model, M, C, num, R, seed)
        got = _batched(model, M, C, num, R, seed)
        _same(got, ref)
    k = min(num, min((4 if "balanced" in mode else 1) * num, M[0].numel() // 4))
    assert got[0].shape == (B, R, k, 4)
    assert B * R == 1 or not torch.equal(got[0][0, 0], got[0][-1, -1])         # items draw different samples


def test_single_item_is_sample(model, warps):
    """B = R = 1 is `sample()` itself, graph replays included."""
    for seed in range(4):
        _same(_batched(model, warps[0][:1], warps[1][:1], 500, 1, seed), _loop(model, warps[0][:1], warps[1][:1], 500, 1, seed))


@pytest.mark.parametrize("mode", MODES)
def test_more_draws_than_pixels(model, mode):
    model.sample_mode = mode
    g = torch.Generator().manual_seed(5)
    M = (torch.rand(2, 8, 12, 4, generator=g) * 2 - 1).to(DEV)
    C = torch.rand(2, 8, 12, generator=g).to(DEV)
    got = _batched(model, M, C, 500, 2, 11)
    _same(got, _loop(model, M, C, 500, 2, 11))
    assert got[0].shape == (2, 2, 96, 4)


@pytest.mark.parametrize("mode", MODES)
def test_fewer_positive_certainties_than_draws(model, warps, mode):
    """k1 = 2000 (balanced) or 500 draws from maps with 300 positive entries: the zero-weight pixels fill up the draw by index."""
    model.sample_mode = mode
    M = warps[0][:2]
    C = torch.zeros_like(warps[1][:2])
    C.view(2, -1)[:, 1000:1300] = warps[1][:2].reshape(2, -1)[:, 1000:1300] + 0.01
    _same(_batched(model, M, C, 500, 2, 13), _loop(model, M, C, 500, 2, 13))


@pytest.mark.parametrize("num", [500, 5000])
def test_chunk_budget_does_not_change_bits(model, warps, num):
    M, C = warps
    ref = _batched(model, M, C, num, 2, 17)
    for budget in (1, 2 * 2 * sampling._item_bytes(M[0].numel() // 4, num, "balanced" in model.sample_mode)):   # 1 pair, then 2 + 1
        _same(_batched(model, M, C, num, 2, 17, chunk_bytes=budget), ref)


def test_launches_do_not_grow_with_the_batch(model, warps):
    counts = []
    for B, R in ((2, 1), (3, 2), (3, 5)):
        n0 = cabi.kernel_launches()
        _batched(model, warps[0][:B], warps[1][:B], 500, R, 0)
        torch.cuda.synchronize()
        counts.append(cabi.kernel_launches() - n0)
    assert counts[0] == counts[1] == counts[2], counts


def test_roma_multinomial_route_is_the_loop(roma, warps):
    roma.device_sampler = False
    try:
        _same(_batched(roma, warps[0][:2], warps[1][:2], 300, 2, 23), _loop(roma, warps[0][:2], warps[1][:2], 300, 2, 23))
    finally:
        roma.device_sampler = True


# ----------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("n", [3000, 9000])
@pytest.mark.parametrize("half,symmetric", [(True, True), (True, False), (False, False)])
def test_kde_batch_equals_single_calls(n, half, symmetric):
    """n = 3000: one pass; n = 9000: 16 j-splits, the symmetric schedule in half mode with `symmetric`."""
    g = torch.Generator().manual_seed(n)
    x = ((torch.rand(3, n, 4, generator=g) * 2 - 1) * 0.7).to(DEV)
    got = sampling.kde(x, 0.1, half, symmetric)
    for b in range(3):
        assert torch.equal(got[b], sampling.kde(x[b], 0.1, half, symmetric)), b


def _draw_args(items, n, k):
    return dict(out_idx=torch.full((items, k), -1, dtype=torch.int32, device=DEV), out_weights=torch.zeros(items, k, device=DEV),
                keys=torch.empty(items * n, device=DEV), scratch=torch.empty(items * 2056, dtype=torch.int32, device=DEV))


@pytest.mark.parametrize("transform", [cabi.SAMPLE_IDENTITY, cabi.SAMPLE_THRESHOLD])
def test_weighted_sample_seed_stride_and_repeats(transform):
    """Item i of a batched call (seed row i, map i // R) draws exactly what a batch-1 call on map i // R with seed row i draws."""
    P, R, n, k = 3, 2, 20000, 700
    g = torch.Generator().manual_seed(0)
    vals = torch.rand(P, n, generator=g)
    vals[:, ::9] = 0.0
    vals = vals.to(DEV)
    seeds = torch.randint(0, 2 ** 62, (P * R, 2), generator=g, dtype=torch.int64).to(DEV)
    for col in (0, 1):
        a = _draw_args(P * R, n, k)
        cabi.call("romab200_weighted_sample", "rb_sample_args", values=vals, n=n, k=k, batch=P * R, stride=n, seed=0, seed_dev=at(seeds, col),
                  seed_stride=2, repeats=R, transform=transform, param=0.05, **a)
        for i in range(P * R):
            s = _draw_args(1, n, k)
            cabi.call("romab200_weighted_sample", "rb_sample_args", values=vals[i // R], n=n, k=k, batch=1, stride=n, seed=0,
                      seed_dev=at(seeds, 2 * i + col), transform=transform, param=0.05, **s)
            order, ref_order = a["out_idx"][i].sort(), s["out_idx"][0].sort()
            assert torch.equal(order.values, ref_order.values), i
            assert torch.equal(a["out_weights"][i][order.indices], s["out_weights"][0][ref_order.indices]), i
        assert not torch.equal(a["out_idx"][0].sort().values, a["out_idx"][1].sort().values)     # repeats of a pair draw apart


@pytest.mark.parametrize("threshold,R", [(0, 1), (1, 1), (1, 3)])
def test_sample_gather(threshold, R):
    P, n, k = 2, 5000, 800
    g = torch.Generator().manual_seed(1)
    m = torch.randn(P, n, 4, generator=g).to(DEV)
    c = torch.rand(P, n, generator=g).to(DEV)
    idx = torch.stack([torch.randperm(n, generator=g)[:k].sort().values for _ in range(P * R)]).to(DEV, torch.int32)
    om, oc = torch.empty(P * R, k, 4, device=DEV), torch.empty(P * R, k, device=DEV)
    cabi.call("romab200_sample_gather", "rb_sample_gather_args", matches=m, certainty=c, n=n, idx=idx, items=P * R, k=k, repeats=R,
              threshold=threshold, thresh=0.3, out_matches=om, out_certainty=oc)
    for i in range(P * R):
        sel = idx[i].long()
        assert torch.equal(om[i], m[i // R][sel])
        ci = c[i // R][sel]
        assert torch.equal(oc[i], torch.where(ci > 0.3, torch.ones((), device=DEV), ci) if threshold else ci)
