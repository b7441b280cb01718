"""TinyRoMa on the GPU: every new kernel against PyTorch fp64 / the CPU oracle, the backbone against the XFeat module itself,
and match() end to end against the reference's goldens (tests/golden/make_golden_tiny.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from conftest import load_golden  # noqa: E402
from oracle.tiny_oracle import TinyOracle  # noqa: E402
from roma_b200 import synthetic  # noqa: E402
from roma_b200.cabi import call  # noqa: E402

TOL = 1e-4


@pytest.fixture(scope="module")
def tiny():
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    sd = synthetic.make_tiny_weights(0, xf)
    return tiny_roma_v1_outdoor("cuda:0", weights=sd, xfeat=xf), sd, xf


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("k,stride", [(1, 1), (1, 2), (3, 1), (3, 2)])
@pytest.mark.parametrize("cin,cout", [(1, 4), (4, 8), (24, 24), (64, 128), (128, 64), (130, 256), (50, 3)])
def test_tiny_conv_vs_conv2d(k, stride, cin, cout):
    from roma_b200.tiny import pack_conv
    g = torch.Generator().manual_seed(cin * 1000 + cout + 10 * k + stride)
    x = torch.randn(2, cin, 13, 17, generator=g)
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    b = torch.randn(cout, generator=g)
    scale, res = torch.rand(cout, generator=g) + 0.5, None
    L = pack_conv({"c.weight": w, "c.bias": b}, "c", dict(k=k, stride=stride, bias=True, bn=None, relu=True, path="c"), "cuda")
    ref = F.relu(F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=k // 2)) * scale.double()[:, None, None]
    res = torch.randn(ref.shape, generator=g)
    ref = ref + res.double()
    ho, wo = ref.shape[-2:]
    out = torch.empty(2, ho, wo, cout, device="cuda")
    call("romab200_tiny_conv", "rb_tiny_conv_args", **{"in": _nhwc(x).cuda()}, out=out, weight=L["w"], bias=L["b"], col_scale=scale.cuda(),
         R=_nhwc(res.float()).cuda(), ldi=cin, ldo=cout, ldw=L["w"].shape[1], ldr=cout, batch=2, hi=13, wi=17, ho=ho, wo=wo, cin=cin, cout=cout,
         ksize=k, stride=stride, relu=1)
    err = (out.cpu().double() - _nhwc(ref)).abs().max().item()
    assert err < 1e-5 * max(1.0, ref.abs().max().item()), err


@pytest.mark.parametrize("variant", ["standin", "narrow"])
def test_backbone_vs_xfeat_module(variant):
    from roma_b200.tiny import TinyRoMa
    xf = synthetic.xfeat_standin() if variant == "standin" else synthetic.xfeat_standin(widths=(8, 16, 24, 32, 48), fusion_extra=False)
    sd = synthetic.make_tiny_weights(1, xf)
    orc = TinyOracle(sd, xf)
    model = TinyRoMa(xf, sd, "cuda:0")       # "narrow": 32-d features, which only the backbone can run (the heads take 64)
    g = torch.Generator().manual_seed(5)
    img = torch.rand(2, 3, 96, 128, generator=g)
    with torch.no_grad():
        rx2, rf = orc.backbone(img)
    x2, feats = model._backbone(img.cuda(), "t")
    for ours, ref in ((x2, rx2), (feats, rf)):
        err = (ours.cpu() - _nhwc(ref)).abs().max().item()
        assert err < 1e-4 * max(1.0, ref.abs().max().item()), err


def _pos_embed(f0, f1, exact):
    B, h0, w0, c = f0.shape
    h1, w1 = f1.shape[1:3]
    state = torch.empty(B, h0, w0, 3, device="cuda")
    lin = lambda lo, n: torch.linspace(-1 + lo, 1 - lo, n).cuda()
    call("romab200_tiny_pos_embed", "rb_tiny_pos_embed_args", f0=f0.cuda().contiguous(), f1=f1.cuda().contiguous(), state=state, batch=B,
         h0=h0, w0=w0, h1=h1, w1=w1, c=c, scale=8.0, exact=int(exact), grid_x=lin(1 / w1, w1), grid_y=lin(1 / h1, h1),
         grid_lr_x=lin(4 / w1, w1 // 4), grid_lr_y=lin(4 / h1, h1 // 4))
    return state.cpu()


@pytest.mark.parametrize("case", ["random", "unequal", "small_best", "ties", "exact"])
def test_pos_embed_vs_oracle(case):
    g = torch.Generator().manual_seed(11)
    h0, w0, h1, w1 = (12, 20, 16, 12) if case == "unequal" else (16, 20, 16, 20)
    f0 = torch.randn(2, 64, h0, w0, generator=g)
    f1 = torch.randn(2, 64, h1, w1, generator=g)
    if case == "small_best":
        # every pixel of image 0 matches pixel 5 of image 1 best, with scores of the size of that index: the extra logit (5.0)
        # mixes with the sub-sampled softmax instead of taking all the weight
        u = torch.ones(64) / 8
        f1 = 0.05 * f1
        f1[:, :, 0, :6] = (8 * u[:, None] * torch.linspace(1, 2, 6))[None]
        f0 = u[None, :, None, None] * (2 + 2 * torch.rand(2, 1, h0, w0, generator=g)) + 0.1 * f0
    if case == "ties":
        f1[:, :, 5, 7] = f1[:, :, 2, 3]                 # identical vectors: identical scores, the first index must win
        f0[:, :, 3, 4] = f1[:, :, 2, 3] * 3
    pos, best, gap = TinyOracle.pos_embed(f0.double(), f1.double(), exact=case == "exact")
    ours = _pos_embed(_nhwc(f0), _nhwc(f1), case == "exact")
    assert torch.all(ours[..., 2] == 0)
    if case == "small_best":
        assert best.max().item() == 5 and (ours[..., 0] - torch.linspace(-1 + 1 / w1, 1 - 1 / w1, w1)[5]).abs().min() > 1e-3
    if case == "ties":
        assert best[0, 3, 4].item() == 2 * w1 + 3 and ours[0, 3, 4, :2].tolist() != [0.0, 0.0]
    keep = gap > 1e-3
    err = (ours[..., :2] - _nhwc(pos).float())[keep].abs().max().item()
    assert err < 1e-5, err
    if case == "ties":
        lin = torch.linspace(-1 + 1 / w1, 1 - 1 / w1, w1)
        linv = torch.linspace(-1 + 1 / h1, 1 - 1 / h1, h1)
        assert abs(ours[0, 3, 4, 0].item() - lin[3].item()) < 1e-6 and abs(ours[0, 3, 4, 1].item() - linv[2].item()) < 1e-6


def test_warp_concat_vs_grid_sample():
    g = torch.Generator().manual_seed(3)
    f0, f1 = torch.randn(2, 24, 10, 14, generator=g), torch.randn(2, 24, 8, 12, generator=g)
    flow = torch.rand(2, 2, 10, 14, generator=g) * 2.4 - 1.2            # partly outside [-1, 1]: zero padding
    state = torch.cat((flow, torch.randn(2, 1, 10, 14, generator=g)), 1)
    ref = torch.cat((f0, F.grid_sample(f1, flow.permute(0, 2, 3, 1), mode="bilinear", align_corners=False), flow), 1)
    out = torch.zeros(2, 10, 14, 52, device="cuda")
    call("romab200_tiny_warp_concat", "rb_tiny_warp_concat_args", f0=_nhwc(f0).cuda(), f1=_nhwc(f1).cuda(), state=_nhwc(state).cuda(), out=out,
         ldf0=24, ldf1=24, lds=3, ldo=52, batch=2, h0=10, w0=14, h1=8, w1=12, c=24)
    assert (out[..., :50].cpu() - _nhwc(ref)).abs().max().item() < 1e-5
    assert torch.all(out[..., 50:] == 0)


def _check(name, warp, cert):
    gd = load_golden(name)
    step = int(gd["meta"][2])
    w, c = warp[:, ::step, ::step].cpu().numpy(), cert[:, ::step, ::step].cpu().numpy()
    ew, ec = np.abs(w - gd["warp"]).max(), np.abs(c - gd["certainty"]).max()
    print(f"{name}: warp max-abs {ew:.2e}, certainty max-abs {ec:.2e}")
    assert ew <= TOL and ec <= TOL, (ew, ec)


def _images(gd):
    g = torch.Generator().manual_seed(int(gd["meta"][0]))
    return torch.rand(*gd["shape0"], generator=g), torch.rand(*gd["shape1"], generator=g)


@pytest.mark.parametrize("name", ["tiny_b2", "tiny_unequal", "tiny_exact", "tiny_full"])
def test_match_vs_reference_golden(tiny, name):
    model = tiny[0]
    gd = load_golden(name)
    model.exact_softmax = bool(gd["meta"][1])
    try:
        a, b = _images(gd)
        warp, cert = model.match(a.cuda(), b.cuda())
    finally:
        model.exact_softmax = False
    assert warp.shape == (a.shape[0], a.shape[2], a.shape[3], 4) and cert.shape == warp.shape[:3]
    _check(name, warp, cert)


def test_match_pil_unbatched_and_stages(tiny):
    model, sd, xf = tiny
    a, b = synthetic.make_pil_pair(int(load_golden("tiny_pil")["meta"][0]))
    warp, cert = model.match(a, b)
    assert warp.shape == (a.height, a.width, 4) and cert.shape == (a.height, a.width)
    _check("tiny_pil", warp[None], cert[None])
    gd, st = load_golden("tiny_b2"), load_golden("tiny_b2_stages")
    A, B = _images(gd)
    out = model.forward({"im_A": A.cuda(), "im_B": B.cuda()})
    assert out[8]["flow"].shape == (2, 2, 32, 40) and out[4]["certainty"].shape == (2, 1, 64, 80)
    for s in (8, 4):
        ours = torch.cat((out[s]["flow"], out[s]["certainty"]), 1).cpu().numpy()
        assert np.abs(ours - st[f"corresps{s}"]).max() <= TOL


def test_match_graph_replay_bit_equal(tiny):
    model = tiny[0]
    g = torch.Generator().manual_seed(9)
    a, b = torch.rand(1, 3, 96, 128, generator=g).cuda(), torch.rand(1, 3, 96, 128, generator=g).cuda()
    outs = [model.match(a, b) for _ in range(4)]          # eager, eager + capture, replay, replay
    key = next(k for k in model._graphs if k[0] == (1, 3, 96, 128))
    assert model._graphs[key]["graph"] is not None
    model.free_buffers()                                  # drops the graphs with the buffers they point into
    outs += [model.match(a, b) for _ in range(3)]
    graph = model._graphs[key]["graph"]
    model.arena.free()                                    # the buffers alone: the graph recorded over them must not be replayed
    outs += [model.match(a, b) for _ in range(3)]
    assert model._graphs[key]["graph"] not in (None, graph)
    for w, c in outs[1:]:
        assert torch.equal(w, outs[0][0]) and torch.equal(c, outs[0][1])


def test_rejects_small_images_and_cpu(tiny):
    from roma_b200 import tiny_roma_v1_outdoor
    with pytest.raises(ValueError):
        tiny[0].match(torch.rand(1, 3, 31, 64).cuda(), torch.rand(1, 3, 64, 64).cuda())
    with pytest.raises(RuntimeError):
        tiny_roma_v1_outdoor("cpu", weights=tiny[1], xfeat=tiny[2])


def test_sample_distribution_vs_oracle_tiny(tiny):
    """The shared device sampler under TinyRoMa.sample (num=5000 default) against the oracle's two torch.multinomial draws
    around the fp16 KDE: two-sample Kolmogorov-Smirnov per coordinate and on the certainty over 20 seeds each."""
    from scipy import stats
    model, sd, xf = tiny
    gd = load_golden("tiny_b2")
    A, B = _images(gd)
    warp, cert = model.match(A[:1].cuda(), B[:1].cuda())
    warp, cert = warp[0], cert[0]
    orc = TinyOracle(sd, xf)
    ours, ref = [], []
    for seed in range(20):
        torch.manual_seed(100 + seed)
        m, c = model.sample(warp, cert, num=1000)
        assert m.shape == (1000, 4) and c.shape == (1000,)
        ours.append(torch.cat((m, c[:, None]), 1).cpu())
        torch.manual_seed(900 + seed)
        m, c = orc.sample(warp.cpu(), cert.cpu(), num=1000)
        ref.append(torch.cat((m, c[:, None].float()), 1))
    ours, ref = torch.cat(ours).numpy(), torch.cat(ref).numpy()
    rows = {tuple(r) for r in warp.reshape(-1, 4).cpu().numpy().view("uint32").tolist()}
    assert all(tuple(r) in rows for r in np.ascontiguousarray(ours[:, :4]).view("uint32").tolist())
    for j in range(5):
        p = stats.ks_2samp(ours[:, j], ref[:, j]).pvalue
        assert p > 1e-3, (j, p)
    m, c = model.sample(warp, cert)
    assert m.shape == (5000, 4)
