"""CPU tests of TinyRoMa's host side: the oracle against the reference's goldens, the backbone structure walker, the strict
checkpoint check, BatchNorm folding without affine parameters, and pair sharding with caller-given input shapes."""
import os

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from conftest import load_golden
from oracle.tiny_oracle import TinyOracle
from roma_b200 import synthetic
from roma_b200.packing import fold_bn
from roma_b200.tiny import check_state_dict, walk_layers, xfeat_plan


@pytest.fixture(scope="module")
def tiny_weights():
    xf = synthetic.xfeat_standin()
    return synthetic.make_tiny_weights(0, xf), xf


def _images(gd):
    g = torch.Generator().manual_seed(int(gd["meta"][0]))
    return torch.rand(*gd["shape0"], generator=g), torch.rand(*gd["shape1"], generator=g)


def _close(a, b, tol=1e-6):
    err = np.abs(np.asarray(a) - np.asarray(b)).max()
    assert err <= tol, err


@pytest.mark.parametrize("name", ["tiny_b2", "tiny_unequal", "tiny_exact", "tiny_pil", "tiny_full"])
def test_oracle_vs_reference_golden(tiny_weights, name):
    sd, xf = tiny_weights
    gd = load_golden(name)
    orc = TinyOracle(sd, xf, exact_softmax=bool(gd["meta"][1]))
    orc.trace = {}
    if gd["meta"][3]:
        a, b = synthetic.make_pil_pair(int(gd["meta"][0]))
        A, B = (torch.from_numpy(np.array(im)).permute(2, 0, 1)[None].float().div(255) for im in (a, b))     # ToTensor
    else:
        A, B = _images(gd)
    warp, cert = orc.match(A, B)
    step = int(gd["meta"][2])
    _close(warp[:, ::step, ::step], gd["warp"])
    _close(cert[:, ::step, ::step], gd["certainty"])
    _close(orc.trace["gap"][0], gd["gap"], 1e-5)
    if name == "tiny_b2":
        st = load_golden("tiny_b2_stages")
        for key in ("x2", "feats", "pos_embed", "corresps8", "corresps4"):
            cs, ss = st[key + "__step"]
            _close(orc.trace[key][0][:, ::cs, ::ss, ::ss], st[key])


def test_walker_rejects_unsupported_layers_by_path():
    with pytest.raises(NotImplementedError, match=r"block9\.1"):
        walk_layers(nn.Sequential(nn.Conv2d(4, 4, 3, padding=1), nn.GELU()), "block9")
    with pytest.raises(NotImplementedError, match=r"b\.0 "):
        walk_layers(nn.Sequential(nn.Conv2d(4, 4, 3, padding=1, dilation=2)), "b")
    with pytest.raises(NotImplementedError, match=r"b\.0 "):
        walk_layers(nn.Sequential(nn.Conv2d(4, 4, 5, padding=2)), "b")
    with pytest.raises(NotImplementedError, match=r"b\.0 "):
        walk_layers(nn.Sequential(nn.BatchNorm2d(4)), "b")
    with pytest.raises(NotImplementedError, match=r"b\.1 "):
        walk_layers(nn.Sequential(nn.Conv2d(4, 4, 1), nn.MaxPool2d(2)), "b")
    xf = synthetic.xfeat_standin()
    xf.block3[1] = nn.Conv2d(64, 64, 3, padding=1, groups=2)
    with pytest.raises(NotImplementedError, match=r"block3\.1"):
        xfeat_plan(xf)
    ops = walk_layers(synthetic.xfeat_standin().block1, "block1")       # single-child wrappers (`.layer`) are descended
    assert [o["path"] for o in ops] == [f"block1.{i}.layer.0" for i in range(4)]
    assert all(o["relu"] and o["bn"] == o["path"][:-1] + "1" for o in ops) and [o["stride"] for o in ops] == [1, 2, 1, 2]


def test_strict_checkpoint_keys(tiny_weights):
    sd, xf = tiny_weights
    check_state_dict(sd, xf)
    missing = dict(sd)
    del missing["xfeat.0.block2.1.layer.1.running_var"]
    with pytest.raises(RuntimeError, match="missing"):
        check_state_dict(missing, xf)
    extra = dict(sd, **{"xfeat.0.heatmap_head.weight": torch.zeros(1)})
    with pytest.raises(RuntimeError, match="unexpected"):
        check_state_dict(extra, xf)
    bad = dict(sd, **{"coarse_matcher.4.bias": torch.zeros(4)})
    with pytest.raises(RuntimeError, match="size mismatch"):
        check_state_dict(bad, xf)


def test_fold_bn_without_affine_matches_batchnorm():
    g = torch.Generator().manual_seed(0)
    bn = nn.BatchNorm2d(8, affine=False).eval()
    bn.running_mean.copy_(torch.randn(8, generator=g))
    bn.running_var.copy_(torch.rand(8, generator=g) + 0.5)
    conv = nn.Conv2d(4, 8, 3, padding=1, bias=False)
    sd = {f"bn.{k}": v for k, v in bn.state_dict().items()}
    assert "bn.weight" not in sd
    w, b = fold_bn(conv.weight.detach(), torch.zeros(8), sd, "bn")
    x = torch.randn(2, 4, 7, 9, generator=g)
    with torch.no_grad():
        assert (F.conv2d(x, w, b, padding=1) - bn(conv(x))).abs().max() < 2e-5


class _FakeTiny:
    """Stands in for TinyRoMa: no configured resolution, output at the size of im_A."""
    device = torch.device("cpu")

    def match(self, a, b):
        s = a.mean(dim=(1, 2, 3)) + 2 * b.mean(dim=(1, 2, 3))
        n, _, h, w = a.shape
        return s.view(n, 1, 1, 1).expand(n, h, w, 4).contiguous(), s.view(n, 1, 1).expand(n, h, w).contiguous()


def _worker(rank, world, port, n_pairs, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from roma_b200.sharding import match_sharded
    model = _FakeTiny()
    g = torch.Generator().manual_seed(0)
    A, B = torch.randn(n_pairs, 1, 40, 36, generator=g), torch.randn(n_pairs, 3, 32, 48, generator=g)
    shapes = ((1, 40, 36), (3, 32, 48))
    if rank == 0:
        res = match_sharded(model, A, B, pair_shapes=shapes)
        ref_w, ref_c = model.match(A, B)
        q.put((torch.equal(res[0], ref_w), torch.equal(res[1], ref_c), tuple(res[0].shape)))
    else:
        assert match_sharded(model, None, None, n_pairs=n_pairs, pair_shapes=shapes) is None
    dist.barrier()
    dist.destroy_process_group()


def test_match_sharded_pair_shapes_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, 3, q)) for r in range(2)]
    for p in procs:
        p.start()
    ok_w, ok_c, shape = q.get(timeout=120)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    assert ok_w and ok_c and shape == (3, 40, 36, 4)
