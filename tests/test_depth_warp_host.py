"""CPU tests of the depth-based warps: the torch oracle against the reference's goldens (tests/golden/make_golden_depth_warp.py),
the synthetic scenes, the argument handling of the public functions and the generated C structs."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import depth_warp as oracle
from roma_b200 import cabi, depth_warp, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(ours, gold, rtol=1e-12):
    ours, gold = np.asarray(ours), np.asarray(gold)
    assert ours.shape == gold.shape
    assert np.array_equal(np.isnan(ours), np.isnan(gold)) and np.array_equal(np.isinf(ours), np.isinf(gold))
    fin = np.isfinite(gold)
    assert np.all(np.abs(ours[fin] - gold[fin]) <= rtol * np.maximum(1.0, np.abs(gold[fin])))


@pytest.fixture(scope="module")
def gold():
    gd = load_golden("depth_warp")
    return gd, [torch.from_numpy(gd[k]) for k in ("depth0", "depth1", "T", "K0", "K1")]


@pytest.mark.parametrize("mode", ["bilinear", "nearest"])
def test_oracle_matches_reference_golden(gold, mode):
    gd, views = gold
    valid, warped = oracle.warp_kpts(torch.from_numpy(gd["kpts"]), *views, depth_interpolation_mode=mode)
    assert np.array_equal(valid.numpy(), gd[f"valid_{mode}"])
    _same(warped.numpy(), gd[f"warped_{mode}"])
    for tag, hw in (("", {}), ("_hw", dict(H=30, W=44))):
        x2, prob = oracle.get_gt_warp(*views, depth_interpolation_mode=mode, **hw)
        assert prob.dtype == torch.float32 and np.array_equal(prob.numpy(), gd[f"prob{tag}_{mode}"])
        _same(x2.numpy(), gd[f"x2{tag}_{mode}"])


def test_golden_covers_the_hard_points(gold):
    gd, _ = gold
    w = gd["warped_bilinear"]
    assert 0.2 < gd["valid_bilinear"].mean() < 0.8
    assert (np.abs(gd["kpts"]) > 1).any() and (np.abs(w[np.isfinite(w)]) > 1).any()


def test_oracle_metric_is_the_harness_statement():
    """`gd[prob == 1]`, its mean and the PCKs, written out as the harness has them, on a noisy ground-truth warp."""
    views = synthetic.depth_scene(3, 2, 40, 56)
    x2, prob = oracle.get_gt_warp(*views)
    g = torch.Generator().manual_seed(0)
    xs, ys = torch.linspace(-1 + 1 / 56, 1 - 1 / 56, 56), torch.linspace(-1 + 1 / 40, 1 - 1 / 40, 40)
    grid = torch.stack((xs[None].expand(40, 56), ys[:, None].expand(40, 56)), -1)[None].expand(2, -1, -1, -1)
    dm = torch.cat((grid, x2.float() + 0.05 * torch.randn(2, 40, 56, 2, generator=g)), dim=-1)
    out = oracle.dense_geometric_dist(*views, dm)
    assert torch.equal(out["prob"], prob) and 0.2 < prob.mean() < 0.9
    px = lambda p: torch.stack((56 * (p[..., 0] + 1) / 2, 40 * (p[..., 1] + 1) / 2), -1)      # noqa: E731
    vec = (px(dm[..., 2:]) - px(x2)).norm(dim=-1)[prob == 1]
    assert torch.equal(out["gd"][prob == 1], vec) and torch.isnan(out["gd"][prob != 1]).all()
    assert out["epe"] == vec.mean() and 0.1 < out["epe"] < 5
    for k, t in enumerate((1.0, 3.0, 5.0)):
        assert out["pck"][k] == (vec < t).float().mean()
        assert out["pair_count"][:, k + 1].sum() == (vec < t).sum()
    assert out["pair_count"][:, 0].sum() == vec.numel()
    assert abs(out["pair_sum"].sum() - vec.sum()) <= 1e-12 * vec.sum()


def _classes(views, pts=None):
    """Fractions of points with zero depth, then not covisible, then depth-inconsistent, then valid."""
    d = {}
    if pts is None:
        _, prob = oracle.get_gt_warp(*views, details=d)
        valid = prob.flatten(1) == 1
    else:
        valid, _ = oracle.warp_kpts(pts, *views, details=d)
    (h1, w1) = views[1].shape[1:]
    zero = d["d0"] == 0
    outside = ~zero & ~((d["u"] > 0) & (d["u"] < w1 - 1) & (d["v"] > 0) & (d["v"] < h1 - 1))
    inconsistent = ~zero & ~outside & ~valid
    return [m.double().mean().item() for m in (zero, outside, inconsistent, valid)]


@pytest.mark.parametrize("seed, shape", [(0, (2, 96, 128)), (5, (2, 48, 64, 60, 80)), (21, (3, 60, 80, 48, 64))])
def test_depth_scene_is_seeded_and_fills_every_class(seed, shape):
    a, b = synthetic.depth_scene(seed, *shape), synthetic.depth_scene(seed, *shape)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[0], synthetic.depth_scene(seed + 1, *shape)[0])
    B, h0, w0 = shape[:3]
    h1, w1 = shape[3:] or (h0, w0)
    assert a[0].shape == (B, h0, w0) and a[1].shape == (B, h1, w1) and a[0].dtype == a[1].dtype == torch.float32
    assert a[2].shape == (B, 4, 4) and a[3].shape == a[4].shape == (B, 3, 3) and a[2].dtype == a[3].dtype == torch.float64
    fr = _classes(a)
    assert min(fr) >= 0.05 and abs(sum(fr) - 1) < 1e-12, fr


def test_depth_scene_views_are_consistent():
    """Away from holes and depth edges the two exact depth maps agree to interpolation error: most covisible points are valid at a
    threshold 50 times tighter than the default."""
    views = synthetic.depth_scene(2, 2, 96, 128)
    d = {}
    oracle.get_gt_warp(*views, details=d)
    assert (d["rel"] < 1e-3).double().mean() > 0.3


# ---- argument handling (everything below raises before a device is needed) ------------------------------------------------------------
def _views(B=2):
    return list(synthetic.depth_scene(1, B, 12, 16))


def test_refused_options_and_modes():
    v = _views()
    k = torch.zeros(2, 5, 2)
    with pytest.raises(NotImplementedError, match="smooth_mask"):
        depth_warp.warp_kpts(k, *v, smooth_mask=0.1)
    with pytest.raises(NotImplementedError, match="return_relative_depth_error"):
        depth_warp.warp_kpts(k, *v, return_relative_depth_error=True)
    for mode in ("combined", "nearest-exact", "linear"):
        # what the reference does with these: F.grid_sample refuses the mode ("combined" runs "nearest-exact")
        with pytest.raises(ValueError, match="expected mode"):
            torch.nn.functional.grid_sample(v[0][:, None], k[:, :, None], mode="nearest-exact" if mode == "combined" else mode, align_corners=False)
        with pytest.raises(ValueError, match="expected mode"):
            depth_warp.warp_kpts(k, *v, depth_interpolation_mode=mode)
        with pytest.raises(ValueError, match="expected mode"):
            depth_warp.get_gt_warp(*v, depth_interpolation_mode=mode)
    with pytest.raises(NotImplementedError, match="bicubic"):
        depth_warp.get_gt_warp(*v, depth_interpolation_mode="bicubic")


def test_shape_and_dtype_errors():
    v = _views()
    k, dm = torch.zeros(2, 5, 2), torch.zeros(2, 12, 16, 4)
    bad_shape = [
        lambda: depth_warp.warp_kpts(torch.zeros(2, 5, 3), *v),
        lambda: depth_warp.warp_kpts(torch.zeros(3, 5, 2), *v),
        lambda: depth_warp.warp_kpts(k, v[0][0], *v[1:]),
        lambda: depth_warp.warp_kpts(k, v[0], v[1][:1], *v[2:]),
        lambda: depth_warp.warp_kpts(k, v[0], v[1], v[2][:, :2], v[3], v[4]),
        lambda: depth_warp.warp_kpts(k, v[0], v[1], v[2], v[3][:, :2], v[4]),
        lambda: depth_warp.get_gt_warp(*v[:4], v[4][0]),
        lambda: depth_warp.get_gt_warp(*v, H=10),
        lambda: depth_warp.dense_geometric_dist(*v, dm[..., :3]),
        lambda: depth_warp.dense_geometric_dist(*v, dm[0]),
        lambda: depth_warp.dense_geometric_dist(*v, dm[:1]),
    ]
    for f in bad_shape:
        with pytest.raises(ValueError):
            f()
    bad_type = [
        lambda: depth_warp.warp_kpts(k.half(), *v),
        lambda: depth_warp.warp_kpts(k.numpy(), *v),
        lambda: depth_warp.warp_kpts(k, v[0].half(), *v[1:]),
        lambda: depth_warp.warp_kpts(k, v[0], v[1].long(), *v[2:]),
        lambda: depth_warp.get_gt_warp(v[0], v[1], v[2].long(), v[3], v[4]),
        lambda: depth_warp.dense_geometric_dist(*v, dm.double()),
        lambda: depth_warp.dense_geometric_dist(*v, None),
    ]
    for f in bad_type:
        with pytest.raises(TypeError):
            f()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the error raised without a CUDA device")
def test_no_device_is_an_error_not_a_fallback():
    v = _views()
    for f in (lambda: depth_warp.warp_kpts(torch.zeros(2, 5, 2), *v), lambda: depth_warp.get_gt_warp(*v),
              lambda: depth_warp.dense_geometric_dist(*v, torch.zeros(2, 12, 16, 4))):
        with pytest.raises(RuntimeError, match=r"runs on the GPU only \(there is no CPU fallback\)"):
            f()


def test_lazy_exports():
    import roma_b200
    assert roma_b200.warp_kpts is depth_warp.warp_kpts and roma_b200.get_gt_warp is depth_warp.get_gt_warp
    assert roma_b200.dense_geometric_dist is depth_warp.dense_geometric_dist


def test_result_type_unpacks_like_the_harness():
    r = depth_warp.DenseGeometricDist(*range(8))
    gd, p1, p3, p5, prob = r
    assert (gd, p1, p3, p5, prob) == (0, 1, 2, 3, 4) == (r.gd, r.pck_1, r.pck_3, r.pck_5, r.prob)
    assert (r.epe, r.pair_sum, r.pair_count) == (5, 6, 7) and len(r) == 5


# ---- the C ABI ------------------------------------------------------------------------------------------------------------------------
SHARED = ["depth0", "depth1", "depth_dtype", "h0", "w0", "h1", "w1", "T", "T_rows", "K0", "K1", "batch", "rel_threshold"]
FIELDS = {
    "rb_warp_kpts_args": SHARED + ["mode", "kpts", "kpts_dtype", "L", "warped", "valid"],
    "rb_gt_warp_args": SHARED + ["mode", "grid_x", "grid_y", "H", "W", "x2", "prob"],
    "rb_dense_geometric_dist_args": SHARED + ["dense_matches", "dm_sb", "dm_sy", "dm_sx", "dm_sc", "H", "W", "gd", "prob", "partial_sum",
                                               "partial_cnt", "pair_sum", "pair_cnt", "pck", "epe"],
}


def test_structs_have_the_fields_the_python_side_passes():
    for struct, fields in FIELDS.items():
        types = dict(cabi.STRUCT_FIELDS[struct])
        assert set(types) == set(fields), struct
        assert types["rel_threshold"] is ctypes.c_double and types["depth0"] is ctypes.c_void_p and types["depth_dtype"] is ctypes.c_int32
        assert set(cabi._FIELD_DTYPES[struct]) == {f for f, t in types.items() if t is ctypes.c_void_p}, struct
    assert dict(cabi.STRUCT_FIELDS["rb_warp_kpts_args"])["L"] is ctypes.c_int64
    assert all(dict(cabi.STRUCT_FIELDS["rb_dense_geometric_dist_args"])[f] is ctypes.c_int64 for f in ("dm_sb", "dm_sy", "dm_sx", "dm_sc"))
    assert "MAX_CTAS 512" in open(cabi.HEADER).read() and depth_warp.MAX_CTAS == 512
    assert cabi.RB_F64 == 4 and "RB_F64 = 4" in open(cabi.HEADER).read()
    for fn in ("romab200_warp_kpts", "romab200_gt_warp", "romab200_dense_geometric_dist"):
        assert fn in cabi.FUNCTIONS


_CHILD = r"""
import ctypes, json, sys
from roma_b200 import cabi
lib = cabi.load_library()
out = []
for fn, struct, fields in json.load(sys.stdin):
    args = cabi.STRUCTS[struct]()
    for k, v in fields.items():
        setattr(args, k, v)
    rc = getattr(lib, "romab200_" + fn)(ctypes.byref(args), None)
    out.append([rc, lib.romab200_last_error().decode()])
print(json.dumps(out))
"""


def test_entry_points_refuse_bad_codes_before_any_cuda_call():
    """The float64 code is accepted only where a kernel exists for it: the three new entry points refuse any other depth or point
    code, an unknown mode and a bad shape, and an older entry point refuses the float64 code.  Run without a visible device."""
    addr = 1 << 20
    base = dict(depth0=addr, depth1=addr, T=addr, K0=addr, K1=addr, h0=4, w0=4, h1=4, w1=4, T_rows=4, batch=1, depth_dtype=cabi.RB_F64)
    kp = dict(base, kpts=addr, warped=addr, valid=addr, L=3, kpts_dtype=cabi.RB_F32)
    gt = dict(base, grid_x=addr, grid_y=addr, x2=addr, prob=addr, H=4, W=4)
    dn = dict(base, dense_matches=addr, gd=addr, prob=addr, partial_sum=addr, partial_cnt=addr, pair_sum=addr, pair_cnt=addr, pck=addr, epe=addr,
              H=4, W=4)
    calls = [
        ("warp_kpts", "rb_warp_kpts_args", dict(kp, depth_dtype=cabi.RB_F16), "warp_kpts: unsupported dtype 1"),
        ("warp_kpts", "rb_warp_kpts_args", dict(kp, kpts_dtype=cabi.RB_F16S), "warp_kpts: unsupported dtype 3"),
        ("warp_kpts", "rb_warp_kpts_args", dict(kp, mode=2), "warp_kpts: interpolation mode 2 unsupported (0 bilinear, 1 nearest)"),
        ("warp_kpts", "rb_warp_kpts_args", dict(kp, T_rows=2), "warp_kpts: T must be [batch, 3 or 4, 4] (got 2 rows)"),
        ("gt_warp", "rb_gt_warp_args", dict(gt, depth_dtype=7), "gt_warp: unsupported dtype 7"),
        ("gt_warp", "rb_gt_warp_args", dict(gt, batch=0), "gt_warp: batch 0 outside 1 .. 65535"),
        ("dense_geometric_dist", "rb_dense_geometric_dist_args", dict(dn, depth_dtype=cabi.RB_BF16), "dense_geometric_dist: unsupported dtype 2"),
        ("dense_geometric_dist", "rb_dense_geometric_dist_args", dict(dn, pck=0), "dense_geometric_dist: null argument"),
        ("row_norms", "rb_rownorm_args", dict(rows=4, cols=8, ldx=8, dtype=cabi.RB_F64), "row_norms: unsupported dtype 4"),
        ("copy2d", "rb_copy2d_args", dict(rows=4, cols=8, lds=8, ldd=8, dtype_src=cabi.RB_F32, dtype_dst=cabi.RB_F64), "copy2d: unsupported dtype 4"),
    ]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, "-c", _CHILD], input=json.dumps([c[:3] for c in calls]), capture_output=True, text=True, cwd=ROOT,
                         env=env, timeout=600)
    assert res.returncode == 0, res.stderr
    for (fn, _, _, want), (rc, msg) in zip(calls, json.loads(res.stdout.strip().splitlines()[-1])):
        assert rc != 0 and msg == want, (fn, rc, msg)
