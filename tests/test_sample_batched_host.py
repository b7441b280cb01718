"""CPU tests of `sample_batched`: its argument rules (checked before any device work), the generated C structs of the batched
sampler fields, the shim's checks of `romab200_sample_gather` operands, and the seed layout that makes a batched draw equal the
`sample()` loop."""
import ctypes

import pytest
import torch

from roma_b200 import cabi
from roma_b200.matcher import RegressionMatcher
from roma_b200.tiny import TinyRoMa
from test_host_logic import fake


def _roma(mode="threshold_balanced"):
    return RegressionMatcher(None, sample_mode=mode)        # the CPU route of sample() never reaches the engine


def _tiny():
    m = TinyRoMa.__new__(TinyRoMa)
    m.sample_mode, m.sample_thresh, m.use_cuda_graph = "threshold_balanced", 0.05, True
    return m


def _warp(B=2, h=6, w=8):
    g = torch.Generator().manual_seed(0)
    return torch.rand(B, h, w, 4, generator=g) * 2 - 1, torch.rand(B, h, w, generator=g)


@pytest.mark.parametrize("make", [_roma, _tiny])
def test_argument_rules(make):
    model = make()
    M, C = _warp()
    for bad, why in (((M, C[:1]), "leading shape"), ((M, C[..., :4]), "leading shape"), ((M[..., :3], C), "leading shape"),
                     ((M[0, 0, 0], C[0, 0, 0]), "leading shape"), ((M[:0], C[:0]), "empty"), ((M.double(), C), "fp32")):
        with pytest.raises(ValueError, match=why):
            model.sample_batched(*bad, 10)
    for num, repeats, why in ((0, 1, "num"), (-3, 1, "num"), (2.5, 1, "num"), (10, 0, "repeats"), (10, -1, "repeats"), (10, 1.0, "repeats")):
        with pytest.raises(ValueError, match=why):
            model.sample_batched(M, C, num, repeats=repeats)


@pytest.mark.parametrize("make", [_roma, _tiny])
def test_cpu_tensors_raise_what_sample_raises(make):
    model = make()
    M, C = _warp()
    with pytest.raises(RuntimeError, match="needs CUDA tensors") as batched:
        model.sample_batched(M, C, 10, repeats=2)
    if isinstance(model, RegressionMatcher):           # TinyRoMa.sample takes the unbatched warp only
        with pytest.raises(RuntimeError) as single:
            model.sample(M[0], C[0], 10)
        assert str(single.value) == str(batched.value)


def test_roma_cpu_route_is_the_sample_loop():
    """Without the device sampler (or for CPU tensors) a non-balanced mode is the `torch.multinomial` loop of `sample()`."""
    model = _roma("threshold")
    model.device_sampler = False
    M, C = _warp(3)
    torch.manual_seed(4)
    m, c = model.sample_batched(M, C, 7, repeats=2)
    torch.manual_seed(4)
    ref = [model.sample(M[b], C[b], 7) for b in range(3) for _ in range(2)]
    assert m.shape == (3, 2, 7, 4) and c.shape == (3, 2, 7)
    assert torch.equal(m.reshape(6, 7, 4), torch.stack([x for x, _ in ref])) and torch.equal(c.reshape(6, 7), torch.stack([y for _, y in ref]))


def test_header_exposes_the_batched_sampler():
    f = dict(cabi.STRUCT_FIELDS["rb_sample_args"])
    assert [n for n, _ in cabi.STRUCT_FIELDS["rb_sample_args"][-2:]] == ["seed_stride", "repeats"]
    assert f["seed_stride"] is ctypes.c_int64 and f["repeats"] is ctypes.c_int32
    assert cabi.STRUCT_FIELDS["rb_kde_args"][-1] == ("batch", ctypes.c_int32)
    g = cabi.STRUCT_FIELDS["rb_sample_gather_args"]
    assert [n for n, _ in g] == ["matches", "certainty", "n", "idx", "items", "k", "repeats", "threshold", "thresh", "out_matches", "out_certainty"]
    assert {n for n, t in g if t is ctypes.c_void_p} == {"matches", "certainty", "idx", "out_matches", "out_certainty"}
    assert "romab200_sample_gather" in cabi.FUNCTIONS
    assert set(cabi._FIELD_DTYPES["rb_sample_gather_args"]) == {"matches", "certainty", "idx", "out_matches", "out_certainty"}


def _gather_kw(P=2, R=3, n=50, k=7):
    return dict(matches=fake(torch.zeros(P, n, 4)), certainty=fake(torch.zeros(P, n)), n=n, idx=fake(torch.zeros(P * R, k, dtype=torch.int32)),
                items=P * R, k=k, repeats=R, threshold=1, thresh=0.05, out_matches=fake(torch.zeros(P * R, k, 4)),
                out_certainty=fake(torch.zeros(P * R, k)))


def test_shim_checks_sample_gather_operands():
    kw = _gather_kw()
    cabi._validate("romab200_sample_gather", "rb_sample_gather_args", kw)
    for field, bad in (("idx", fake(torch.zeros(6, 7, dtype=torch.int64))), ("matches", fake(torch.zeros(2, 50, 4, dtype=torch.float16))),
                       ("out_certainty", fake(torch.zeros(6, 7, dtype=torch.float64)))):
        with pytest.raises(RuntimeError, match=f"`{field}` has dtype"):
            cabi._validate("romab200_sample_gather", "rb_sample_gather_args", dict(kw, **{field: bad}))
    with pytest.raises(RuntimeError, match="`certainty` holds 50 elements, the described geometry needs 100"):
        cabi._validate("romab200_sample_gather", "rb_sample_gather_args", dict(kw, certainty=fake(torch.zeros(1, 50))))
    with pytest.raises(RuntimeError, match="`out_matches` holds 164 elements, the described geometry needs 168"):
        cabi._validate("romab200_sample_gather", "rb_sample_gather_args", dict(kw, out_matches=fake(torch.zeros(164))))
    with pytest.raises(RuntimeError, match="expected the current CUDA device"):
        cabi.call("romab200_sample_gather", "rb_sample_gather_args", **dict(kw, idx=torch.zeros(6, 7, dtype=torch.int32)))
    with pytest.raises(TypeError, match="pointer field `idx`"):
        cabi.call("romab200_sample_gather", "rb_sample_gather_args", **dict(kw, idx=kw["idx"].data_ptr()))


def test_shim_checks_batched_sample_extents():
    """`repeats` items per map read (batch - 1) // repeats + 1 maps; `seed_stride` spaces the items' seeds."""
    kw = dict(values=fake(torch.zeros(2, 100)), n=100, k=10, batch=6, stride=100, repeats=3, seed_dev=fake(torch.zeros(11, dtype=torch.int64)),
              seed_stride=2, out_idx=fake(torch.zeros(6, 10, dtype=torch.int32)), keys=fake(torch.zeros(600)),
              scratch=fake(torch.zeros(6 * 2056, dtype=torch.int32)))
    cabi._validate("romab200_weighted_sample", "rb_sample_args", kw)
    with pytest.raises(RuntimeError, match="`values` holds 200 elements, the described geometry needs 300"):
        cabi._validate("romab200_weighted_sample", "rb_sample_args", dict(kw, repeats=2))
    with pytest.raises(RuntimeError, match="`seed_dev` holds 11 elements, the described geometry needs 16"):
        cabi._validate("romab200_weighted_sample", "rb_sample_args", dict(kw, seed_stride=3))


@pytest.mark.parametrize("items", [1, 2, 7, 64])
def test_seed_rows_equal_successive_sample_seeds(items):
    """Row i of one CPU randint of [items, 2] holds the two seeds the i-th of `items` successive sample() calls draws."""
    for seed in (0, 12345):
        torch.manual_seed(seed)
        rows = torch.randint(0, 2 ** 62, (items, 2), dtype=torch.int64)
        torch.manual_seed(seed)
        calls = torch.stack([torch.randint(0, 2 ** 62, (1, 2), dtype=torch.int64)[0] for _ in range(items)])
        torch.manual_seed(seed)
        legacy = torch.stack([torch.randint(0, 2 ** 62, (2,), dtype=torch.int64) for _ in range(items)])
        assert torch.equal(rows, calls) and torch.equal(rows, legacy)

