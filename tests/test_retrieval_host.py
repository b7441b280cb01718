"""Retrieval on the host: the oracle's DINOv2 tokens against the reference's (golden fixture), the oracle's descriptor, neighbour and
pair rules on hand-made cases, the argument rules of `select_pairs` and `global_descriptors`, the C-ABI structs, and a dry run of
`Engine.global_descriptors` with the recording stand-in for `cabi.call`."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, load_golden
from oracle import retrieval as oracle
from oracle.roma_oracle import RomaOracle
from roma_b200 import arch, cabi
from roma_b200.matcher import RegressionMatcher
from roma_b200.retrieval import select_pairs
from test_host_logic import fake, host_engine
from test_match_pairs_host import _PairRecorder


def test_oracle_tokens_match_the_reference(weights):
    """`reference_tokens` (roma_oracle's ViT blocks) against the reference's `forward_features` on the same weights and image."""
    g = load_golden("retrieval_dinov2")
    tokens = oracle.reference_tokens(RomaOracle(*weights, coarse_res=(42, 56)), torch.from_numpy(g["image"])).numpy()
    ref = np.concatenate((g["x_norm_clstoken"][:, None], g["x_norm_patchtokens"]), axis=1)
    assert tokens.shape == ref.shape == (1, 13, arch.VIT_DIM)
    err = np.abs(tokens - ref).max() / np.abs(ref).max()
    assert err <= 1e-5, err
    d, d_ref = oracle.descriptor(tokens), oracle.descriptor(ref)
    assert np.abs(d - d_ref).max() <= 1e-5


def test_descriptor_rules():
    rng = np.random.default_rng(0)
    t = rng.standard_normal((3, 6, 5)).astype(np.float32)
    t[1, 0] = 0                                          # a zero class token: its half stays zero
    t[2, 1:] = 0                                         # zero patch tokens: the mean half stays zero
    d = oracle.descriptor(t)
    assert d.dtype == np.float32 and d.shape == (3, 10)
    for e in range(3):
        c, s = t[e, 0], np.float32(0)
        m = []
        for ch in range(5):
            s = np.float32(0)
            for k in range(1, 6):
                s = np.float32(s + t[e, k, ch])
            m.append(np.float32(s / np.float32(5)))
        for half, v in ((0, c), (1, np.array(m, dtype=np.float32))):
            q = np.float32(0)
            for x in v:
                q = np.float32(q + np.float32(x * x))
            den = np.float32(oracle.SQRT2 * np.float32(np.sqrt(q)))
            want = np.zeros(5, np.float32) if q == 0 else (v / den).astype(np.float32)
            assert np.array_equal(d[e, 5 * half:5 * half + 5], want), (e, half)
    assert np.all(d[1, :5] == 0) and np.all(d[2, 5:] == 0)
    assert abs(np.linalg.norm(d[0].astype(np.float64)) - 1) < 1e-6


def test_neighbour_rules_on_hand_made_cases():
    # ties: rows 1, 2 and 3 are identical, so row 0 scores them equally and takes the lower indices first
    X = np.array([[1, 0], [1, 0], [1, 0], [1, 0], [0, 1]], dtype=np.float32)
    nb, sc, pairs = oracle.select_pairs(X, 2)
    assert nb.tolist() == [[1, 2], [0, 2], [0, 1], [0, 1], [0, 1]]
    assert sc[4].tolist() == [0, 0] and sc[0].tolist() == [1, 1]
    assert pairs.tolist() == [[0, 1], [0, 2], [0, 3], [0, 4], [1, 2], [1, 3], [1, 4]]
    # -0 counts as +0: j = 1 (-0) and j = 2 (+0) tie, the lower index first
    S = np.array([[0, -0.0, 0, -1], [0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0]], dtype=np.float32)
    assert oracle.neighbors(S, 2)[0][0].tolist() == [1, 2]
    # k >= N - 1: the exhaustive graph
    X = np.random.default_rng(1).standard_normal((6, 4)).astype(np.float32)
    nb, _, pairs = oracle.select_pairs(X, 10)
    assert nb.shape == (6, 5) and pairs.tolist() == [[i, j] for i in range(6) for j in range(i + 1, 6)]
    # mutual neighbours are one pair; every image is in at least k pairs and P <= N k
    X = np.array([[4, 0], [3, 1], [0, 4], [1, 3]], dtype=np.float32)
    nb, _, pairs = oracle.select_pairs(X, 1)
    assert nb[:, 0].tolist() == [1, 0, 3, 2] and pairs.tolist() == [[0, 1], [2, 3]]
    # N = 2
    nb, sc, pairs = oracle.select_pairs(np.array([[1, 2], [3, 4]], dtype=np.float32), 20)
    assert nb.tolist() == [[1], [0]] and sc.tolist() == [[11], [11]] and pairs.tolist() == [[0, 1]]


def test_select_pairs_argument_rules():
    ok = torch.zeros(4, 8)
    cases = [(np.zeros((4, 8), np.float32), {}, "floating-point CUDA tensor"), (torch.zeros(4, 8, dtype=torch.int32), {}, "floating-point"),
             (torch.zeros(4, 8, 2), {}, r"\[N, D\]"), (torch.zeros(1, 8), {}, "1 images"), (torch.zeros(65536, 1), {}, "65536 images"),
             (torch.zeros(4, 0), {}, "at least one component"), (ok, dict(num_neighbors=0), "num_neighbors"),
             (ok, dict(num_neighbors=129), "num_neighbors"), (ok, dict(num_neighbors=2.0), "num_neighbors"),
             (ok, dict(num_neighbors=True), "num_neighbors"), (ok, dict(workspace_bytes=15), "holds no row"),
             (ok, {}, "got one on cpu")]
    for x, kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            select_pairs(x, **kw)


def test_global_descriptors_argument_rules(weights, monkeypatch):
    m = RegressionMatcher.__new__(RegressionMatcher)
    m.engine = host_engine(weights, monkeypatch, "fp32", _PairRecorder())
    m.h_resized = m.w_resized = 56
    with pytest.raises(ValueError, match="max_batch"):
        m.global_descriptors(torch.zeros(2, 3, 56, 56), max_batch=0)
    with pytest.raises(ValueError, match=r"\[N, 3, h, w\]"):
        m.global_descriptors(torch.zeros(3, 56, 56))
    with pytest.raises(ValueError, match="Unsupported input type"):
        m.global_descriptors(["a.jpg", 3])


def test_structs_and_validators():
    desc = dict(cabi.STRUCT_FIELDS["rb_global_descriptor_args"])
    ret = dict(cabi.STRUCT_FIELDS["rb_retrieval_args"])
    for struct, types in (("rb_global_descriptor_args", desc), ("rb_retrieval_args", ret)):
        assert set(cabi._FIELD_DTYPES[struct]) == {f for f, t in types.items() if t is ctypes.c_void_p}, struct
    assert ret["ld_scores"] is ctypes.c_int64 and ret["num_pairs"] is ctypes.c_int64 and ret["k"] is ctypes.c_int32
    for fn in ("romab200_global_descriptor", "romab200_retrieval_select", "romab200_retrieval_pairs_count", "romab200_retrieval_pairs_emit"):
        assert fn in cabi.FUNCTIONS
    assert (cabi.RB_RETRIEVAL_MAX_IMAGES, cabi.RB_RETRIEVAL_MAX_K) == (65535, 128)
    N, k = 10, 3
    kw = dict(num_images=N, k=k, scores=fake(torch.zeros(4 * N)), ld_scores=N, row_begin=2, row_end=6, neighbors=fake(torch.zeros(N, k, dtype=torch.int64)),
              neighbor_scores=fake(torch.zeros(N, k)), status=fake(torch.zeros(1, dtype=torch.int32)))
    cabi._validate("romab200_retrieval_select", "rb_retrieval_args", kw)
    with pytest.raises(RuntimeError, match="`scores` holds 39 elements, the described geometry needs 40"):
        cabi._validate("romab200_retrieval_select", "rb_retrieval_args", dict(kw, scores=fake(torch.zeros(39))))
    with pytest.raises(RuntimeError, match="`neighbors` has dtype torch.int32"):
        cabi._validate("romab200_retrieval_select", "rb_retrieval_args", dict(kw, neighbors=fake(torch.zeros(N, k, dtype=torch.int32))))
    pk = dict(num_images=N, k=k, neighbors=kw["neighbors"], keys=fake(torch.zeros(N * k, dtype=torch.int64)), keys_alt=fake(torch.zeros(N * k, dtype=torch.int64)),
              hist=fake(torch.zeros(257, dtype=torch.int32)), offsets=fake(torch.zeros(N * k + 1, dtype=torch.int64)))
    cabi._validate("romab200_retrieval_pairs_count", "rb_retrieval_args", pk)
    with pytest.raises(RuntimeError, match="`offsets` holds 30 elements"):
        cabi._validate("romab200_retrieval_pairs_count", "rb_retrieval_args", dict(pk, offsets=fake(torch.zeros(N * k, dtype=torch.int64))))
    with pytest.raises(RuntimeError, match="`pairs` holds 10 elements, the described geometry needs 12"):
        cabi._validate("romab200_retrieval_pairs_emit", "rb_retrieval_args", dict(pk, num_pairs=6, pairs=fake(torch.zeros(5, 2, dtype=torch.int64))))
    dk = dict(tokens=fake(torch.zeros(2, 5, 8, dtype=torch.float16)), out=fake(torch.zeros(2, 16)), batch=2, n_tokens=5, dim=8, tokens_dtype=cabi.RB_F16)
    cabi._validate("romab200_global_descriptor", "rb_global_descriptor_args", dk)
    with pytest.raises(RuntimeError, match="`tokens` has dtype torch.float16, the call describes it as torch.float32"):
        cabi._validate("romab200_global_descriptor", "rb_global_descriptor_args", dict(dk, tokens_dtype=cabi.RB_F32))
    with pytest.raises(RuntimeError, match="`out` holds 30 elements, the described geometry needs 32"):
        cabi._validate("romab200_global_descriptor", "rb_global_descriptor_args", dict(dk, out=fake(torch.zeros(30))))


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


def test_entry_points_refuse_bad_arguments_before_any_cuda_call():
    addr = 1 << 20
    desc = dict(tokens=addr, out=addr, batch=2, n_tokens=5, dim=1024, tokens_dtype=cabi.RB_F32)
    sel = dict(num_images=10, k=3, scores=addr, ld_scores=10, row_begin=0, row_end=10, neighbors=addr, neighbor_scores=addr, status=addr)
    pk = dict(num_images=10, k=3, neighbors=addr, keys=addr, keys_alt=addr, hist=addr, offsets=addr, pairs=addr)
    calls = [
        ("global_descriptor", "rb_global_descriptor_args", dict(desc, tokens_dtype=cabi.RB_F16S), "global_descriptor: unsupported dtype 3"),
        ("global_descriptor", "rb_global_descriptor_args", dict(desc, dim=1025),
         "global_descriptor: bad shape batch=2 n_tokens=5 dim=1025 (dim <= 1024)"),
        ("global_descriptor", "rb_global_descriptor_args", dict(desc, n_tokens=1), "global_descriptor: bad shape batch=2 n_tokens=1 dim=1024 (dim <= 1024)"),
        ("retrieval_select", "rb_retrieval_args", dict(sel, k=10), "retrieval_select: k 10 outside [1, min(128, num_images - 1)]"),
        ("retrieval_select", "rb_retrieval_args", dict(sel, num_images=65536, ld_scores=65536),
         "retrieval_select: num_images 65536 outside [2, 65535]"),
        ("retrieval_select", "rb_retrieval_args", dict(sel, row_end=11), "retrieval_select: rows [0, 11) of 10 images, ld_scores 10"),
        ("retrieval_select", "rb_retrieval_args", dict(sel, status=0), "retrieval_select: null argument"),
        ("retrieval_pairs_count", "rb_retrieval_args", dict(pk, hist=0), "retrieval_pairs_count: null argument"),
        ("retrieval_pairs_emit", "rb_retrieval_args", dict(pk, k=129, num_images=200), "retrieval_pairs_emit: k 129 outside [1, min(128, num_images - 1)]"),
    ]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    flags = ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable, *flags, "-c", _CHILD], input=json.dumps([c[:3] for c in calls]), capture_output=True, text=True, cwd=ROOT,
                         env=env, timeout=600)
    assert res.returncode == 0, res.stderr
    for (fn, _, _, want), (rc, msg) in zip(calls, json.loads(res.stdout.strip().splitlines()[-1])):
        assert rc != 0 and msg == want, (fn, rc, msg)


@pytest.mark.parametrize("precision", ["fp32", "fp32_simt", "fp16", "bf16"])
def test_engine_global_descriptors_dry_run(weights, monkeypatch, precision):
    """`Engine.global_descriptors` launches DINOv2's calls exactly as match()'s image stage does, without the class-token drop, the
    CNN branch or the GP, then one descriptor call over the whole token array; every pointer lies inside a tracked tensor."""
    E, H, W = 3, 56, 70
    rec = _PairRecorder()
    eng = host_engine(weights, monkeypatch, precision, rec)
    images, out = torch.zeros(E, 3, H, W), torch.zeros(E, 2 * arch.VIT_DIM)
    rec.track(images)
    rec.track(out)
    eng.global_descriptors(images, out)
    calls = [(fn, sc) for fn, _, sc, _ in rec.log]
    rec2 = _PairRecorder()
    eng2 = host_engine(weights, monkeypatch, precision, rec2)
    rec2.track(images)
    eng2.dinov2(images)
    vit = [(fn, sc) for fn, _, sc, _ in rec2.log]
    assert vit[-E:] == [c for c in vit[-E:] if c[0] == "romab200_copy2d"] and len(vit) > 24 * 5
    assert calls[:-1] == vit[:-E]
    fn, _, scalars, kw = rec.log[-1]
    n = (H // 14) * (W // 14)
    assert fn == "romab200_global_descriptor" and dict(scalars) == dict(batch=E, n_tokens=n + 1, dim=arch.VIT_DIM, tokens_dtype=eng.dt)
    assert kw["out"] is out and kw["tokens"].shape == (E * (n + 1), arch.VIT_DIM) and kw["tokens"].dtype == eng.dtype


def test_mixed_high_res_inputs_are_refused(weights, monkeypatch):
    """`_device_inputs`, now built on the coarse half that `global_descriptors` shares, still names every input when only some
    high-resolution tensors are given."""
    m = RegressionMatcher.__new__(RegressionMatcher)
    m.engine = host_engine(weights, monkeypatch, "fp32", _PairRecorder())
    m.h_resized = m.w_resized = 56
    m.upsample_preds, m.upsample_res = True, (84, 84)
    t = torch.zeros(1, 3, 56, 56)
    with pytest.raises(ValueError, match="(?s)Invalid upsample_preds and high_res inputs with im_A=.*im_A_high_res=.*im_B=.* and im_B_high_res=None"):
        m._device_inputs([t, t], [torch.zeros(1, 3, 84, 84), None], ("im_A", "im_B"))
    lo, hi = m._device_inputs([t, t], [t, t], ("im_A", "im_B"))
    assert lo[0] is t and hi[1] is t
