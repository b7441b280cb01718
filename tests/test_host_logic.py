"""CPU tests of the host side: C-ABI library loads and exports what the header declares, weight packing
(BN folding) is right, and a dry run of the whole engine with a recording fake of `cabi.call` checks every
kernel call's argument names, dtypes and that every pointer range stays inside an allocated buffer."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from roma_b200 import arch, cabi, synthetic
from roma_b200.packing import PackedWeights, Split, at, fold_bn, pad8


def test_library_exports_every_declared_symbol():
    lib = cabi.load_library()
    assert lib.romab200_abi_version() == 4
    assert len(cabi.FUNCTIONS) >= 20
    for fn in cabi.FUNCTIONS:
        assert hasattr(lib, fn), fn
    assert ctypes.sizeof(cabi.STRUCTS["rb_gemm_args"]) == 368


def test_fold_bn_matches_batchnorm(weights):
    sd = weights[0]
    x = torch.randn(2, 64, 9, 9)
    w, b = sd["encoder.cnn.layers.3.weight"], sd["encoder.cnn.layers.3.bias"]
    ref = F.batch_norm(F.conv2d(x, w, b, padding=1), sd["encoder.cnn.layers.4.running_mean"], sd["encoder.cnn.layers.4.running_var"],
                       sd["encoder.cnn.layers.4.weight"], sd["encoder.cnn.layers.4.bias"], False, 0.0, 1e-5)
    w2, b2 = fold_bn(w, b, sd, "encoder.cnn.layers.4")
    assert (F.conv2d(x, w2, b2, padding=1) - ref).abs().max() < 2e-5


def test_packing_layouts(weights):
    pw = PackedWeights(weights[0], weights[1], torch.device("cpu"), torch.float32)
    assert pw.vgg[0]["w"].shape == (64, 27) and pw.vgg[1]["w"].shape == (64, 576)
    # 3x3 weights are (ky, kx, cin)-major
    w, _ = fold_bn(weights[0]["encoder.cnn.layers.3.weight"], weights[0]["encoder.cnn.layers.3.bias"], weights[0], "encoder.cnn.layers.4")
    assert torch.equal(pw.vgg[1]["w"].reshape(64, 3, 3, 64)[5, 1, 2], w[5, :, 1, 2])
    R = pw.refiner[16]
    assert R["c"] == 1377 and R["cp"] == 1384 and R["blocks"][0]["dw_w"].shape == (25, 1384)
    assert R["blocks"][0]["pw_w"].shape == (1377, 1384) and (R["blocks"][0]["pw_w"][:, 1377:] == 0).all()
    assert pw.vit_patch_w.shape == (1024, 592)
    with pytest.raises(RuntimeError):
        bad = dict(weights[0]); bad.pop("decoder.gps.16.pos_conv.bias")
        PackedWeights(bad, weights[1], torch.device("cpu"), torch.float32)


class _Recorder:
    """Stands in for cabi.call: validates field names, that every pointer field is a tensor (offsets are views) or None, and that
    pointer ranges lie inside live tensors."""

    def __init__(self):
        self.calls = []
        self.allocs = {}

    def track(self, t):
        self.allocs[t.data_ptr()] = t.numel() * t.element_size()

    def _inside(self, ptr, nbytes, what):
        if isinstance(ptr, torch.Tensor):
            ptr = ptr.data_ptr()
        for base, size in self.allocs.items():
            if base <= ptr and ptr + nbytes <= base + size:
                return
        raise AssertionError(f"{what}: pointer range [{ptr}, +{nbytes}) not inside any tracked buffer")

    def __call__(self, fn, struct, **kw):
        valid = {f for f, _ in cabi.STRUCT_FIELDS[struct]}
        assert set(kw) <= valid, (fn, set(kw) - valid)
        ptrs = {f for f, t in cabi.STRUCT_FIELDS[struct] if t is ctypes.c_void_p}
        raw = {k: type(v).__name__ for k, v in kw.items() if k in ptrs and v is not None and not isinstance(v, torch.Tensor)}
        assert not raw, (fn, "pointer fields take tensors or None", raw)
        self.calls.append(fn)
        es = {0: 4, 1: 2, 2: 2, 3: 2}
        if fn == "romab200_gemm":
            if kw["dtype_ab"] == cabi.RB_F16S:        # split pairs: the second planes have the same geometry
                assert kw.get("A_lo") is not None and kw.get("B_lo") is not None
                lo = dict(kw, A=kw["A_lo"], B=kw["B_lo"], A_lo=None, B_lo=None, dtype_ab=cabi.RB_F16)
                if kw["dtype_c"] == cabi.RB_F16S:
                    lo.update(C=kw["C_lo"], dtype_c=cabi.RB_F16)
                self.calls.pop()
                self(fn, struct, **{k: v for k, v in lo.items() if v is not None})
            if kw["dtype_c"] == cabi.RB_F16S:
                assert kw.get("C_lo") is not None
            b0, b1 = kw.get("batch0", 1), kw.get("batch1", 1)
            M, N, K = kw["M"], kw["N"], kw["K"]
            ea, ec = es[kw["dtype_ab"]], es[kw["dtype_c"]]
            nt = kw.get("ntaps", 1)
            kt = K // nt
            off = (b0 - 1) * kw.get("sa0", 0) + (b1 - 1) * kw.get("sa1", 0)
            if nt == 1:
                self._inside(kw["A"], (off + (M - 1) * kw["lda"] + kt) * ea, f"{fn}.A")
            else:
                assert kw["a_rows"] == M
                self._inside(kw["A"], ((kw["a_rows"] - 1) * kw["lda"] + kt) * ea, f"{fn}.A")
            offb = (b0 - 1) * kw.get("sb0", 0) + (b1 - 1) * kw.get("sb1", 0)
            if kw.get("trans_b", 0):
                self._inside(kw["B"], (offb + (K - 1) * kw["ldb"] + N) * ea, f"{fn}.B")
            else:
                self._inside(kw["B"], (offb + (N - 1) * kw["ldb"] + K) * ea, f"{fn}.B")
            offc = (b0 - 1) * kw.get("sc0", 0) + (b1 - 1) * kw.get("sc1", 0)
            rows_out = M
            if kw.get("rowmap", 0) == cabi.ROWMAP_PAD_TO_COMPACT:
                rows_out = M // (kw["pad_h"] * kw["pad_w"]) * (kw["pad_h"] - 2) * (kw["pad_w"] - 2)
            self._inside(kw["C"], (offc + (rows_out - 1) * kw["ldc"] + N) * ec, f"{fn}.C")
            assert kw["lda"] % 4 == 0 and kw["ldb"] % 4 == 0, "vector path wants 16-byte pitches"
            if ea == 2:
                assert kw["lda"] % 8 == 0 and kw["ldb"] % 8 == 0, "TMA wants 16-byte pitches"
        for k, v in kw.items():
            if isinstance(v, torch.Tensor):
                assert v.is_contiguous(), (fn, k)
                self._inside(v, 1, f"{fn}.{k}")


class _ArgRecorder(_Recorder):
    """_Recorder that also keeps the arguments of every call"""

    def __init__(self):
        super().__init__()
        self.args = []

    def __call__(self, fn, struct, **kw):
        self.args.append((fn, kw))
        super().__call__(fn, struct, **kw)


def host_engine(weights, monkeypatch, precision, rec):
    """A host-only Engine of `precision` (CPU tensors, CNN inline) whose C-ABI calls go to the recording stand-in `rec`, which
    tracks every weight, arena buffer and constant of the engine."""
    import roma_b200.engine as engine_mod
    eng = engine_mod.Engine.__new__(engine_mod.Engine)
    engine_mod.BufferArena.__init__(eng, "cpu")
    eng.precision, eng.dtype = precision, engine_mod.PRECISIONS[precision]
    eng.dt, eng.split, eng._lane = cabi.DTYPE_CODE[eng.dtype], precision == "fp32", "main"
    eng.w = PackedWeights(weights[0], weights[1], eng.device, eng.dtype, split=eng.split)
    eng.debug, eng.profile, eng.gemm_profile, eng.use_flash_attn, eng.gp_algo = None, None, None, True, (2 if precision == "fp32_simt" else 3)
    eng.overlap_cnn, eng._side, eng.gp_tensor_core, eng.fused_c144, eng.fused_small_f32 = False, None, True, True, True
    eng.lc_table16, eng.lc_tile_radii, eng.side_ctas = True, (2,), 0
    eng._bank, eng.bank_version = None, 0
    for t in _tensors(eng.w):
        rec.track(t)
    orig_buf, orig_const = eng.buf, eng.const

    def buf(*a, **k):
        t = orig_buf(*a, **k); rec.track(t); return t

    def const(*a, **k):
        t = orig_const(*a, **k); rec.track(t); return t
    eng.buf, eng.const = buf, const
    monkeypatch.setattr(engine_mod, "call", rec)
    return eng


@pytest.mark.parametrize("symmetric,upsample,split", [(True, True, True), (True, True, False), (False, True, True), (True, False, False),
                                                      (False, True, False), (False, False, True), (False, False, False), (True, False, True)])
def test_engine_dry_run(weights, monkeypatch, symmetric, upsample, split):
    rec = _Recorder()
    eng = host_engine(weights, monkeypatch, "fp32" if split else "fp32_simt", rec)
    chains, orig_chain = [], eng.refine_chain

    def refine_chain(state, scales, feats, sizes, *a, **k):
        out = orig_chain(state, scales, feats, sizes, *a, **k)
        chains.append((sizes, out))
        return out
    eng.refine_chain = refine_chain
    b, coarse, up = 1, 112, 168
    A, B, Ah, Bh = synthetic.make_pair(b, coarse, up, 1)
    images, hi = torch.cat((A, B)), (torch.cat((Ah, Bh)) if upsample else None)
    D, H = (2 * b if symmetric else b), (up if upsample else coarse)
    wout = 2 * H if symmetric else H
    warp, cert = torch.empty(b, H, wout, 4), torch.empty(b, H, wout)
    for t in (images, hi, warp, cert):
        if t is not None:
            rec.track(t)
    eng.run_match(images, hi, b, symmetric, coarse / 560, up / 560, False, warp, cert)
    assert len(chains) == (2 if upsample else 1)
    sizes, (state, states) = chains[0]
    assert sizes == {1: (112, 112), 2: (56, 56), 4: (28, 28), 8: (14, 14), 16: (8, 8)}
    assert state.shape == (D, 112, 112, 3) and states[16].shape == (D, 8, 8, 3)
    if upsample:
        state = chains[1][1][0]
        assert state.shape == (D, 168, 168, 3)
    n_gemm = rec.calls.count("romab200_gemm")
    per_pass_refiner = 9 * (5 if not upsample else 5 + 4)
    # refiner pointwise GEMMs (the stride-1 blocks are fused kernels) + 24 ViT blocks x 4 linears (+ 2 attention GEMMs un-fused)
    assert n_gemm > per_pass_refiner * 4 // 5 + 24 * 4
    assert rec.calls.count("romab200_gp_solve") == 1
    assert rec.calls.count("romab200_refiner_prologue") == (9 if upsample else 5)


@pytest.mark.parametrize("precision", ["fp32", "fp32_simt", "fp16", "bf16"])
@pytest.mark.parametrize("coarse,up", [((126, 182), (182, 238)), ((560, 784), None)])
def test_engine_dry_run_token_grids(weights, monkeypatch, precision, coarse, up):
    """Coarse grids of 9 x 13 = 117 tokens (odd: the GP solve's last block) and of 40 x 56 = 2240 tokens (decoder rows longer than
    2048) through run_match under the recorder's bounds checks, symmetric, with the GP solve and the softmax calls they reach."""
    rec = _ArgRecorder()
    eng = host_engine(weights, monkeypatch, precision, rec)
    b = 1
    A, B, Ah, Bh = synthetic.make_pair(b, coarse, up, 1)
    images, hi = torch.cat((A, B)), (torch.cat((Ah, Bh)) if up else None)
    H, W = up or coarse
    warp, cert = torch.empty(b, H, 2 * W, 4), torch.empty(b, H, 2 * W)
    for t in (images, hi, warp, cert):
        if t is not None:
            rec.track(t)
    scale = lambda r: (r[0] * r[1] / 560 ** 2) ** 0.5    # noqa: E731
    eng.run_match(images, hi, b, True, scale(coarse), scale(up or coarse), False, warp, cert)
    n = (coarse[0] // 14) * (coarse[1] // 14)
    solves = [kw for fn, kw in rec.args if fn == "romab200_gp_solve"]
    assert len(solves) == 1 and solves[0]["n"] == n and solves[0]["batch"] == 2 * b
    s = solves[0]
    assert s["ldw"] == pad8(n) and s["stride"] == (n + s["nrhs"]) * s["ldw"] and s["algo"] == (2 if precision == "fp32_simt" else 3)
    if s["algo"] == 3:                   # the workspace the header asks of algo 3
        need = s["batch"] * (-(-n // 128) * 65536 + 4 * max((n + s["nrhs"]) * 128 + 16384, s["nrhs"] * 128 + 16384 + 128 * s["ldw"]))
        assert s["workspace_bytes"] >= need
    long_rows = [kw for fn, kw in rec.args if fn == "romab200_softmax_rows" and kw["cols"] == n]
    if precision == "fp32":              # the parity decoder: QK^T, the split-output softmax, PV in each of its 5 blocks
        assert len(long_rows) == 5 and all(kw["out_hi"] is not None and kw["ldo"] == pad8(n) for kw in long_rows)


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        yield obj
    elif isinstance(obj, dict):
        for v in obj.values():
            yield from _tensors(v)
    elif isinstance(obj, (list, tuple)):
        for v in obj:
            yield from _tensors(v)
    elif hasattr(obj, "hi") and hasattr(obj, "lo"):          # packing.Split (RB_F16S pair)
        yield from _tensors([obj.hi, obj.lo])
    elif hasattr(obj, "__dict__"):
        yield from _tensors(vars(obj))


def test_layout_product_never_imports_oracle():
    """The shipped package must not route through the oracle (or the reference) anywhere."""
    import os
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "roma_b200")
    for dirpath, _, files in os.walk(root):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text and "romatch import" not in text, f


def test_cabi_call_validates_tensors():
    """The ctypes shim refuses tensors whose device / dtype / layout / size contradict the call's description (a raw pointer of
    the wrong kind would be silent garbage on the device)."""
    a = torch.zeros(8, 8)
    with pytest.raises(RuntimeError, match="expected the current CUDA device"):
        cabi.call("romab200_gemm", "rb_gemm_args", A=a, B=a, C=a, M=8, N=8, K=8, lda=8, ldb=8, ldc=8, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32)
    with pytest.raises(TypeError):
        cabi.call("romab200_gemm", "rb_gemm_args", not_a_field=1)
    # dtype / contiguity / size rules, exercised on the validator itself with the device check satisfied by a stand-in
    half, f32 = fake(torch.zeros(8, 8, dtype=torch.float16)), fake(torch.zeros(8, 8))
    kw = dict(A=half, B=half, C=f32, M=8, N=8, K=8, lda=8, ldb=8, ldc=8, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32)
    with pytest.raises(RuntimeError, match="dtype"):
        cabi._validate("romab200_gemm", "rb_gemm_args", kw)
    kw.update(A=f32, B=f32, M=16)
    with pytest.raises(RuntimeError, match="needs"):
        cabi._validate("romab200_gemm", "rb_gemm_args", kw)
    kw.update(M=8, A=fake(torch.zeros(8, 16)[:, :8]))
    with pytest.raises(RuntimeError, match="contiguous"):
        cabi._validate("romab200_gemm", "rb_gemm_args", kw)
    kw.update(A=f32)
    cabi._validate("romab200_gemm", "rb_gemm_args", kw)


class FakeCuda(torch.Tensor):
    """A host tensor that the shim takes for one on the current CUDA device."""
    is_cuda = True

    @property
    def device(self):
        return type("D", (), {"type": "cuda", "index": torch.cuda.current_device() if torch.cuda.is_available() else None})()


def fake(t):
    return t.as_subclass(FakeCuda)


def test_cabi_call_refuses_raw_addresses():
    """A pointer field takes a tensor or None: an int (a hand-built address) is refused before the library is called."""
    a = fake(torch.zeros(8, 8))
    for field in ("A", "bias"):
        kw = dict(A=a, B=a, C=a, M=8, N=8, K=8, lda=8, ldb=8, ldc=8, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32)
        kw[field] = a.data_ptr() + 64
        with pytest.raises(TypeError, match=f"romab200_gemm: pointer field `{field}`"):
            cabi.call("romab200_gemm", "rb_gemm_args", **kw)


def test_cabi_host_fields():
    """The refiner block's pointwise weights are read on the host: contiguous fp32 CPU tensors; its maps stay device tensors."""
    m = fake(torch.zeros(2, 16, 16, 24))
    kw = dict(out=fake(torch.zeros(2, 16, 16, 24)), ld=24, dw_weight=fake(torch.zeros(25, 24)), ldw=24, dw_bias=fake(torch.zeros(24)),
              pw_weight_host=torch.zeros(24, 24), pw_bias_host=torch.zeros(24), batch=2, h=16, w=16, c=24, dtype=cabi.RB_F32)
    kw["in"] = m
    cabi._validate("romab200_refiner_block_small", "rb_refiner_block_small_args", kw)
    for bad, why in ((fake(torch.zeros(24, 24)), "read on the host"), (torch.zeros(24, 24, dtype=torch.float16), "dtype"),
                     (torch.zeros(24, 48)[:, :24], "contiguous")):
        with pytest.raises(RuntimeError, match=why):
            cabi._validate("romab200_refiner_block_small", "rb_refiner_block_small_args", dict(kw, pw_weight_host=bad))
    with pytest.raises(RuntimeError, match="expected the current CUDA device"):
        cabi._validate("romab200_refiner_block_small", "rb_refiner_block_small_args", dict(kw, dw_bias=torch.zeros(24)))


def test_split_at_returns_offset_views():
    hi, lo = torch.arange(24, dtype=torch.float16).view(4, 6), torch.zeros(4, 6, dtype=torch.float16)
    s = Split(hi, lo).at(7)
    for view, base in ((s.hi, hi), (s.lo, lo)):
        assert view.untyped_storage().data_ptr() == base.untyped_storage().data_ptr()
        assert view.data_ptr() == base.data_ptr() + 7 * 2 and view.numel() == 24 - 7 and view.dtype == torch.float16
    assert s.hi[0] == 7 and torch.equal(s.at(5).hi, at(hi, 12))
    with pytest.raises(RuntimeError):
        at(hi[:, :3], 1)                # only a contiguous buffer has a flat view


def test_cabi_offset_views_checked_against_geometry():
    """An operand that starts inside a buffer must still hold what the described geometry reads (GEMM, copy2d, gather_rows)."""
    buf = torch.zeros(8, 8)
    gemm = dict(B=fake(buf), C=fake(buf), M=8, N=8, K=8, lda=8, ldb=8, ldc=8, dtype_ab=cabi.RB_F32, dtype_c=cabi.RB_F32)
    cabi._validate("romab200_gemm", "rb_gemm_args", dict(gemm, A=fake(at(buf, 0)), M=7))
    with pytest.raises(RuntimeError, match="`A` holds 56 elements, the described geometry needs 64"):
        cabi._validate("romab200_gemm", "rb_gemm_args", dict(gemm, A=fake(at(buf, 8))))
    copy = dict(src=fake(at(buf, 40)), dst=fake(buf), rows=3, cols=8, lds=8, ldd=8, dtype_src=cabi.RB_F32, dtype_dst=cabi.RB_F32)
    cabi._validate("romab200_copy2d", "rb_copy2d_args", copy)
    with pytest.raises(RuntimeError, match="`src` holds 23 elements, the described geometry needs 24"):
        cabi._validate("romab200_copy2d", "rb_copy2d_args", dict(copy, src=fake(at(buf, 41))))
    with pytest.raises(RuntimeError, match="`dst` holds 15 elements, the described geometry needs 24"):
        cabi._validate("romab200_copy2d", "rb_copy2d_args", dict(copy, dst=fake(at(buf, 49))))
    rows = dict(src=fake(at(buf, 16)), dst=fake(buf), count=3, row_bytes=64, ld_src=64, ld_dst=64, src_rows=3, dst_rows=3)
    cabi._validate("romab200_gather_rows", "rb_gather_rows_args", rows)         # 48 fp32 = 192 bytes = 2 * 64 + 64
    with pytest.raises(RuntimeError, match="`src` holds 44 elements, the described geometry needs 48"):
        cabi._validate("romab200_gather_rows", "rb_gather_rows_args", dict(rows, src=fake(at(buf, 20))))
    with pytest.raises(RuntimeError, match="`dst` holds 48 elements, the described geometry needs 64"):
        cabi._validate("romab200_gather_rows", "rb_gather_rows_args", dict(rows, dst=fake(at(buf, 16)), ld_dst=96))


def test_romatch_import_shim():
    """`import romatch` through shim/ gives the reference's import surface backed by this package (romatch/__init__.py:2-8)."""
    import importlib
    import os
    import sys
    shim = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "shim")
    sys.path.insert(0, shim)
    try:
        for m in [k for k in sys.modules if k == "romatch" or k.startswith("romatch.")]:
            del sys.modules[m]
        romatch = importlib.import_module("romatch")
        import roma_b200
        assert romatch.roma_outdoor is roma_b200.roma_outdoor and romatch.roma_indoor is roma_b200.roma_indoor
        assert romatch.tiny_roma_v1_outdoor is roma_b200.tiny_roma_v1_outdoor
        assert (romatch.DEBUG_MODE, romatch.GLOBAL_STEP, romatch.STEP_SIZE, romatch.LOCAL_RANK) == (False, 0, 1, -1) and isinstance(romatch.RANK, int)
        zoo = importlib.import_module("romatch.models.model_zoo")
        assert "outdoor" in zoo.weight_urls["romatch"] and zoo.roma_model is roma_b200.model_zoo.roma_model
        assert importlib.import_module("romatch.models.matcher").RegressionMatcher is roma_b200.matcher.RegressionMatcher
    finally:
        sys.path.remove(shim)
        for m in [k for k in sys.modules if k == "romatch" or k.startswith("romatch.")]:
            del sys.modules[m]


def test_prologue_tiles_matches_kernel_geometry():
    """cabi.prologue_tiles (the size of the `tile_done` workspace callers allocate) follows the tile shapes compiled into the kernels."""
    import os, re
    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "roma_b200", "csrc", "refiner_common.cuh")).read()
    generic = re.search(r"template <int R> struct LcTile \{ static constexpr int TQX = (\d+), TQY = (\d+)", text)
    r7 = re.search(r"struct LcTile<7> \{ static constexpr int TQX = (\d+), TQY = (\d+)", text)
    r2 = re.search(r"struct LcTile<2> \{ static constexpr int TQX = (\d+), TQY = (\d+)", text)
    shapes = {3: tuple(map(int, generic.groups())), 7: tuple(map(int, r7.groups())), 2: tuple(map(int, r2.groups()))}
    for r, (tx, ty) in shapes.items():
        for h, w in ((40, 40), (70, 70), (108, 108), (13, 9), (1, 1)):
            assert cabi.prologue_tiles(r, h, w) == -(-h // ty) * -(-w // tx), (r, h, w)


def test_graph_cache_policy(monkeypatch):
    """GraphCache: eager on call 1, eager then capture on call 2, replay from call 3 (counting the captured launches); an entry
    of an older arena generation is made again; a disabled entry is neither kept nor captured.  CUDA graphs are a host stand-in."""
    from contextlib import contextmanager
    from roma_b200 import cache
    events, launches = [], [0]

    class FakeGraph:
        def replay(self):
            events.append("replay")

    @contextmanager
    def capture(graph):
        events.append("capture")
        yield
    monkeypatch.setattr(torch.cuda, "CUDAGraph", FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", capture)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a: None)
    monkeypatch.setattr(cache.cabi, "kernel_launches", lambda: launches[0])

    def work(i):
        events.append("run")
        launches[0] += 3
        return i
    gc, outs = cache.GraphCache(), []
    for i in range(4):
        e = gc.entry("k", lambda: {"i": i}, True, 0)
        outs.append(gc.run(e, lambda: work(i)))
    assert events == ["run", "run", "capture", "run", "replay", "replay"]
    assert outs == [(0, False), (1, False), (1, True), (1, True)] and e["bufs"] == {"i": 0} and gc.launches == 6
    e2 = gc.entry("k", lambda: {"i": 9}, True, 1)
    assert e2 is not e and e2["bufs"] == {"i": 9} and gc.run(e2, lambda: work(9)) == (9, False) and gc["k"] is e2
    events.clear()
    for _ in range(3):
        assert gc.run(gc.entry("off", lambda: {}, False), lambda: work(5)) == (5, False)
    assert events == ["run"] * 3 and "off" not in gc
    gc.clear()
    assert not gc and gc.launches == 6
