"""CPU dry run of `match_pairs` with the recording stand-in for `cabi.call` of test_host_logic.py: which images are encoded and in
which batches, that a decode chunk launches exactly the pair work match() launches for b = P, and that every pointer, including
every row the bank gathers and scatters move, stays inside a tracked tensor.  Also the host-side argument rules."""
import ctypes
import math

import pytest
import torch

from roma_b200 import arch, cabi, synthetic
from roma_b200.cache import GraphCache
from roma_b200.matcher import RegressionMatcher, pair_tensor, plan_pairs
from test_host_logic import _Recorder, _tensors, host_engine

# the calls of Engine.image_stage other than gp_rows, which a decode chunk runs again on the gathered p16
IMAGE_STAGE = ("dinov2", "encode_cnn", "gp_project", "gp_solve_images")


class _PairRecorder(_Recorder):
    """Keeps (function, stage, scalar arguments) of every call, the image an im2col call reads, and checks every row a gather moves."""

    def __init__(self):
        super().__init__()
        self.log, self.encoded, self.image_stage = [], [], 0

    def __call__(self, fn, struct, **kw):
        super().__call__(fn, struct, **kw)
        ptrs = {f for f, t in cabi.STRUCT_FIELDS[struct] if t is ctypes.c_void_p}
        scalars = tuple((k, v) for k, v in sorted(kw.items()) if k not in ptrs and not isinstance(v, torch.Tensor))
        self.log.append((fn, self.image_stage > 0, scalars, kw))
        if fn == "romab200_im2col_patch":
            self.encoded.append(kw["image"].clone())
        if fn == "romab200_gather_rows":
            base = {k: kw[k].data_ptr() for k in ("src", "dst")}
            for i in range(kw["count"]):
                s = int(kw["src_index"][i]) if kw.get("src_index") is not None else i
                d = int(kw["dst_index"][i]) if kw.get("dst_index") is not None else i
                assert 0 <= s < kw["src_rows"] and 0 <= d < kw["dst_rows"], (s, d)
                self._inside(base["src"] + s * kw["ld_src"], kw["row_bytes"], "gather_rows.src")
                self._inside(base["dst"] + d * kw["ld_dst"], kw["row_bytes"], "gather_rows.dst")


def _engine(weights, monkeypatch, precision):
    """A host-only Engine of `precision` whose C-ABI calls go to a _PairRecorder."""
    rec = _PairRecorder()
    eng = host_engine(weights, monkeypatch, precision, rec)
    for name in IMAGE_STAGE:           # mark the calls of the per-image stage
        def wrapped(*a, _f=getattr(eng, name), **k):
            rec.image_stage += 1
            try:
                return _f(*a, **k)
            finally:
                rec.image_stage -= 1
        setattr(eng, name, wrapped)
    return eng, rec


class _TrackingCache(GraphCache):
    def __init__(self, rec):
        super().__init__()
        self.rec = rec

    def entry(self, key, make, enabled=True, generation=0):
        e = super().entry(key, make, enabled, generation)
        for t in _tensors(e["bufs"]):
            self.rec.track(t)
        return e


@pytest.mark.parametrize("symmetric,upsample,split", [(True, True, True), (False, True, False), (True, False, False), (True, True, False),
                                                      (False, True, True), (True, False, True), (False, False, True), (False, False, False)])
def test_match_pairs_dry_run(weights, monkeypatch, symmetric, upsample, split):
    eng, rec = _engine(weights, monkeypatch, "fp32" if split else "fp32_simt")
    coarse, up = 112, 168
    A, B, Ah, Bh = synthetic.make_pair(3, coarse, up, 2)
    images, images_hi = torch.cat((A, B)), torch.cat((Ah, Bh))         # 6 images; image 5 is in no pair
    model = RegressionMatcher(eng, h=coarse, w=coarse, upsample_preds=upsample, symmetric=symmetric, upsample_res=(up, up))
    model.use_cuda_graph = False
    model._pair_graphs = _TrackingCache(rec)
    pairs = pair_tensor([(0, 1), (2, 3), (4, 0), (1, 1), (3, 2)], 6)
    plan = plan_pairs(pairs, 2)
    assert plan["used"] == [0, 1, 2, 3, 4] and plan["chunks"] == [(0, 2, 0, 4), (2, 4, 4, 8), (4, 5, 8, 10)]
    ho = up if upsample else coarse
    wout = 2 * ho if symmetric else ho
    warp, cert = model._match_pairs_device(images, images_hi if upsample else None, plan, (coarse, coarse), (up, up) if upsample else (0, 0),
                                           (ho, wout), None)
    assert warp.shape == (5, ho, wout, 4) and cert.shape == (5, ho, wout)

    # encode: one batch of 2, 2, 1 images, each referenced image once, image 5 never
    solves = [kw["batch"] for fn, _, _, kw in rec.log if fn == "romab200_gp_solve"]
    assert solves == [2, 2, 1]
    assert [x.shape[0] for x in rec.encoded] == [2, 2, 1]
    encoded = torch.cat(rec.encoded)
    assert torch.equal(encoded, images[:5])
    first_decode = next(i for i, (fn, stage, _, _) in enumerate(rec.log) if fn == "romab200_gather_rows" and (rec.log[i][3].get("src_index") is not None))
    assert "romab200_refiner_prologue" not in [fn for fn, _, _, _ in rec.log[:first_decode]]

    # decode: after its gathers, every chunk launches the pair work of match(b = P), i.e. the calls of run_match outside the
    # image stage, call for call with the same scalar arguments
    decode = [(fn, sc) for fn, _, sc, _ in rec.log[first_decode:] if fn != "romab200_gather_rows"]
    expect = []
    for b in (2, 2, 1):
        n0 = len(rec.log)
        imgs = torch.cat((images[:b], images[b:2 * b])); rec.track(imgs)
        hi = torch.cat((images_hi[:b], images_hi[b:2 * b])) if upsample else None
        out = (torch.empty(b, ho, wout, 4), torch.empty(b, ho, wout))
        for t in (hi, *out):
            if t is not None:
                rec.track(t)
        eng.run_match(imgs, hi, b, symmetric, math.sqrt(coarse * coarse / 560 ** 2), math.sqrt(up * up / 560 ** 2), False, *out)
        expect += [(fn, sc) for fn, stage, sc, _ in rec.log[n0:] if not stage]
    # the one difference: mu = K_xy @ alpha reads alpha^T from the gathered [2P, 512, ldw] rows rather than from rows n.. of the
    # solve's [2P, n + 512, ldw] workspace, so its per-image B stride differs
    def mu_stride_free(calls):
        return [(fn, tuple((k, v) for k, v in sc if not (k == "sb0" and dict(sc).get("ldc") == arch.DEC_DIM and dict(sc).get("N") == arch.GP_DIM)))
                for fn, sc in calls]
    assert mu_stride_free(decode) == mu_stride_free(expect)
    n_gathers = sum(fn == "romab200_gather_rows" and kw.get("src_index") is not None for fn, _, _, kw in rec.log[:len(rec.log)])
    assert n_gathers == 3 * (2 + 4 * (2 if upsample else 1))


def test_pair_arguments():
    assert pair_tensor([(0, 1), (2, 2)], 3).tolist() == [[0, 1], [2, 2]]
    assert pair_tensor(torch.tensor([[1, 0]], dtype=torch.int32), 2).dtype == torch.int64
    assert pair_tensor([], 3).shape == (0, 2) and pair_tensor(torch.empty(0, 2, dtype=torch.long), 3).shape == (0, 2)
    with pytest.raises(IndexError):
        pair_tensor([(0, 3)], 3)
    with pytest.raises(IndexError):
        pair_tensor(torch.tensor([[0, -1]]), 3)
    for bad in (torch.zeros(2, 3, dtype=torch.long), torch.zeros(4, dtype=torch.long), torch.zeros(2, 2), [(0, 1, 2)], [(0, 0.5)], [0, 1]):
        with pytest.raises(ValueError):
            pair_tensor(bad, 3)
    plan = plan_pairs(torch.tensor([[3, 1], [1, 3], [5, 5]]), 8)
    assert plan["used"] == [1, 3, 5] and plan["index"].tolist() == [1, 0, 2, 0, 1, 2] and plan["chunks"] == [(0, 3, 0, 6)]


@pytest.mark.parametrize("precision,symmetric", [("fp16", True), ("bf16", False), ("fp32", True), ("fp16", False), ("bf16", True),
                                               ("fp32", False), ("fp32_simt", True), ("fp32_simt", False)])
def test_debug_captures_are_inert(weights, monkeypatch, precision, symmetric):
    """`engine.debug = {}` only clones stage tensors: a dry run of match()'s device side (`run_match`: both passes and the
    epilogue) makes the same C-ABI calls, in the same order and with the same scalar arguments, as with `debug = None` (the CNN
    overlap is off in both), and keeps every stage tensor tests/test_fast_mode_stages_gpu.py reads, in its documented shape."""
    b, coarse, up = 2, 112, 168
    A, B, Ah, Bh = synthetic.make_pair(b, coarse, up, 2)
    logs = {}
    for debug in (None, {}):
        eng, rec = _engine(weights, monkeypatch, precision)
        eng.debug = debug
        images, hi = torch.cat((A, B)), torch.cat((Ah, Bh))
        wout = 2 * up if symmetric else up
        out = (torch.empty(b, up, wout, 4), torch.empty(b, up, wout))
        for t in (images, hi, *out):
            rec.track(t)
        eng.run_match(images, hi, b, symmetric, coarse / 560, up / 560, True, *out)
        logs[debug is None] = [(fn, sc) for fn, _, sc, _ in rec.log]
    assert logs[True] == logs[False] and len(logs[True]) > 300
    dbg, E, D, n = eng.debug, 2 * b, (2 * b if symmetric else b), (coarse // 14) ** 2
    assert dbg["vit.feat16"].shape == (E, n, arch.VIT_DIM) and dbg["gp.p16"].shape == (E, n, arch.PROJ[16][1])
    assert dbg["tokens"].shape == (D, n, arch.DEC_DIM) and dbg["gp.mu"].shape == (D, n, arch.GP_DIM)
    for tag, res in (("lo", coarse), ("up", up)):
        for s in (1, 2, 4, 8):
            assert dbg[f"{tag}.vgg{s}"].shape == (E, res // s, res // s, arch.PROJ[s][0]) and dbg[f"{tag}.vgg{s}"].dtype == torch.float32
        for s in ((16, 8, 4, 2, 1) if tag == "lo" else (8, 4, 2, 1)):
            h = res // s if s < 16 else coarse // 14
            for k in ("state_in", "state_out", "delta"):
                assert dbg[f"{tag}{s}.{k}"].shape == (D, h, h, 3), (tag, s, k)
