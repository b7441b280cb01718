"""Device JPEG decoding (roma_b200/csrc/jpeg.cu) against the installed Pillow and the host oracle, and the path routes of
`match` / `match_from_path` against their PIL inputs."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from roma_b200 import jpeg, synthetic

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.abspath(__file__))
FIXTURES = [os.path.join(ROOT, "golden", "jpeg", f) for f in ("sacre_coeur_A.jpg", "sacre_coeur_B.jpg", "toronto_A.jpg")]


def bad_huffman_table(data):
    """Moves two codes of the first DHT table to length 1: the segment stays well formed, the code is impossible."""
    j = data.index(b"\xff\xc4")
    b = bytearray(data)
    k = max(range(16), key=lambda t: b[j + 5 + t])
    b[j + 5 + k] -= 2
    b[j + 5] += 2
    return bytes(b)


def _pil(data, mode=None):
    im = Image.open(io.BytesIO(data))
    if mode:
        im = im.convert(mode)
    a = np.asarray(im)
    return a[:, :, None] if a.ndim == 2 else a


@pytest.fixture(scope="module")
def corpus():
    return synthetic.jpeg_corpus(0)


def _accepted(corpus):
    return [(n, d) for n, d, dec in corpus if dec is None]


def test_corpus_one_at_a_time(corpus):
    from roma_b200 import decode_jpeg
    for name, data in _accepted(corpus):
        got = decode_jpeg([data])[0]
        assert torch.equal(got.cpu(), torch.from_numpy(_pil(data))), name
    for path in FIXTURES:
        data = open(path, "rb").read()
        assert torch.equal(decode_jpeg(path)[0].cpu(), torch.from_numpy(_pil(data))), path


def test_batch_mixed_sizes_and_formats(corpus):
    from roma_b200 import decode_jpeg
    items = [d for _, d in _accepted(corpus) if len(d) < 2_000_000] + [open(p, "rb").read() for p in FIXTURES]
    got = decode_jpeg(items, mode="RGB")
    for data, g in zip(items, got):
        assert torch.equal(g.cpu(), torch.from_numpy(_pil(data, "RGB")))


def test_coefficients_match_oracle(corpus):
    from oracle import jpeg_decode as oj
    streams = [open(p, "rb").read() for p in FIXTURES[:2]] + [d for n, d in _accepted(corpus) if "rst" in n]
    passes = []
    for data in streams:
        blocks, status, npass = jpeg.decode_coefficients(data)
        assert status == 0
        want = oj.entropy_decode(data)
        for b, w in zip(blocks, want):
            assert np.array_equal(b, w)
        passes.append(npass)
    assert max(passes[:2]) > 1, passes         # the resynchronisation path runs on real camera data


def test_declined_raise_not_implemented(corpus):
    from roma_b200 import decode_jpeg
    for name, data, dec in corpus:
        if dec is not None:
            with pytest.raises(NotImplementedError, match=dec):
                decode_jpeg([data])


def corrupt_streams():
    """Fixed, deterministic edits of sacre_coeur_A.jpg and a restart-marker file."""
    base = open(FIXTURES[0], "rb").read()
    info = jpeg.parse(base)
    s0 = info.scan_data
    out = {f"trunc_{k}": base[:s0 + (len(base) - s0) * k // 4] for k in (1, 2, 3)}
    flip = bytearray(base)
    flip[s0 + 5000] ^= 0x5A
    out["flip"] = bytes(flip)
    rst = [d for n, d, _ in synthetic.jpeg_corpus(0, max_pixels=640 * 480) if n == "rgb_640x480_rst3"][0]
    i = rst.index(b"\xff\xd2")
    bad = bytearray(rst)
    bad[i + 1] = 0xD5
    out["rst_number"] = bytes(bad)
    out["huffman"] = bad_huffman_table(base)
    return out


def test_corrupt_streams_decode_exactly_or_raise():
    from roma_b200 import decode_jpeg
    for name, data in corrupt_streams().items():
        try:
            want = _pil(data, "RGB")
        except Exception:
            want = None
        try:
            got = decode_jpeg([data], mode="RGB")[0].cpu().numpy()
        except ValueError:
            continue
        assert want is not None and np.array_equal(got, want), name


def test_edits_match_pillow_or_decline():
    """The DQT and bit-flip edits in one batch: every stream the device accepts gives Pillow's bytes, and it accepts exactly
    the streams the oracle accepts."""
    from oracle import jpeg_decode as oj
    items = []
    for name, data in synthetic.jpeg_edits(0):
        try:
            items.append((name, data, jpeg.parse(data)))
        except jpeg.JpegDecline:
            pass
    res, _ = jpeg.decode_device([d for _, d, _ in items], [i for _, _, i in items], "cuda", [True] * len(items))
    n_ok = 0
    for (name, data, _), r in zip(items, res):
        try:
            want_oracle = oj.decode(data, "RGB")
        except ValueError:
            want_oracle = None
        if isinstance(r, str):
            assert want_oracle is None, (name, r)
            continue
        n_ok += 1
        assert want_oracle is not None, name
        assert np.array_equal(r.cpu().numpy(), _pil(data, "RGB")), name
    assert n_ok > 200


def test_large_decode_memory(corpus):
    from roma_b200 import decode_jpeg
    name, data = [(n, d) for n, d in _accepted(corpus) if "6000x4000" in n][0]
    info = jpeg.parse(data)
    mx, my, bpm, _ = info.geometry()
    coef_bytes = mx * my * bpm * 128
    out_bytes = info.width * info.height * 3
    plane_bytes = sum(h * w for h, w in (info.plane_shape(c) for c in range(info.ncomp)))
    sz = jpeg._Plan([(data, info)], [False]).sizes
    # compressed stream + compacted stream + chunk / interval / sync-state tables + coefficients + planes
    need = len(data) + sz["comp"] + 8 * sz["chunks"] + 4 * sz["intervals"] + (24 + 8) * sz["slots"] + coef_bytes + plane_bytes
    assert need <= coef_bytes + plane_bytes + 3 * len(data)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    got = decode_jpeg([data])[0]
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base - out_bytes
    assert extra <= need + (1 << 20), (extra, need)
    assert torch.equal(got.cpu(), torch.from_numpy(_pil(data)))


# ---- routes through match() ------------------------------------------------------------------------------------------
def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


@pytest.fixture(scope="module")
def roma(weights):
    from roma_b200 import roma_outdoor
    return roma_outdoor("cuda:0", weights=weights[0], dinov2_weights=weights[1], coarse_res=112, upsample_res=168,
                        amp_dtype=torch.float32)


def test_roma_match_paths(roma, corpus, tmp_path):
    gray = [d for n, d, _ in corpus if n == "gray_640x480_q90"][0]
    prog = [d for n, d, _ in corpus if n == "progressive_64x48"][0]
    pairs = [tuple(FIXTURES[:2]), (_write(tmp_path, "g.jpg", gray), _write(tmp_path, "g2.jpg", gray)),
             (_write(tmp_path, "p.jpg", prog), FIXTURES[0])]
    for a, b in pairs:
        w, c = roma.match(a, b)
        wr, cr = roma.match(Image.open(a).convert("RGB"), Image.open(b).convert("RGB"))
        assert torch.equal(w, wr) and torch.equal(c, cr), (a, b)
    w, c = roma.match(FIXTURES[0], Image.open(FIXTURES[1]).convert("RGB"))
    wr, cr = roma.match(Image.open(FIXTURES[0]).convert("RGB"), Image.open(FIXTURES[1]).convert("RGB"))
    assert torch.equal(w, wr) and torch.equal(c, cr)


def test_roma_match_corrupt_paths(roma, tmp_path):
    for name, data in corrupt_streams().items():
        p = _write(tmp_path, name + ".jpg", data)
        try:
            want = roma.match(Image.open(p).convert("RGB"), Image.open(FIXTURES[1]).convert("RGB"))
        except Exception as e:          # noqa: BLE001 - the same exception type must come from the path route
            with pytest.raises(type(e)):
                roma.match(p, FIXTURES[1])
            continue
        got = roma.match(p, FIXTURES[1])
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]), name


def test_tiny_match_from_path(corpus, tmp_path):
    from roma_b200 import tiny_roma_v1_outdoor
    xf = synthetic.xfeat_standin()
    model = tiny_roma_v1_outdoor("cuda:0", weights=synthetic.make_tiny_weights(0, xf), xfeat=xf)
    gray = [d for n, d, _ in corpus if n == "gray_640x480_q90"][0]
    g = _write(tmp_path, "g.jpg", gray)
    for a, b in (tuple(FIXTURES[:2]), (g, g)):
        w, c = model.match_from_path(a, b)
        wr, cr = model.match(Image.open(a), Image.open(b))
        assert torch.equal(w, wr) and torch.equal(c, cr), (a, b)
