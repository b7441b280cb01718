"""JPEG header parse, the host oracle pinned to the installed Pillow, and the fallback of the path route (no GPU)."""
import io
import os

import numpy as np
import pytest
from PIL import Image

from oracle import jpeg_decode as oj
from roma_b200 import jpeg, synthetic

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
    return synthetic.jpeg_corpus(0, max_pixels=640 * 480)


def test_parser_accepts_and_declines(corpus):
    names = {n for n, _, _ in corpus}
    assert {"progressive_64x48", "cmyk_64x48", "rgb_64x48_440", "gray_640x480_q90", "rgb_640x480_rst1"} <= names
    for name, data, decline in corpus:
        if decline is None:
            info = jpeg.parse(data)
            assert info.mode == Image.open(io.BytesIO(data)).mode, name
        else:
            with pytest.raises(jpeg.JpegDecline, match=decline) as e:
                jpeg.parse(data)
            assert not e.value.malformed, name
    for path in FIXTURES:
        info = jpeg.parse(open(path, "rb").read())
        assert (info.width, info.height) == Image.open(path).size and info.comps[0][1:3] == (2, 2)


def test_parser_declines_malformed_headers():
    base = open(FIXTURES[0], "rb").read()
    for cut in (1, 3, 20, 200):
        with pytest.raises(jpeg.JpegDecline) as e:
            jpeg.parse(base[:cut])
        assert e.value.malformed
    with pytest.raises(jpeg.JpegDecline, match="impossible code"):
        jpeg.parse(bad_huffman_table(base))
    i = base.index(b"\xff\xc0")
    dnl = bytearray(base)
    dnl[i + 5:i + 7] = b"\x00\x00"              # height 0: the height would come from a DNL marker
    with pytest.raises(jpeg.JpegDecline, match="DNL"):
        jpeg.parse(bytes(dnl))
    b12 = bytearray(base)
    b12[i + 4] = 12
    with pytest.raises(jpeg.JpegDecline, match="12-bit"):
        jpeg.parse(bytes(b12))


def test_oracle_matches_pillow_corpus(corpus):
    for name, data, decline in corpus:
        if decline is not None:
            continue
        assert np.array_equal(oj.decode(data), _pil(data)), name
        if name.startswith("gray"):
            assert np.array_equal(oj.decode(data, "RGB"), _pil(data, "RGB")), name


@pytest.mark.slow
def test_oracle_matches_pillow_fixtures():
    for path in FIXTURES[:2]:
        data = open(path, "rb").read()
        assert np.array_equal(oj.decode(data), _pil(data)), path


def test_oracle_declines_corrupt_streams():
    """The corrupt streams the GPU test feeds the device decoder: the oracle either reproduces Pillow or declines."""
    base = open(FIXTURES[0], "rb").read()
    s0 = jpeg.parse(base).scan_data
    for k in (1, 2, 3):
        with pytest.raises(ValueError, match="EOI"):
            oj.entropy_decode(base[:s0 + (len(base) - s0) * k // 4])
    flip = bytearray(base)
    flip[s0 + 5000] ^= 0x5A
    try:
        got = oj.decode(bytes(flip))
    except ValueError:
        got = None
    if got is not None:
        assert np.array_equal(got, _pil(bytes(flip)))


def test_oracle_edits_match_pillow_or_decline():
    """Quantisation tables edited past the 16-bit IDCT's range and single-bit flips of the entropy data: the oracle (which
    declines where the device decoder does) either gives Pillow's bytes or declines."""
    accepted = set()
    for name, data in synthetic.jpeg_edits(0):
        try:
            got = oj.decode(data, "RGB")
        except (ValueError, jpeg.JpegDecline):
            continue
        accepted.add(name)
        assert np.array_equal(got, _pil(data, "RGB")), name
    assert {"dqt1_gray_16x16", "dqt2_rgb_16x16"} <= accepted and not accepted & {"dqt8_gray_16x16", "dqt32_rgb_16x16"}
    assert sum("flip" in n for n in accepted) > 200


def test_declined_files_take_the_host_route(corpus, tmp_path, monkeypatch):
    from roma_b200 import cabi
    from roma_b200.preprocess import open_inputs

    def refuse(*a, **k):
        raise AssertionError("a declined file reached the C ABI")

    monkeypatch.setattr(cabi, "call", refuse)
    for name in ("progressive_64x48", "cmyk_64x48", "rgb_64x48_440"):
        data = [d for n, d, _ in corpus if n == name][0]
        p = tmp_path / f"{name}.jpg"
        p.write_bytes(data)
        (rgb,) = open_inputs([str(p)], "cuda", rgb=True)
        assert isinstance(rgb, Image.Image) and np.array_equal(np.asarray(rgb), _pil(data, "RGB"))
        (raw,) = open_inputs([str(p)], "cuda", rgb=False)
        assert isinstance(raw, Image.Image) and raw.mode == Image.open(p).mode


def test_path_route_keeps_pillow_errors(tmp_path, monkeypatch):
    from roma_b200 import cabi
    from roma_b200.preprocess import open_inputs

    monkeypatch.setattr(cabi, "call", lambda *a, **k: (_ for _ in ()).throw(AssertionError("reached the C ABI")))
    p16 = tmp_path / "i16.png"
    Image.fromarray(np.arange(64, dtype=np.uint16).reshape(8, 8)).save(p16)
    assert Image.open(p16).mode == "I;16"
    with pytest.raises(NotImplementedError, match="16 bit"):
        open_inputs([str(p16)], "cuda")
    big = tmp_path / "big.jpg"
    big.write_bytes(open(FIXTURES[0], "rb").read())
    monkeypatch.setattr(Image, "MAX_IMAGE_PIXELS", 1000)
    with pytest.raises(Image.DecompressionBombError):
        open_inputs([str(big)], "cuda")
