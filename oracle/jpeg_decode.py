"""Host statement of the device JPEG decoder (roma_b200/csrc/jpeg.cu) in numpy and plain Python, for the tests.

It restates libjpeg-turbo's default decompression for the subset `roma_b200.jpeg.parse` accepts, step by step:
  - `parse`               the header parse (the package's own parser: the oracle pins what it returns);
  - `entropy_decode`      sequential Huffman decode (jdhuff.c decode_mcu), restart intervals, DC prediction ->
                          int16 coefficient blocks per component [by, bx, 64] in natural order;
  - `idct_islow`          dequantise + jpeg_idct_islow (CONST_BITS 13, PASS1_BITS 2, range_limit[x & RANGE_MASK]);
  - `upsample`            h2v1 / h2v2 fancy upsampling (jdsample.c), plain replication for components <= 2 samples wide;
  - `ycc_to_rgb`          the fixed-point ycc_rgb_convert tables (jdcolor.c).
`decode(data, mode)` chains them; tests pin its bytes to the installed Pillow's.  The entropy decode declines (ValueError)
exactly where the device decoder does: an invalid code, a run past coefficient 63, bits past the end of an interval,
restart markers out of sequence, a scan not followed by EOI.
"""
from __future__ import annotations

import numpy as np

from roma_b200.jpeg import JpegInfo, ZIGZAG, parse  # noqa: F401  (parse is part of the oracle's surface)


def unstuff(scan: bytes):
    """Entropy-coded bytes of the scan -> (list of interval byte strings, end offset).  FF 00 -> FF, fill FFs dropped,
    RSTn splits intervals (checked to run 0, 1, ..., 7, 0, ...); the first other marker ends the scan and must be EOI."""
    out = []
    cur = bytearray()
    i, n = 0, len(scan)
    nrst = 0
    while True:
        if i >= n:
            raise ValueError("no EOI marker after the scan (truncated file)")
        b = scan[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        j = i + 1
        while j < n and scan[j] == 0xFF:
            j += 1
        if j >= n:
            raise ValueError("no EOI marker after the scan (truncated file)")
        m = scan[j]
        if m == 0:
            cur.append(0xFF)
            i = j + 1
        elif 0xD0 <= m <= 0xD7:
            if m - 0xD0 != nrst % 8:
                raise ValueError("restart markers missing or out of sequence")
            nrst += 1
            out.append(bytes(cur))
            cur = bytearray()
            i = j + 1
        elif m == 0xD9:
            out.append(bytes(cur))
            return out
        else:
            raise ValueError("no EOI marker after the scan (truncated file)")


class _Bits:
    def __init__(self, data: bytes):
        self.d = bytes(data) + bytes(8)        # bits past the end read as zero (only a decode that consumes them is an error)
        self.n = len(data) * 8
        self.pos = 0

    def peek(self, k):
        p = self.pos
        w = int.from_bytes(self.d[p >> 3:(p >> 3) + 4], "big")
        return (w >> (32 - (p & 7) - k)) & ((1 << k) - 1)

    def take(self, k):
        r = self.peek(k)
        self.pos += k
        return r


def _huff(bits: _Bits, t):
    k = 0
    for length in range(1, 17):
        code = bits.peek(length)
        n = t.bits[length - 1]
        first = _first_code(t, length)
        if n and first <= code < first + n:
            bits.pos += length
            return t.vals[k + code - first]
        k += n
    raise ValueError("corrupt entropy-coded data (invalid Huffman code)")


_FIRST = {}


def _first_code(t, length):
    key = (t.bits, length)
    f = _FIRST.get(key)
    if f is None:
        code = 0
        for l in range(1, length):
            code = (code + t.bits[l - 1]) << 1
        _FIRST[key] = f = code
    return f


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(data: bytes, info: JpegInfo = None):
    """-> list per frame component of int16 [by, bx, 64] coefficient blocks (natural order, DC resolved)."""
    info = info or parse(data)
    intervals = unstuff(data[info.scan_data:])
    mx, my, bpm, slots = info.geometry()
    total = mx * my
    R = info.restart_interval or total
    if len(intervals) != -(-total // R):
        raise ValueError("restart markers missing or out of sequence")
    tabs = {ci: (dc, ac) for ci, dc, ac in info.scan}
    blocks = [np.zeros((info.plane_shape(ci)[0] // 8, info.plane_shape(ci)[1] // 8, 64), np.int16) for ci in range(info.ncomp)]
    for j, iv in enumerate(intervals):
        bits = _Bits(iv)
        pred = [0] * info.ncomp
        for m in range(j * R, min((j + 1) * R, total)):
            for ci, dy, dx in slots:
                dc, ac = tabs[ci]
                blk = np.zeros(64, np.int64)
                s = _huff(bits, dc)
                diff = _extend(bits.take(s), s)
                pred[ci] += diff
                blk[0] = pred[ci]
                k = 1
                while k < 64:
                    rs = _huff(bits, ac)
                    r, s = rs >> 4, rs & 15
                    if s:
                        k += r
                        if k > 63:
                            raise ValueError("corrupt entropy-coded data (run past coefficient 63)")
                        blk[ZIGZAG[k]] = _extend(bits.take(s), s)
                        k += 1
                    elif r == 15:
                        k += 16
                        if k > 64:
                            raise ValueError("corrupt entropy-coded data (run past coefficient 63)")
                    else:
                        break
                if bits.pos > bits.n:
                    raise ValueError("corrupt entropy-coded data (bits past the end of the interval)")
                if info.single:
                    by, bx = divmod(m, mx)
                else:
                    _, h, v, _ = info.comps[ci]
                    by, bx = (m // mx) * v + dy, (m % mx) * h + dx
                blocks[ci][by, bx] = blk.astype(np.int16)       # JCOEF: int16, wraps like the C cast
    return blocks


_C = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
          c2053=16819, c2562=20995, c3072=25172)


def _idct_1d(x0, x1, x2, x3, x4, x5, x6, x7):
    c = _C
    z1 = (x2 + x6) * c["c0541"]
    tmp2 = z1 + x6 * -c["c1847"]
    tmp3 = z1 + x2 * c["c0765"]
    tmp0 = (x0 + x4) << 13
    tmp1 = (x0 - x4) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x7, x5, x3, x1
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * c["c1175"]
    tmp0 = tmp0 * c["c0298"]
    tmp1 = tmp1 * c["c2053"]
    tmp2 = tmp2 * c["c3072"]
    tmp3 = tmp3 * c["c1501"]
    z1 = z1 * -c["c0899"]
    z2 = z2 * -c["c2562"]
    z3 = z3 * -c["c1961"] + z5
    z4 = z4 * -c["c0390"] + z5
    tmp0 += z1 + z3
    tmp1 += z2 + z4
    tmp2 += z2 + z3
    tmp3 += z1 + z4
    return (t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


# Pillow's libjpeg-turbo runs the SIMD build of jpeg_idct_islow: 16-bit lanes for the dequantised coefficients, the pass-1
# workspace and the pairwise sums of both (z0 +- z4, c7 + c3, c5 + c1), 32-bit products, packssdw / packsswb saturation at
# the end.  It equals the C arithmetic restated here exactly while every dequantised coefficient and every pass-1 output
# lies in [-16384, 16383] (pairwise sums fit 16 bits, the DC-only column shortcut 4 * z0 fits) and every pass-2 output in
# [-512, 511] (there range_limit[x & 1023] and the saturation give the same sample).  Outside, the decode declines.
LANE_LIMIT = 16384
OUT_LIMIT = 512


def idct_islow(blocks: np.ndarray, qt: np.ndarray) -> np.ndarray:
    """int16 [by, bx, 64] natural-order coefficients, quant table [64] -> uint8 plane [by * 8, bx * 8].  ValueError when a
    block leaves the range where the SIMD and C IDCTs agree."""
    by, bx, _ = blocks.shape
    c = blocks.reshape(-1, 8, 8).astype(np.int64) * qt.reshape(8, 8).astype(np.int64)
    # pass 1: columns
    cols = _idct_1d(*[c[:, r, :] for r in range(8)])
    ws = np.stack([_descale(v, 13 - 2) for v in cols], axis=1)             # [n, row, col]
    rows = _idct_1d(*[ws[:, :, k] for k in range(8)])
    out = np.stack([_descale(v, 13 + 2 + 3) for v in rows], axis=2)        # [n, row, col]
    if (c.size and (c.min() < -LANE_LIMIT or c.max() >= LANE_LIMIT or ws.min() < -LANE_LIMIT or ws.max() >= LANE_LIMIT
                    or out.min() < -OUT_LIMIT or out.max() >= OUT_LIMIT)):
        raise ValueError("coefficients outside the range of the 16-bit IDCT")
    pix = np.clip(out + 128, 0, 255).astype(np.uint8)       # = range_limit[out & 1023] inside [-512, 511]
    return pix.reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)


def upsample(plane: np.ndarray, dh: int, dw: int, h: int, v: int) -> np.ndarray:
    """Chroma plane (valid region dh x dw) -> (v * dh) x (h * dw), libjpeg-turbo's h2v1 / h2v2 fancy upsampling, or
    replication when the component is at most 2 samples wide."""
    p = plane[:dh, :dw].astype(np.int32)
    if h == 1 and v == 1:
        return p
    if dw <= 2:
        return np.repeat(np.repeat(p, v, axis=0), h, axis=1)
    left = np.concatenate([p[:, :1], p[:, :-1]], axis=1)
    right = np.concatenate([p[:, 1:], p[:, -1:]], axis=1)
    if v == 1:
        even = (3 * p + left + 1) >> 2
        odd = (3 * p + right + 2) >> 2
        even[:, 0] = p[:, 0]
        odd[:, -1] = p[:, -1]
        out = np.empty((dh, 2 * dw), np.int32)
        out[:, 0::2], out[:, 1::2] = even, odd
        return out
    above = np.concatenate([p[:1], p[:-1]], axis=0)
    below = np.concatenate([p[1:], p[-1:]], axis=0)
    out = np.empty((2 * dh, 2 * dw), np.int32)
    for r, nb in ((0, above), (1, below)):
        cs = 3 * p + nb
        cl = np.concatenate([cs[:, :1], cs[:, :-1]], axis=1)
        cr = np.concatenate([cs[:, 1:], cs[:, -1:]], axis=1)
        even = (3 * cs + cl + 8) >> 4
        odd = (3 * cs + cr + 7) >> 4
        even[:, 0] = (4 * cs[:, 0] + 8) >> 4
        odd[:, -1] = (4 * cs[:, -1] + 7) >> 4
        out[r::2, 0::2], out[r::2, 1::2] = even, odd
    return out


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
    y = y.astype(np.int64)
    xb = cb.astype(np.int64) - 128
    xr = cr.astype(np.int64) - 128
    r = y + ((91881 * xr + 32768) >> 16)
    g = y + ((-22554 * xb + 32768 - 46802 * xr) >> 16)
    b = y + ((116130 * xb + 32768) >> 16)
    return np.clip(np.stack([r, g, b], axis=-1), 0, 255).astype(np.uint8)


def decode(data: bytes, mode=None) -> np.ndarray:
    """uint8 [H, W, C] equal to np.asarray(Image.open(...)) (or .convert("RGB") with mode="RGB")."""
    info = parse(data)
    blocks = entropy_decode(data, info)
    H, W = info.height, info.width
    planes = [idct_islow(blocks[ci], info.qtables[ci]) for ci in range(info.ncomp)]
    if info.ncomp == 1:
        g = planes[0][:H, :W]
        return np.repeat(g[:, :, None], 3, axis=2) if mode == "RGB" else g[:, :, None].copy()
    y = planes[0][:H, :W]
    h0, v0 = info.comps[0][1], info.comps[0][2]
    dw, dh = -(-W // h0), -(-H // v0)
    cb = upsample(planes[1], dh, dw, h0, v0)[:H, :W]
    cr = upsample(planes[2], dh, dw, h0, v0)[:H, :W]
    return ycc_to_rgb(y, cb, cr)
