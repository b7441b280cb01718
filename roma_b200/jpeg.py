"""JPEG decoding on the device: header parse on the host, entropy decode, IDCT and colour conversion in `csrc/jpeg.cu`.

The decoder restates libjpeg-turbo's default decompression (the one Pillow runs: ISLOW integer IDCT, fancy upsampling,
table-driven YCbCr -> RGB), so its output is byte-identical to `np.asarray(Image.open(src))`.  It covers what cameras and
Pillow's encoder write:

  - 8-bit, Huffman-coded, sequential (SOF0 / SOF1), one scan holding every component (Ss=0, Se=63, Ah=Al=0);
  - 1 component (grayscale), or 3 components that libjpeg treats as YCbCr;
  - luma sampling (1,1), (2,1) or (2,2) with chroma at (1,1): 4:4:4, 4:2:2, 4:2:0;
  - any restart interval.

Everything else is declined by `parse` with the reason named (`JpegDecline`), before any device work: progressive and
arithmetic coding, 12-bit and lossless, multi-scan files, 4 components, 3 components libjpeg treats as RGB, other sampling
layouts, a DNL marker (height 0), and truncated or malformed headers.  Callers that have a host route (`match` with
paths) fall back to Pillow for those files.

Device pipeline (one launch set for a whole batch; all per-image numbers live in an int64 descriptor row, `D_*` below,
whose layout `csrc/jpeg.cu` shares):
  romab200_jpeg_entropy   unstuff + restart markers, self-synchronising parallel Huffman decode, coefficient emit,
                          DC prediction -> int16 coefficients [blocks, 64] in natural order, a status word per image;
  romab200_jpeg_pixels    dequantise + ISLOW IDCT into per-component planes, upsample + colour convert -> uint8 [H, W, C].
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from typing import List, Optional, Sequence, Tuple

import numpy as np

SUBSEQ_BITS = 512          # bits per Huffman-decode subsequence (one thread each); must match JPG_SUBSEQ_BITS in jpeg.cu
CHUNK_BYTES = 4096         # bytes per CTA of the unstuff kernels; must match JPG_CHUNK in jpeg.cu
STREAM_PAD = 16            # zero bytes after every compacted stream, so that bit lookahead stays in bounds

# descriptor row (int64 per image), shared with csrc/jpeg.cu
D_STREAM_OFF, D_STREAM_LEN, D_COMP_OFF, D_N_INTERVALS, D_IV_OFF, D_SLOT_OFF, D_N_SLOTS, D_CHUNK_OFF, D_N_CHUNKS, \
    D_BLOCK_OFF, D_N_BLOCKS, D_MCUS_PER_IV, D_BPM, D_MCUS_X, D_MCUS_Y, D_TOTAL_MCUS, D_WIDTH, D_HEIGHT, D_NCOMP, \
    D_OUT_OFF, D_OUT_CH, D_SINGLE = range(22)
D_PLANE_OFF, D_PLANE_PITCH, D_PLANE_H, D_HSAMP, D_VSAMP, D_SLOT_COMP = 24, 28, 32, 36, 40, 44   # [3] / [3] / ... / [10]
DESC_LEN = 64
# Huffman lookup of one table in `tables` (int32): lut[512] = (code length << 8) | symbol for codes of <= 9 bits (0: longer),
# maxcode[18] (maxcode[l] = largest code of length l, -1 if none; maxcode[17] sentinel), valoff[18], vals[256]
LUT_BITS = 9
TAB_INTS = (1 << LUT_BITS) + 18 + 18 + 256
IMG_TAB_INTS = 6 * TAB_INTS + 3 * 64        # per scan component: DC table, AC table; then the 3 quantisation tables
# status bits (per image): the device decode declined the stream
ST_DATA, ST_RST, ST_END, ST_SYNC, ST_RANGE, ST_SIZE = 1, 2, 4, 8, 16, 32
_STATUS_TEXT = {ST_DATA: "corrupt entropy-coded data", ST_RST: "restart markers missing or out of sequence",
                ST_END: "no EOI marker after the scan (truncated file)",
                ST_SYNC: "Huffman decode did not converge within the pass limit",
                ST_RANGE: "coefficients outside the range where the 16-bit IDCT Pillow runs is exact",
                ST_SIZE: "entropy-coded data over 512 MB"}
MAX_SCAN_BYTES = 1 << 29   # bit offsets on the device are 32-bit

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
                   61, 54, 47, 55, 62, 63], dtype=np.int32)    # zigzag index -> natural index (jpeg_natural_order)


class JpegDecline(Exception):
    """The stream is outside what the device decoder handles.  `malformed` tells a broken header from a valid but
    unsupported file."""

    def __init__(self, reason: str, malformed: bool = False):
        super().__init__(reason)
        self.reason = reason
        self.malformed = malformed


@dataclass
class HuffTable:
    bits: Tuple[int, ...]          # counts of codes of length 1..16
    vals: bytes


@dataclass
class JpegInfo:
    width: int
    height: int
    comps: List[Tuple[int, int, int, int]]     # frame order: (id, h, v, quant table id)
    qtables: np.ndarray                        # [ncomp, 64] int32, natural order, the table each component uses
    restart_interval: int                      # MCUs per interval, 0 = none
    scan: List[Tuple[int, HuffTable, HuffTable]]   # scan order: (frame index, DC table, AC table)
    scan_data: int                             # offset of the first entropy-coded byte
    mode: str = ""                             # "L" or "RGB": what Image.open gives
    hmax: int = 1
    vmax: int = 1

    @property
    def ncomp(self):
        return len(self.comps)

    @property
    def single(self):
        return len(self.scan) == 1

    def geometry(self):
        """(mcus_x, mcus_y, blocks per MCU, [(frame comp, dy, dx) per MCU slot]) in libjpeg's terms."""
        if self.single:
            return (self.width + 7) // 8, (self.height + 7) // 8, 1, [(self.scan[0][0], 0, 0)]
        mx = -(-self.width // (8 * self.hmax))
        my = -(-self.height // (8 * self.vmax))
        slots = []
        for ci, _, _ in self.scan:
            _, h, v, _ = self.comps[ci]
            slots += [(ci, dy, dx) for dy in range(v) for dx in range(h)]
        return mx, my, len(slots), slots

    def plane_shape(self, ci):
        """(rows, cols) of component ci's IDCT output plane, padded to its block grid."""
        mx, my, _, _ = self.geometry()
        if self.single:
            return my * 8, mx * 8
        _, h, v, _ = self.comps[ci]
        return my * v * 8, mx * h * 8

    def n_intervals(self):
        mx, my, _, _ = self.geometry()
        total = mx * my
        return 1 if self.restart_interval == 0 else -(-total // self.restart_interval)


def _u16(data, i):
    if i + 2 > len(data):
        raise JpegDecline("truncated header", malformed=True)
    return (data[i] << 8) | data[i + 1]


def parse(data: bytes) -> JpegInfo:
    """Reads the markers of one JPEG byte string up to the first scan.  Raises `JpegDecline` for anything the device decoder
    does not handle, naming it."""
    data = bytes(data)
    if len(data) < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise JpegDecline("not a JPEG stream (no SOI marker)", malformed=True)
    i = 2
    qt = {}
    huff = {}
    sof = None
    restart = 0
    jfif = False
    adobe = None
    while True:
        if i >= len(data) or data[i] != 0xFF:
            raise JpegDecline("truncated header or garbage between markers", malformed=True)
        while i < len(data) and data[i] == 0xFF:       # fill bytes
            i += 1
        if i >= len(data):
            raise JpegDecline("truncated header", malformed=True)
        m = data[i]
        i += 1
        if m == 0xD8 or m == 0xD9 or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise JpegDecline(f"unexpected marker 0x{m:02X} before the scan", malformed=True)
        seglen = _u16(data, i)
        if seglen < 2 or i + seglen > len(data):
            raise JpegDecline("truncated header", malformed=True)
        seg = data[i + 2:i + seglen]
        i += seglen
        if m == 0xC0 or m == 0xC1:
            if sof is not None:
                raise JpegDecline("two frame headers", malformed=True)
            sof = seg
        elif m == 0xC2 or m == 0xC6 or m == 0xCA or m == 0xCE:
            raise JpegDecline("progressive JPEG" + (" with arithmetic coding" if m >= 0xCA else ""))
        elif m == 0xC3 or m == 0xC7 or m == 0xCB or m == 0xCF:
            raise JpegDecline("lossless JPEG")
        elif m == 0xC5:
            raise JpegDecline("hierarchical (differential) JPEG")
        elif m == 0xC9 or m == 0xCC:
            raise JpegDecline("arithmetic coding")
        elif m == 0xC4:
            j = 0
            while j < len(seg):
                tc, th = seg[j] >> 4, seg[j] & 15
                if tc > 1 or th > 3 or j + 17 > len(seg):
                    raise JpegDecline("malformed DHT segment", malformed=True)
                bits = tuple(seg[j + 1:j + 17])
                n = sum(bits)
                if n > 256 or j + 17 + n > len(seg):
                    raise JpegDecline("malformed DHT segment", malformed=True)
                huff[(tc, th)] = HuffTable(bits, bytes(seg[j + 17:j + 17 + n]))
                j += 17 + n
        elif m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                n = 128 if pq else 64
                if pq > 1 or tq > 3 or j + 1 + n > len(seg):
                    raise JpegDecline("malformed DQT segment", malformed=True)
                raw = seg[j + 1:j + 1 + n]
                zz = np.frombuffer(raw, dtype=">u2" if pq else np.uint8).astype(np.int32)
                nat = np.zeros(64, np.int32)
                nat[ZIGZAG] = zz
                qt[tq] = nat
                j += 1 + n
        elif m == 0xDD:
            if len(seg) != 2:
                raise JpegDecline("malformed DRI segment", malformed=True)
            restart = (seg[0] << 8) | seg[1]
        elif m == 0xE0:
            if len(seg) >= 14 and seg[:5] == b"JFIF\0":
                jfif = True
        elif m == 0xEE:
            if len(seg) >= 12 and seg[:5] == b"Adobe":
                adobe = seg[11]
        elif 0xE1 <= m <= 0xEF or m == 0xFE:
            pass
        elif m == 0xDA:
            break
        elif m == 0xDC:
            raise JpegDecline("DNL marker")
        else:
            raise JpegDecline(f"unsupported marker 0x{m:02X} before the scan", malformed=True)
    if sof is None:
        raise JpegDecline("scan before the frame header", malformed=True)
    if len(sof) < 6:
        raise JpegDecline("malformed SOF segment", malformed=True)
    prec, height, width, nf = sof[0], (sof[1] << 8) | sof[2], (sof[3] << 8) | sof[4], sof[5]
    if prec != 8:
        raise JpegDecline(f"{prec}-bit samples")
    if height == 0:
        raise JpegDecline("DNL marker (height 0 in the frame header)")
    if width == 0 or len(sof) != 6 + 3 * nf or nf == 0:
        raise JpegDecline("malformed SOF segment", malformed=True)
    comps = []
    for c in range(nf):
        cid, hv, tq = sof[6 + 3 * c], sof[7 + 3 * c], sof[8 + 3 * c]
        h, v = hv >> 4, hv & 15
        if not (1 <= h <= 4 and 1 <= v <= 4) or tq > 3:
            raise JpegDecline("malformed SOF segment", malformed=True)
        comps.append((cid, h, v, tq))
    if nf not in (1, 3):
        raise JpegDecline(f"{nf} components" + (" (CMYK or YCCK)" if nf == 4 else ""))
    if nf == 3:
        if jfif:
            rgb = False
        elif adobe is not None:
            rgb = adobe == 0
        else:
            rgb = [c[0] for c in comps] == [82, 71, 66]
        if rgb:
            raise JpegDecline("3 components stored as RGB (no YCbCr transform)")
        (_, h0, v0, _), (_, h1, v1, _), (_, h2, v2, _) = comps
        if (h1, v1, h2, v2) != (1, 1, 1, 1) or (h0, v0) not in ((1, 1), (2, 1), (2, 2)):
            raise JpegDecline(f"sampling layout {[(c[1], c[2]) for c in comps]} (supported: luma (1,1), (2,1) or (2,2), "
                              "chroma (1,1))")
    # SOS header (i points at its length field)
    i -= seglen
    sos_len = seglen
    if i + sos_len > len(data) or sos_len < 3:
        raise JpegDecline("truncated header", malformed=True)
    sos = data[i + 2:i + sos_len]
    ns = sos[0]
    if len(sos) != 4 + 2 * ns or ns == 0:
        raise JpegDecline("malformed SOS segment", malformed=True)
    if ns != nf:
        raise JpegDecline("multi-scan sequential JPEG (the first scan does not hold every component)")
    scan = []
    seen = set()
    for c in range(ns):
        cs, t = sos[1 + 2 * c], sos[2 + 2 * c]
        idx = [k for k, cc in enumerate(comps) if cc[0] == cs]
        if len(idx) != 1 or idx[0] in seen:
            raise JpegDecline("malformed SOS segment", malformed=True)
        seen.add(idx[0])
        td, ta = t >> 4, t & 15
        if (0, td) not in huff or (1, ta) not in huff:
            raise JpegDecline("Huffman table not defined before the scan")
        scan.append((idx[0], huff[(0, td)], huff[(1, ta)]))
    ss, se, ahal = sos[1 + 2 * ns], sos[2 + 2 * ns], sos[3 + 2 * ns]
    if ss != 0 or se != 63 or ahal != 0:
        raise JpegDecline("scan parameters are not sequential (Ss, Se, Ah, Al)")
    for c in comps:
        if c[3] not in qt:
            raise JpegDecline("quantisation table not defined before the scan", malformed=True)
    for _, dc, ac in scan:
        build_lookup(dc, is_dc=True)
        build_lookup(ac, is_dc=False)
    if len(data) - (i + sos_len) >= MAX_SCAN_BYTES:
        raise JpegDecline("entropy-coded data over 512 MB")
    info = JpegInfo(width=width, height=height, comps=comps, qtables=np.stack([qt[c[3]] for c in comps]),
                    restart_interval=restart, scan=scan, scan_data=i + sos_len, mode="L" if nf == 1 else "RGB",
                    hmax=max(c[1] for c in comps), vmax=max(c[2] for c in comps))
    return info


def build_lookup(t: HuffTable, is_dc: bool) -> np.ndarray:
    """Canonical Huffman code -> the int32 lookup form of `tables` (TAB_INTS).  Rejects tables libjpeg rejects
    (jpeg_make_d_derived_tbl): over-subscribed code lengths, DC symbols above 15."""
    out = np.zeros(TAB_INTS, np.int32)
    lut = out[:1 << LUT_BITS]
    maxcode = out[1 << LUT_BITS:(1 << LUT_BITS) + 18]
    valoff = out[(1 << LUT_BITS) + 18:(1 << LUT_BITS) + 36]
    vals = out[(1 << LUT_BITS) + 36:]
    if is_dc and any(v > 15 for v in t.vals):
        raise JpegDecline("DC Huffman table with a symbol above 15", malformed=True)
    vals[:len(t.vals)] = np.frombuffer(t.vals, np.uint8)
    code, k = 0, 0
    maxcode[:] = -1
    for length in range(1, 17):
        n = t.bits[length - 1]
        if n:
            valoff[length] = k - code
            for _ in range(n):
                if length <= LUT_BITS:
                    sh = LUT_BITS - length
                    lut[code << sh:(code + 1) << sh] = (length << 8) | t.vals[k]
                code += 1
                k += 1
            maxcode[length] = code - 1
        if code >= (1 << length):          # no code may be all ones
            raise JpegDecline("Huffman table with an impossible code (over-subscribed lengths)", malformed=True)
        code <<= 1
    maxcode[17] = 0x7FFFFFFF
    return out


def read_source(src) -> bytes:
    if isinstance(src, (bytes, bytearray, memoryview)):
        return bytes(src)
    with open(os.fspath(src), "rb") as f:
        return f.read()


# ---------------------------------------------------------------------------------------------------------------------
# device driver
# ---------------------------------------------------------------------------------------------------------------------
class _Plan:
    """Host-side layout of one batch: descriptors, tables and the buffer sizes, from the parsed headers alone."""

    def __init__(self, items: Sequence[Tuple[bytes, JpegInfo]], rgb: Sequence[bool]):
        n = len(items)
        self.desc = np.zeros((n, DESC_LEN), np.int64)
        self.tables = np.zeros((n, IMG_TAB_INTS), np.int32)
        streams = []
        so = co = io = sl = ch = bo = oo = po = 0
        self.shapes = []
        for b, ((data, info), want_rgb) in enumerate(zip(items, rgb)):
            d = self.desc[b]
            scan = data[info.scan_data:]
            L = len(scan)
            mx, my, bpm, slots = info.geometry()
            niv = info.n_intervals()
            nslots = niv + (L * 8) // SUBSEQ_BITS + 1
            nch = max(1, -(-L // CHUNK_BYTES))
            total = mx * my
            d[D_STREAM_OFF], d[D_STREAM_LEN], d[D_COMP_OFF] = so, L, co
            d[D_N_INTERVALS], d[D_IV_OFF], d[D_SLOT_OFF], d[D_N_SLOTS] = niv, io, sl, nslots
            d[D_CHUNK_OFF], d[D_N_CHUNKS], d[D_BLOCK_OFF], d[D_N_BLOCKS] = ch, nch, bo, total * bpm
            d[D_MCUS_PER_IV] = info.restart_interval if info.restart_interval else total
            d[D_BPM], d[D_MCUS_X], d[D_MCUS_Y], d[D_TOTAL_MCUS] = bpm, mx, my, total
            d[D_WIDTH], d[D_HEIGHT], d[D_NCOMP], d[D_SINGLE] = info.width, info.height, info.ncomp, int(info.single)
            ch_out = 3 if (info.ncomp == 3 or want_rgb) else 1
            d[D_OUT_OFF], d[D_OUT_CH] = oo, ch_out
            for ci in range(info.ncomp):
                ph, pw = info.plane_shape(ci)
                d[D_PLANE_OFF + ci], d[D_PLANE_PITCH + ci], d[D_PLANE_H + ci] = po, pw, ph
                d[D_HSAMP + ci], d[D_VSAMP + ci] = info.comps[ci][1], info.comps[ci][2]
                po += ph * pw
            for s, (ci, dy, dx) in enumerate(slots):
                d[D_SLOT_COMP + s] = ci | (dy << 4) | (dx << 8) | ([k for k, sc in enumerate(info.scan) if sc[0] == ci][0] << 12)
            for k, (ci, dc, ac) in enumerate(info.scan):
                self.tables[b, (2 * k) * TAB_INTS:(2 * k + 1) * TAB_INTS] = build_lookup(dc, True)
                self.tables[b, (2 * k + 1) * TAB_INTS:(2 * k + 2) * TAB_INTS] = build_lookup(ac, False)
            self.tables[b, 6 * TAB_INTS:6 * TAB_INTS + 64 * info.ncomp] = info.qtables.reshape(-1)
            streams.append(scan)
            pad = (-L) % 16 + STREAM_PAD
            streams.append(bytes(pad))
            so += L + pad
            co += L + STREAM_PAD
            io += niv + 1
            sl += nslots
            ch += nch
            bo += total * bpm
            oo += info.width * info.height * ch_out
            self.shapes.append((info.height, info.width, ch_out))
        self.stream = np.frombuffer(bytearray(b"".join(streams)), np.uint8)
        self.sizes = dict(comp=co, intervals=io, slots=sl, chunks=ch, blocks=bo, out=oo, planes=po)


def _launch(plan: _Plan, device, pixels=True):
    """Runs the decode of one batch on the current stream.  Returns (out uint8 flat, coef int16 [blocks, 64], state int32
    [batch, 8], flags int32 [8])."""
    import torch
    from . import cabi
    dev = torch.device(device)
    sz = plan.sizes
    n = plan.desc.shape[0]
    u8 = dict(dtype=torch.uint8, device=dev)
    i32 = dict(dtype=torch.int32, device=dev)
    stream = torch.from_numpy(plan.stream).to(dev)
    desc = torch.from_numpy(plan.desc).to(dev)
    tables = torch.from_numpy(plan.tables).to(dev)
    comp = torch.empty(sz["comp"], **u8)
    chunks = torch.empty(2 * sz["chunks"], **i32)
    istart = torch.empty(sz["intervals"], **i32)
    exits = torch.empty(3 * sz["slots"], dtype=torch.int64, device=dev)
    counts = torch.empty(2 * sz["slots"], **i32)
    coef = torch.zeros(sz["blocks"], 64, dtype=torch.int16, device=dev)
    state = torch.empty(n, 8, **i32)
    flags = torch.zeros(8, **i32)
    kw = dict(batch=n, stream=stream, desc=desc, tables=tables, comp=comp, chunks=chunks, istart=istart, exits=exits,
              counts=counts, coef=coef, state=state, flags=flags, max_chunks=int(plan.desc[:, D_N_CHUNKS].max()),
              max_intervals=int(plan.desc[:, D_N_INTERVALS].max()), total_slots=sz["slots"], total_blocks=sz["blocks"])
    with torch.cuda.device(dev):
        cabi.call("romab200_jpeg_entropy", "rb_jpeg_args", **kw)
        out = None
        if pixels:
            planes = torch.empty(max(sz["planes"], 1), **u8)
            out = torch.empty(max(sz["out"], 1), **u8)
            max_pix = int((plan.desc[:, D_WIDTH] * plan.desc[:, D_HEIGHT]).max())
            cabi.call("romab200_jpeg_pixels", "rb_jpeg_args", **kw, planes=planes, out=out, max_pixels=max_pix)
            del planes
    return out, coef, state, flags


def decode_coefficients(data: bytes, device="cuda"):
    """Entropy stage alone for one stream: (per frame component int16 [by, bx, 64] natural-order blocks with DC resolved,
    status word, sync passes)."""
    info = parse(data)
    plan = _Plan([(data, info)], [False])
    _, coef, state, flags = _launch(plan, device, pixels=False)
    coef = coef.cpu().numpy()
    mx, my, bpm, slots = info.geometry()
    blocks = [np.zeros((info.plane_shape(ci)[0] // 8, info.plane_shape(ci)[1] // 8, 64), np.int16) for ci in range(info.ncomp)]
    if info.single:
        blocks[slots[0][0]][:] = coef.reshape(my, mx, 64)
    else:
        c = coef.reshape(my, mx, bpm, 64)
        for s, (ci, dy, dx) in enumerate(slots):
            h, v = info.comps[ci][1], info.comps[ci][2]
            blocks[ci][dy::v, dx::h] = c[:, :, s]
    return blocks, int(state[0, 1]), int(flags[3])


def status_text(code: int) -> str:
    return "; ".join(t for bit, t in _STATUS_TEXT.items() if code & bit) or "ok"


def decode_device(datas: Sequence[bytes], infos: Sequence[JpegInfo], device, rgb: Sequence[bool]):
    """Decodes already-parsed streams in one launch set.  Returns a list with, per image, a uint8 [H, W, C] tensor on
    `device` or the status text of a stream the device decoder rejected, and the number of sync passes the batch took."""
    import torch
    plan = _Plan(list(zip(datas, infos)), rgb)
    out, _, state, flags = _launch(plan, device)
    host = torch.cat((state[:, 1], flags[3:4])).cpu().tolist()        # one device -> host read per batch
    st, passes = host[:-1], host[-1]
    res = []
    for b, (h, w, c) in enumerate(plan.shapes):
        if st[b]:
            res.append(status_text(st[b]))
            continue
        o = int(plan.desc[b, D_OUT_OFF])
        res.append(out[o:o + h * w * c].view(h, w, c))
    return res, passes


def decode_jpeg(sources, device="cuda", mode=None):
    """Decodes JPEG files or byte strings on the device, all in one launch set.

    Each result is a uint8 [H, W, C] tensor on `device`, byte-identical to `np.asarray(Image.open(src))` ("L" -> C = 1,
    YCbCr -> C = 3), or to `np.asarray(Image.open(src).convert("RGB"))` with `mode="RGB"`.  Raises NotImplementedError
    naming the feature for a file outside the supported subset, ValueError for a stream the decoder rejects."""
    if mode not in (None, "RGB"):
        raise ValueError(f"decode_jpeg: mode must be None or 'RGB', got {mode!r}")
    if isinstance(sources, (str, bytes, bytearray, os.PathLike)):
        sources = [sources]
    datas, infos = [], []
    for src in sources:
        data = read_source(src)
        try:
            info = parse(data)
        except JpegDecline as e:
            if e.malformed:
                raise ValueError(f"decode_jpeg: {e.reason}") from None
            raise NotImplementedError(f"decode_jpeg: {e.reason}") from None
        datas.append(data)
        infos.append(info)
    if not datas:
        return []
    res, _ = decode_device(datas, infos, device, [mode == "RGB"] * len(datas))
    for r in res:
        if isinstance(r, str):
            raise ValueError(f"decode_jpeg: the device decoder rejected the stream: {r}")
    return res


def probe(path) -> Optional[Tuple[bytes, JpegInfo]]:
    """(bytes, header) of a file the device decoder handles, None otherwise (any other format, or a declined JPEG)."""
    try:
        data = read_source(path)
        return data, parse(data)
    except (JpegDecline, OSError):
        return None
