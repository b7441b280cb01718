"""Host-side input handling of `match()`: type checks and PIL -> normalised tensor.

Mirrors `_check_input` (`romatch/models/matcher.py:530-547`), `check_rgb` / `check_not_i16`
(`romatch/utils/utils.py:655-661`) and `get_tuple_transform_ops(resize, normalize=True)`
(`utils.py:164-173`: PIL bicubic resize -> /255 -> ImageNet mean/std).  The reference does the
resize on the host; here `DevicePreprocessor` uploads the raw RGB bytes once and runs Pillow's 8-bit
bicubic resampling + the normalisation as CUDA kernels (`csrc/preprocess.cu`, SURVEY §8f rank 3),
bit-exact with `pil_to_normalized`, which stays as the host statement of the same transform (tests
compare the two).
"""
from __future__ import annotations

import os

import ctypes

import numpy as np
import torch
from PIL import Image

from . import cabi, jpeg

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def check_input(im_input):
    """Path -> RGB PIL; PIL must already be RGB; tensors must be [B,3,H,W] with H,W % 14 == 0."""
    if isinstance(im_input, (str, os.PathLike)):
        im = Image.open(im_input)
        if im.mode == "I;16":
            raise NotImplementedError("Can't handle 16 bit images")
        return im.convert("RGB")
    if isinstance(im_input, Image.Image):
        if im_input.mode != "RGB":
            raise NotImplementedError("Can't handle non-RGB images")
        return im_input
    assert isinstance(im_input, torch.Tensor), "im_input must be a string, path, or PIL image"
    B, C, H, W = im_input.shape
    assert C == 3, "im_input must be a RGB image"
    assert H % 14 == 0, "im_input must be a multiple of 14"
    assert W % 14 == 0, "im_input must be a multiple of 14"
    return im_input


class DeviceImage:
    """An input file decoded on the device: `raw` is uint8 [H, W, C], the bytes Pillow would give."""

    def __init__(self, raw: torch.Tensor):
        self.raw = raw


def open_inputs(inputs, device, rgb: bool = True):
    """Inputs of one `match` call.  Paths are opened with `Image.open` (lazy: the I;16 and decompression-bomb checks and the
    format detection stay Pillow's); the JPEG files among them that `jpeg.parse` accepts are decoded on the device in one
    launch set and come back as `DeviceImage`.  Every other path, and a JPEG the device decoder rejects, takes the host route
    unchanged: `Image.open(p).convert("RGB")` when `rgb`, else the opened image.  Non-path inputs go through `check_input`
    when `rgb`, else are returned as they are."""
    out, pending = [], []
    for x in inputs:
        if isinstance(x, (str, os.PathLike)):
            im = Image.open(x)
            if rgb and im.mode == "I;16":
                raise NotImplementedError("Can't handle 16 bit images")
            found = jpeg.probe(x) if im.format == "JPEG" else None
            if found is not None:
                pending.append((len(out), found, im))
                out.append(None)
                continue
            out.append(im.convert("RGB") if rgb else im)
        else:
            out.append(check_input(x) if rgb else x)
    if pending:
        res, _ = jpeg.decode_device([f[0] for _, f, _ in pending], [f[1] for _, f, _ in pending], device, [rgb] * len(pending))
        for (k, _, im), r in zip(pending, res):
            if isinstance(r, str):
                out[k] = im.convert("RGB") if rgb else im
            else:
                im.close()              # decoded on the device: release the file Image.open keeps open
                out[k] = DeviceImage(r)
    return out


def pil_to_normalized(im: Image.Image, size_hw) -> torch.Tensor:
    """Bicubic PIL resize to (h, w), scale to [0,1], ImageNet-normalise -> float32 [3,h,w]."""
    h, w = size_hw
    im = im.resize((w, h), Image.BICUBIC)           # torchvision Resize on PIL == PIL.resize
    arr = np.asarray(im, dtype=np.float32).transpose(2, 0, 1) / 255.0
    t = torch.from_numpy(np.ascontiguousarray(arr))
    mean = torch.tensor(IMAGENET_MEAN, dtype=torch.float32)[:, None, None]
    std = torch.tensor(IMAGENET_STD, dtype=torch.float32)[:, None, None]
    return (t[:3] - mean) / std


def resample_coeffs(in_size: int, out_size: int):
    """Pillow's bicubic weight table of one axis from the library's host routine: (ksize, bounds [out,2], kk [out,ksize]) int32."""
    lib = cabi.load_library()
    args = cabi.STRUCTS["rb_resample_coeffs_args"]()
    ksize = ctypes.c_int32(0)
    args.in_size, args.out_size = int(in_size), int(out_size)
    args.ksize = ctypes.cast(ctypes.pointer(ksize), ctypes.c_void_p)
    if lib.romab200_resample_coeffs(ctypes.byref(args), None) != 0:
        raise RuntimeError(f"romab200_resample_coeffs failed: {lib.romab200_last_error().decode()}")
    bounds = np.zeros((out_size, 2), dtype=np.int32)
    kk = np.zeros((out_size, ksize.value), dtype=np.int32)
    args.bounds, args.kk = bounds.ctypes.data, kk.ctypes.data
    if lib.romab200_resample_coeffs(ctypes.byref(args), None) != 0:
        raise RuntimeError(f"romab200_resample_coeffs failed: {lib.romab200_last_error().decode()}")
    return ksize.value, bounds, kk


class DevicePreprocessor:
    """PIL image -> normalised fp32 [3,h,w] on `device`: one H2D copy of the raw RGB bytes per image, then
    `romab200_preprocess_rgb8` per target resolution (the coarse and the upsample resolution share the upload)."""

    def __init__(self, device):
        self.device = torch.device(device)
        self._tables = {}      # (in, out) -> (ksize, bounds_dev, kk_dev)
        self._tmp = None

    def _table(self, n_in, n_out):
        key = (int(n_in), int(n_out))
        t = self._tables.get(key)
        if t is None:
            ksize, bounds, kk = resample_coeffs(*key)
            t = (ksize, torch.from_numpy(bounds).to(self.device), torch.from_numpy(kk).to(self.device))
            if len(self._tables) > 256:
                self._tables.clear()
            self._tables[key] = t
        return t

    def upload(self, im: Image.Image) -> torch.Tensor:
        """RGB PIL image -> uint8 [H, W, 3] on the device."""
        if im.mode != "RGB":
            raise NotImplementedError("Can't handle non-RGB images")
        arr = np.asarray(im, dtype=np.uint8)
        return torch.from_numpy(np.ascontiguousarray(arr)).to(self.device, non_blocking=False)

    def resize_normalize(self, raw: torch.Tensor, size_hw, out: torch.Tensor = None, out_u8: torch.Tensor = None) -> torch.Tensor:
        """uint8 [H, W, 3] device image -> fp32 [3, h, w] (written into `out` when given)."""
        assert raw.dtype == torch.uint8 and raw.dim() == 3 and raw.shape[2] == 3 and raw.is_contiguous() and raw.is_cuda
        H, W = int(raw.shape[0]), int(raw.shape[1])
        h, w = int(size_hw[0]), int(size_hw[1])
        if out is None:
            out = torch.empty(3, h, w, dtype=torch.float32, device=raw.device)
        assert out.shape == (3, h, w) and out.dtype == torch.float32 and out.is_contiguous()
        kw = dict(ld_in=W * 3, in_h=H, in_w=W, out_h=h, out_w=w, out=out, out_u8=out_u8,
                  mean=list(IMAGENET_MEAN), std=list(IMAGENET_STD))
        kw["in"] = raw
        if w != W:
            ks, bd, kk = self._table(W, w)
            need = H * w * 3
            if self._tmp is None or self._tmp.numel() < need or self._tmp.device != raw.device:
                self._tmp = torch.empty(need, dtype=torch.uint8, device=raw.device)
            kw.update(bounds_x=bd, kk_x=kk, ksize_x=ks, tmp=self._tmp)
        if h != H:
            ks, bd, kk = self._table(H, h)
            kw.update(bounds_y=bd, kk_y=kk, ksize_y=ks)
        with torch.cuda.device(raw.device):
            cabi.call("romab200_preprocess_rgb8", "rb_preprocess_args", **kw)
        return out
