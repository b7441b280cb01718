"""`TinyRoMa`: the reference's tiny matcher (`romatch/models/tiny.py:30-304`, XFeat backbone) on hand-written sm_90a kernels.

Public surface and arithmetic follow the reference's inference path: fp32 throughout, the BatchNorms in eval mode (folded into
the preceding convolution at construction), `match()` always in eval mode as the reference forces it.  The XFeat backbone is not
part of this package: its layer structure is read from the module the caller passes (`walk_layers`) and its weights from the
`xfeat.0.*` entries of the checkpoint, so any XFeat-shaped network made of the supported layers runs.

Kernels (`csrc/tiny.cu`, include/romab200.h): direct fp32 convolutions for the backbone and the matcher heads, the channel
mean + InstanceNorm, AvgPool2d(4), the fused correlation / argmax / soft-argmax embedding that never materialises the
[h1*w1, h0*w0] correlation volume, the warp-and-concat prologue of the heads and the match() epilogue; the bilinear resizes
are `romab200_bilinear_resize`.  `match()` is captured as one CUDA graph per input shape from its second call on.

Stated differences from the reference:
  * `forward` always runs the inference path (eval BatchNorm, sub-sampled softmax unless `exact_softmax`); the reference's
    training-mode branch is not built;
  * PIL inputs must be of mode "RGB" or "L" (others raise NotImplementedError);
  * images smaller than 32 pixels on a side raise ValueError (the reference fails inside its backbone).
"""
from __future__ import annotations

import math
import os
from pathlib import Path

import numpy as np
import torch
import torch.nn as nn
from PIL import Image

from . import cabi
from .cabi import call
from .cache import BufferArena, GraphCache
from .preprocess import DeviceImage, open_inputs
from .matcher import RegressionMatcher
from .packing import fold_bn
from . import sampling
from .sampling import kde, sample_device

XFEAT_PARTS = ("norm", "skip1", "block1", "block2", "block3", "block4", "block5", "block_fusion")
XFEAT_DELETED = ("heatmap_head", "keypoint_head", "fine_matcher")     # TinyRoMa.__init__ deletes them (tiny.py:41)
HEADS = (("coarse_matcher", 64 + 64 + 2, 256), ("fine_matcher", 24 + 24 + 2, 64))   # (name, input channels, width), tiny.py:47-61
HEAD_DEPTH = 4


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def walk_layers(module: nn.Module, path: str):
    """The layer list of one XFeat part: dicts of kind "conv" (with the BatchNorm / ReLU that follow it folded in), "avgpool4" or
    "instnorm".  Descends into nn.Sequential and into single-child wrappers without parameters of their own (a layer whose
    forward is `self.layer(x)`); any other module raises NotImplementedError naming its path."""
    ops = []

    def unsupported(p, m, why=""):
        raise NotImplementedError(f"TinyRoMa backbone: unsupported layer {p} ({type(m).__name__}{': ' + why if why else ''})")

    def visit(m, p):
        if isinstance(m, nn.Sequential):
            for name, child in m.named_children():
                visit(child, f"{p}.{name}")
        elif isinstance(m, nn.Conv2d):
            k, s = _pair(m.kernel_size), _pair(m.stride)
            if m.groups != 1 or _pair(m.dilation) != (1, 1) or k not in ((1, 1), (3, 3)) or s not in ((1, 1), (2, 2)):
                unsupported(p, m, f"kernel {k}, stride {s}, groups {m.groups}, dilation {m.dilation}")
            if m.padding_mode != "zeros" or isinstance(m.padding, str) or _pair(m.padding) != (k[0] // 2, k[0] // 2):
                unsupported(p, m, f"padding {m.padding!r} ({m.padding_mode})")
            ops.append(dict(kind="conv", path=p, k=k[0], stride=s[0], cin=m.in_channels, cout=m.out_channels, bias=m.bias is not None,
                            bn=None, bn_eps=None, relu=False))
        elif isinstance(m, nn.BatchNorm2d):
            if not ops or ops[-1]["kind"] != "conv" or ops[-1]["bn"] is not None or ops[-1]["relu"]:
                unsupported(p, m, "a BatchNorm2d is supported directly after a Conv2d only")
            if not m.track_running_stats:
                unsupported(p, m, "no running statistics")
            ops[-1]["bn"], ops[-1]["bn_eps"] = p, m.eps
        elif isinstance(m, nn.ReLU):
            if not ops or ops[-1]["kind"] != "conv" or ops[-1]["relu"]:
                unsupported(p, m, "a ReLU is supported after a Conv2d (+ BatchNorm2d) only")
            ops[-1]["relu"] = True
        elif isinstance(m, nn.AvgPool2d):
            if _pair(m.kernel_size) != (4, 4) or _pair(m.stride or m.kernel_size) != (4, 4) or _pair(m.padding) != (0, 0) or m.ceil_mode:
                unsupported(p, m, "AvgPool2d(4, 4) only")
            ops.append(dict(kind="avgpool4", path=p))
        elif isinstance(m, nn.InstanceNorm2d):
            if m.num_features != 1 or m.affine or m.track_running_stats:
                unsupported(p, m, "InstanceNorm2d(1) without affine or running statistics only")
            ops.append(dict(kind="instnorm", path=p, eps=m.eps))
        elif isinstance(m, nn.Identity):
            pass
        else:
            children = list(m.named_children())
            if len(children) == 1 and not list(m.parameters(recurse=False)) and not list(m.buffers(recurse=False)):
                visit(children[0][1], f"{p}.{children[0][0]}")
            else:
                unsupported(p, m)

    visit(module, path)
    return ops


def xfeat_plan(xfeat: nn.Module):
    """{part: layer list} for the parts TinyRoMa.forward_single uses (tiny.py:81-97), with the placement rules checked."""
    plan = {}
    for part in XFEAT_PARTS:
        if not hasattr(xfeat, part):
            raise NotImplementedError(f"TinyRoMa backbone: the XFeat module has no `{part}`")
        plan[part] = walk_layers(getattr(xfeat, part), part)
    if any(op["kind"] != "instnorm" for op in plan["norm"]) or len(plan["norm"]) > 1:
        raise NotImplementedError("TinyRoMa backbone: `norm` must be an InstanceNorm2d(1) (or an identity)")
    for part in XFEAT_PARTS[1:]:
        for op in plan[part]:
            if op["kind"] == "instnorm":
                raise NotImplementedError(f"TinyRoMa backbone: unsupported layer {op['path']} (InstanceNorm2d outside `norm`)")
    if not plan["skip1"] or plan["skip1"][-1]["kind"] != "conv":
        raise NotImplementedError("TinyRoMa backbone: `skip1` must end with a Conv2d (its output is added to block1's)")
    return plan


def expected_state_dict_shapes(xfeat: nn.Module):
    """{key: shape} that `TinyRoMa(xfeat, freeze_xfeat=False).load_state_dict` expects (roma_models.py:21-29)."""
    want = {f"xfeat.0.{k}": tuple(v.shape) for k, v in xfeat.state_dict().items() if k.split(".")[0] not in XFEAT_DELETED}
    for name, cin, c in HEADS:
        for i in range(HEAD_DEPTH):
            want[f"{name}.{i}.layer.0.weight"] = (c, cin if i == 0 else c, 3, 3)
            want[f"{name}.{i}.layer.1.running_mean"] = (c,)
            want[f"{name}.{i}.layer.1.running_var"] = (c,)
            want[f"{name}.{i}.layer.1.num_batches_tracked"] = ()
        want[f"{name}.{HEAD_DEPTH}.weight"] = (3, c, 1, 1)
        want[f"{name}.{HEAD_DEPTH}.bias"] = (3,)
    return want


def check_state_dict(weights, xfeat):
    """Strict key and shape check of a TinyRoMa checkpoint against what the reference would load for this `xfeat`."""
    want = expected_state_dict_shapes(xfeat)
    missing = sorted(k for k in want if k not in weights)
    unexpected = sorted(k for k in weights if k not in want)
    if missing or unexpected:
        raise RuntimeError(f"Error(s) in loading state_dict for TinyRoMa: missing keys {missing[:6]} ({len(missing)}), "
                           f"unexpected keys {unexpected[:6]} ({len(unexpected)})")
    for k, shape in want.items():
        if tuple(weights[k].shape) != shape:
            raise RuntimeError(f"size mismatch for {k}: {tuple(weights[k].shape)} vs {shape}")


def _pad4(n):
    return (n + 3) // 4 * 4


def pack_conv(sd, path, op, device, cin_pad=None):
    """Conv (+ folded BN) -> the [k*k*cin, ldw] tap-major weight of `romab200_tiny_conv` and its fp32 bias (or None)."""
    w = sd[f"{path}.weight"].float()
    cout, cin = w.shape[:2]
    b = sd[f"{path}.bias"].float() if op["bias"] else torch.zeros(cout)
    if op["bn"] is not None:
        w, b = fold_bn(w, b, sd, op["bn_path"], eps=op["bn_eps"])
    cp = cin_pad or cin
    wt = torch.zeros(op["k"], op["k"], cp, _pad4(cout))
    wt[:, :, :cin, :cout] = w.permute(2, 3, 1, 0)
    has_bias = op["bias"] or op["bn"] is not None
    return dict(kind="conv", w=wt.reshape(-1, _pad4(cout)).contiguous().to(device), b=b.contiguous().to(device) if has_bias else None,
                k=op["k"], stride=op["stride"], cin=cp, cout=cout, relu=op["relu"], path=op["path"])


class TinyRoMa:
    """TinyRoMa inference on the H100 (tiny.py:30-304): `match`, `match_from_path`, `forward`, `sample`, the geometry helpers."""

    def __init__(self, xfeat: nn.Module, weights, device, sample_mode="threshold_balanced", symmetric=False, exact_softmax=False):
        self._device = torch.device(device)
        if self._device.type != "cuda":
            raise RuntimeError(f"roma_b200 runs on a CUDA device only (there is no CPU fallback); got device={device!r}")
        cabi.load_library()
        sd = {k: v.detach().cpu() for k, v in weights.items()}
        check_state_dict(sd, xfeat)
        self.plan = xfeat_plan(xfeat)
        self.sample_mode = sample_mode
        self.sample_thresh = 0.05
        self.symmetric = symmetric
        self.exact_softmax = exact_softmax
        self.training = False
        self.use_cuda_graph = True
        self.arena = BufferArena(self._device)
        self._graphs, self._sample_graphs = GraphCache(), GraphCache()
        with torch.cuda.device(self._device):
            xsd = {k[len("xfeat.0."):]: v for k, v in sd.items() if k.startswith("xfeat.0.")}
            self.norm = self.plan["norm"][0] if self.plan["norm"] else None
            self.layers = {part: [self._pack(xsd, op) for op in self.plan[part]] for part in XFEAT_PARTS[1:]}
            self.heads = {}
            for name, cin, c in HEADS:
                layers = []
                for i in range(HEAD_DEPTH + 1):
                    last = i == HEAD_DEPTH
                    op = dict(kind="conv", path=f"{name}.{i}" + ("" if last else ".layer.0"), k=1 if last else 3, stride=1, bias=last,
                              bn=None if last else f"{name}.{i}.layer.1", bn_path=f"{name}.{i}.layer.1", bn_eps=1e-5, relu=not last)
                    layers.append(pack_conv(sd, op["path"], op, self._device, cin_pad=_pad4(cin) if i == 0 else None))
                self.heads[name] = layers

    def _pack(self, xsd, op):
        if op["kind"] != "conv":
            return dict(op)
        op = dict(op, bn_path=op["bn"])
        return pack_conv(xsd, op["path"], op, self._device)

    # ---- nn.Module-ish conveniences -------------------------------------------------------------------
    @property
    def device(self):
        return self._device

    def train(self, mode: bool = True):
        self.training = False       # inference only; match() forces eval mode like the reference (tiny.py:206)
        return self

    def eval(self):
        return self.train(False)

    def to(self, *args, **kwargs):
        return self

    def free_buffers(self):
        """Release every cached activation buffer and the CUDA graphs recorded over them."""
        self._graphs.clear()
        self._sample_graphs.clear()
        self.arena.free()

    # ---- buffers and constants --------------------------------------------------------------------------
    def _b(self, name, shape):
        return self.arena.buf(name, shape, torch.float32, zero=True)     # zero: pad channels must read as 0

    def _linspace(self, lo, n):
        """torch.linspace(-1 + lo, 1 - lo, n) evaluated on the host like the reference, then uploaded."""
        return self.arena.const(("lin", lo, n), lambda: torch.linspace(-1 + lo, 1 - lo, n))

    # ---- device pipeline ------------------------------------------------------------------------------
    def _conv(self, L, x, n, h, w, c, out_name, R=None, col_scale=None):
        if c != L["cin"]:
            raise ValueError(f"TinyRoMa: layer {L['path']} expects {L['cin']} input channels, the map has {c}")
        ho, wo = (h - 1) // L["stride"] + 1, (w - 1) // L["stride"] + 1
        out = self._b(out_name, (n, ho, wo, L["cout"]))
        if R is not None and R.shape != out.shape:
            raise ValueError(f"TinyRoMa: residual of {L['path']} has shape {tuple(R.shape)}, the layer writes {tuple(out.shape)}")
        call("romab200_tiny_conv", "rb_tiny_conv_args", **{"in": x}, out=out, weight=L["w"], bias=L["b"], col_scale=col_scale, R=R,
             ldi=c, ldo=L["cout"], ldw=L["w"].shape[1], ldr=L["cout"], batch=n, hi=h, wi=w, ho=ho, wo=wo, cin=c, cout=L["cout"],
             ksize=L["k"], stride=L["stride"], relu=int(L["relu"]))
        return out, ho, wo, L["cout"]

    def _run_part(self, part, x, n, h, w, c, tag, residual=None):
        layers = self.layers[part]
        for i, L in enumerate(layers):
            name = f"{tag}.{L['path']}"
            if L["kind"] == "avgpool4":
                out = self._b(name, (n, h // 4, w // 4, c))
                call("romab200_tiny_avgpool4", "rb_tiny_avgpool_args", **{"in": x}, out=out, batch=n, hi=h, wi=w, c=c)
                x, h, w = out, h // 4, w // 4
            else:
                x, h, w, c = self._conv(L, x, n, h, w, c, name, R=residual if i == len(layers) - 1 else None)
        return x, h, w, c

    def _backbone(self, img, tag):
        """forward_single (tiny.py:81-100): NCHW image batch (sizes multiples of 32) -> (x2, feats) channels-last."""
        n, C, H, W = img.shape
        gray = self._b(f"{tag}.gray", (n, H, W, 1))
        call("romab200_tiny_gray", "rb_tiny_gray_args", **{"in": img}, out=gray, batch=n, channels=C, h=H, w=W,
             instance_norm=int(self.norm is not None), eps=float(self.norm["eps"]) if self.norm else 0.0)
        x1, h1, w1, c1 = self._run_part("block1", gray, n, H, W, 1, tag)
        s, hs, ws, cs = self._run_part("skip1", gray, n, H, W, 1, tag, residual=x1)        # x1 + skip1(x)
        x2, h2, w2, c2 = self._run_part("block2", s, n, hs, ws, cs, tag)
        x3, h3, w3, c3 = self._run_part("block3", x2, n, h2, w2, c2, tag)
        x4, h4, w4, c4 = self._run_part("block4", x3, n, h3, w3, c3, tag)
        x5, h5, w5, c5 = self._run_part("block5", x4, n, h4, w4, c4, tag)
        if not c3 == c4 == c5:
            raise ValueError(f"TinyRoMa: block3/4/5 channel counts {c3}/{c4}/{c5} cannot be summed")
        up4, up5, fsum = (self._b(f"{tag}.{k}", (n, h3, w3, c3)) for k in ("up4", "up5", "sum345"))
        call("romab200_bilinear_resize", "rb_resize_args", **{"in": x4}, out=up4, batch=n, hi=h4, wi=w4, ho=h3, wo=w3, c=c3)
        call("romab200_bilinear_resize", "rb_resize_args", **{"in": x5}, out=up5, batch=n, hi=h5, wi=w5, ho=h3, wo=w3, c=c3)
        call("romab200_tiny_add3", "rb_tiny_add3_args", a=x3, b=up4, c=up5, out=fsum, n=fsum.numel())
        feats, hf, wf, cf = self._run_part("block_fusion", fsum, n, h3, w3, c3, tag)
        return x2, feats

    def _preprocess(self, im, name):
        """Bilinear resize to multiples of 32 (preprocess_tensor, tiny.py:72-79), the C-channel image before the channel mean."""
        b, c, H, W = im.shape
        Hr, Wr = H // 32 * 32, W // 32 * 32
        out = self._b(name, (b, c, Hr, Wr))
        call("romab200_bilinear_resize", "rb_resize_args", **{"in": im}, out=out, batch=b * c, hi=H, wi=W, ho=Hr, wo=Wr, c=1)
        return out

    def _head(self, name, f0, f1, state, tag):
        """cat(f0, grid_sample(f1, flow), flow) -> 4 x BasicLayer -> 1x1 conv, whose epilogue adds delta * to_normalized to
        `state` (tiny.py:205-215)."""
        B, h0, w0, c = f0.shape
        _, h1, w1, _ = f1.shape
        L0 = self.heads[name][0]
        cat = self._b(f"{tag}.{name}.cat", (B, h0, w0, L0["cin"]))
        call("romab200_tiny_warp_concat", "rb_tiny_warp_concat_args", f0=f0, f1=f1, state=state, out=cat, ldf0=c, ldf1=c, lds=3,
             ldo=L0["cin"], batch=B, h0=h0, w0=w0, h1=h1, w1=w1, c=c)
        if 2 * c + 2 > L0["cin"]:
            raise ValueError(f"TinyRoMa: {name} expects {L0['cin']} input channels, the features give {2 * c + 2}")
        x, h, w, cc = cat, h0, w0, L0["cin"]
        for i, L in enumerate(self.heads[name]):
            last = i == len(self.heads[name]) - 1
            x, h, w, cc = self._conv(L, x, B, h, w, cc, f"{tag}.{name}.{i}", R=state if last else None,
                                     col_scale=self._to_normalized if last else None)
        return x

    def _forward_device(self, im0, im1, exact):
        """Whole forward pass (tiny.py:268-304) on the current stream, no host sync: -> (state8, state4) [B,h,w,3]."""
        B = im0.shape[0]
        p0 = self._preprocess(im0, "pre0")
        p1 = self._preprocess(im1, "pre1")
        H1, W1 = p1.shape[-2:]
        if min(p0.shape[-2:]) < 32 or min(H1, W1) < 32:
            raise ValueError("TinyRoMa needs images of at least 32 x 32 pixels")
        self._to_normalized = self.arena.const(("to_normalized", H1, W1), lambda: torch.tensor((2 / W1, 2 / H1, 1)))
        if p0.shape[1:] == p1.shape[1:]:
            both = self._b("pre01", (2 * B,) + tuple(p0.shape[1:]))
            both[:B].copy_(p0)
            both[B:].copy_(p1)
            x2, feats = self._backbone(both, "ab")
            x2_0, x2_1, f0, f1 = x2[:B], x2[B:], feats[:B], feats[B:]
        else:
            x2_0, f0 = self._backbone(p0, "a")
            x2_1, f1 = self._backbone(p1, "b")
        _, h0, w0, c = f0.shape
        _, hc1, wc1, _ = f1.shape
        state0 = self._b("state0", (B, h0, w0, 3))
        call("romab200_tiny_pos_embed", "rb_tiny_pos_embed_args", f0=f0, f1=f1, state=state0, batch=B, h0=h0, w0=w0, h1=hc1, w1=wc1,
             c=c, scale=math.sqrt(c), exact=int(exact), grid_x=self._linspace(1 / wc1, wc1), grid_y=self._linspace(1 / hc1, hc1),
             grid_lr_x=self._linspace(4 / wc1, wc1 // 4), grid_lr_y=self._linspace(4 / hc1, hc1 // 4))
        state8 = self._head("coarse_matcher", f0, f1, state0, "s8")
        _, hf, wf, _ = x2_0.shape
        up = self._b("state8_up", (B, hf, wf, 3))
        call("romab200_bilinear_resize", "rb_resize_args", **{"in": state8}, out=up, batch=B, hi=h0, wi=w0, ho=hf, wo=wf, c=3)
        state4 = self._head("fine_matcher", x2_0, x2_1, up, "s4")
        return state8, state4

    def _match_device(self, im0, im1, exact, warp, cert):
        B, _, H0, W0 = im0.shape
        _, state4 = self._forward_device(im0, im1, exact)
        _, hf, wf, _ = state4.shape
        full = self._b("state_full", (B, H0, W0, 3))
        call("romab200_bilinear_resize", "rb_resize_args", **{"in": state4}, out=full, batch=B, hi=hf, wi=wf, ho=H0, wo=W0, c=3)
        call("romab200_tiny_match_epilogue", "rb_tiny_epilogue_args", state=full, warp=warp, cert=cert, batch=B, h=H0, w=W0,
             grid_x=self._linspace(1 / W0, W0), grid_y=self._linspace(1 / H0, H0))

    # ---- inputs ---------------------------------------------------------------------------------------
    def _to_tensor(self, im):
        """torchvision ToTensor of an "RGB" or "L" PIL image (or of the same bytes decoded on the device): [1, C, H, W] fp32 in
        [0, 1] on the device."""
        if isinstance(im, DeviceImage):
            return im.raw.permute(2, 0, 1)[None].float().div(255)
        if im.mode not in ("RGB", "L"):
            raise NotImplementedError(f"TinyRoMa: PIL images of mode {im.mode!r} are not supported (RGB or L)")
        arr = torch.from_numpy(np.array(im, copy=True))
        arr = arr[:, :, None] if arr.dim() == 2 else arr
        return arr.to(self._device).permute(2, 0, 1)[None].float().div(255)

    def _check(self, im):
        if not isinstance(im, torch.Tensor) or im.dim() != 4:
            raise ValueError(f"TinyRoMa.match expects [B,C,H,W] tensors, PIL images or paths, got {type(im)}")
        if im.shape[-2] < 32 or im.shape[-1] < 32:
            raise ValueError(f"TinyRoMa needs images of at least 32 x 32 pixels, got {tuple(im.shape[-2:])}")
        return im

    # ---- public API -----------------------------------------------------------------------------------
    @torch.inference_mode()
    def match_from_path(self, im0_path, im1_path):
        # JPEG files are decoded on the device ("RGB" or "L", as Image.open gives them); other files take Image.open
        im0, im1 = open_inputs([im0_path, im1_path], self._device, rgb=False)
        return self.match(im0, im1)

    @torch.inference_mode()
    def match(self, im0, im1, *args, batched=True):
        """Dense warp [B,H0,W0,4] and certainty [B,H0,W0] at the size of image 0 (tiny.py:193-232); PIL / path inputs
        return [H0,W0,4] / [H0,W0]."""
        if isinstance(im0, (str, Path, os.PathLike)):
            return self.match_from_path(im0, im1)
        if isinstance(im0, (Image.Image, DeviceImage)):
            batched = False
            im0, im1 = self._to_tensor(im0), self._to_tensor(im1)
        im0, im1 = self._check(im0), self._check(im1)
        if im0.shape[0] != im1.shape[0]:
            raise ValueError(f"TinyRoMa.match: batch sizes differ ({im0.shape[0]} vs {im1.shape[0]})")
        B, _, H0, W0 = im0.shape
        exact = bool(self.exact_softmax)
        key = (tuple(im0.shape), tuple(im1.shape), exact)
        dev = self._device
        with torch.cuda.device(dev):
            entry = self._graphs.entry(key, lambda: dict(
                im0=torch.empty(im0.shape, device=dev), im1=torch.empty(im1.shape, device=dev),
                warp=torch.empty(B, H0, W0, 4, device=dev), cert=torch.empty(B, H0, W0, device=dev)), self.use_cuda_graph, self.arena.generation)
            bufs = entry["bufs"]
            bufs["im0"].copy_(im0, non_blocking=True)
            bufs["im1"].copy_(im1, non_blocking=True)
            self._graphs.run(entry, lambda: self._match_device(bufs["im0"], bufs["im1"], exact, bufs["warp"], bufs["cert"]))
            warp, cert = bufs["warp"].clone(), bufs["cert"].clone()
        return (warp, cert) if batched else (warp[0], cert[0])

    @torch.inference_mode()
    def forward(self, batch):
        """{8: {"flow" [B,2,h,w], "certainty" [B,1,h,w]}, 4: {...}} (tiny.py:268-304)."""
        im0 = self._check(batch["im_A"].to(self._device, torch.float32).contiguous())
        im1 = self._check(batch["im_B"].to(self._device, torch.float32).contiguous())
        with torch.cuda.device(self._device):
            states = dict(zip((8, 4), self._forward_device(im0, im1, bool(self.exact_softmax))))
            return {s: {"flow": st[..., :2].permute(0, 3, 1, 2).clone(), "certainty": st[..., 2:].permute(0, 3, 1, 2).clone()}
                    for s, st in states.items()}

    __call__ = forward

    def sample(self, matches, certainty, num=5000):
        """Certainty-thresholded, density-balanced sampling (tiny.py:234-266) on the device sampler shared with RoMa."""
        H, W, _ = matches.shape
        if not matches.is_cuda:
            raise RuntimeError("roma_b200.sample needs CUDA tensors (no CPU fallback)")
        return sample_device(self._sample_graphs, kde, matches, certainty, num, self.sample_mode, self.sample_thresh, self.use_cuda_graph)

    def sample_batched(self, matches, certainty, num=5000, *, repeats=1, chunk_bytes=sampling.SAMPLE_CHUNK_BYTES):
        """`repeats` samples of every pair of a batched warp in one call (RegressionMatcher.sample_batched): (m [B, repeats, k, 4],
        c [B, repeats, k]), equal after the same `torch.manual_seed` to `sample(matches[b], certainty[b], num)` called for b in range(B),
        r in range(repeats) in that order."""
        sampling.check_batched(matches, certainty, num, repeats)
        if not matches.is_cuda:
            raise RuntimeError("roma_b200.sample needs CUDA tensors (no CPU fallback)")
        return sampling.sample_batched(self._sample_graphs, kde, matches, certainty, num, repeats, self.sample_mode, self.sample_thresh,
                                       self.use_cuda_graph, chunk_bytes)

    # ---- geometry helpers (identical to RoMa's, tiny.py:102-113) ----------------------------------------
    _to_pixel_coordinates = RegressionMatcher._to_pixel_coordinates
    to_pixel_coordinates = RegressionMatcher.to_pixel_coordinates

    def visualize_warp(self, warp, certainty, im_A=None, im_B=None, im_A_path=None, im_B_path=None, symmetric=True, save_path=None,
                       unnormalize=False):
        """tiny.py:142-176 (RoMa's visualize_warp on the warp's device)."""
        return RegressionMatcher.visualize_warp(self, warp, certainty, im_A=im_A, im_B=im_B, im_A_path=im_A_path, im_B_path=im_B_path,
                                                device=warp.device, symmetric=symmetric, save_path=save_path, unnormalize=unnormalize)
