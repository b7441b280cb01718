"""Weight packing: reference state dicts -> device tensors in the layouts the kernels read.

Done once at construction on the host (fp32), then uploaded:
  * every BatchNorm is in eval mode during `match` (`matcher.py:790`, `encoders.py:53-54`), so it is folded
    into the preceding convolution: w' = w * g/sqrt(var+eps), b' = (b - mean) * g/sqrt(var+eps) + beta;
  * 3x3 VGG convolutions become GEMM operands [cout, 9*cin] with K ordered (ky, kx, cin) to match the
    9-tap shifted-row addressing of `romab200_gemm`; the first (3 -> 64) layer keeps (cin, ky, kx) order
    for the direct kernel;
  * 1x1 convolutions / Linear layers are [out, in] row-major (K contiguous) with the pitch padded to a
    multiple of 8 elements (16 bytes for 16-bit operands: TMA/global vector alignment);
  * depthwise 5x5 filters are stored tap-major [25, C_pad] so that lanes over channels read contiguously.
GEMM operands are stored in the compute dtype (fp32 for the parity mode, fp16/bf16 for the fast mode);
biases, LayerNorm/LayerScale vectors, depthwise filters and the fp32 heads stay fp32.
"""
from __future__ import annotations

from typing import Dict

import torch

from . import arch


def pad8(n: int) -> int:
    return (n + 7) // 8 * 8


def at(t: torch.Tensor, elems: int) -> torch.Tensor:
    """The flat view of contiguous `t` from element `elems` on: an operand that starts inside a buffer, with the buffer's dtype,
    device and remaining extent for the C-ABI checks (cabi.call)."""
    return t.view(-1)[elems:]


def fold_bn(w: torch.Tensor, b: torch.Tensor, sd: Dict[str, torch.Tensor], bn: str, eps: float = arch.BN_EPS):
    """Fold eval-mode BatchNorm `bn` into the conv (w [cout, ...], b [cout]).  A BatchNorm2d(affine=False) has no
    `weight` / `bias` entries: gamma = 1, beta = 0."""
    gamma = sd[f"{bn}.weight"].double() if f"{bn}.weight" in sd else 1.0
    beta = sd[f"{bn}.bias"].double() if f"{bn}.bias" in sd else 0.0
    scale = gamma / torch.sqrt(sd[f"{bn}.running_var"].double() + eps)
    w2 = w.double() * scale.view(-1, *([1] * (w.dim() - 1)))
    b2 = (b.double() - sd[f"{bn}.running_mean"].double()) * scale + beta
    return w2.float(), b2.float()


class Split:
    """An RB_F16S matrix (include/romab200.h): fp16 hi plane + fp16 lo plane of identical geometry, value = hi + lo * 2^-11
    with hi = fp16(x), lo = fp16((x - hi) * 2^11).  `hi` / `lo` are fp16 tensors of the same shape."""
    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo):
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return self.hi.shape

    def at(self, elems: int) -> "Split":
        """The pair of flat views starting `elems` elements further into both planes."""
        return Split(at(self.hi, elems), at(self.lo, elems))

    def join(self) -> torch.Tensor:
        """fp32 reconstruction (tests / debug)."""
        return self.hi.float() + self.lo.float() / 2048.0


def split_f16s(w: torch.Tensor):
    """fp32 tensor -> (hi, lo) fp16 planes of the RB_F16S format (the host twin of csrc/common.cuh::split_f16s)."""
    w = w.float()
    hi = w.to(torch.float16)
    lo = ((w - hi.float()) * 2048.0).to(torch.float16)
    return hi, lo


def _mat(w: torch.Tensor, dtype, device, pitch=None, split=False):
    """[n, k] fp32 -> [n, pitch] compute-dtype matrix (zero padded along k); an RB_F16S pair in the parity mode."""
    n, k = w.shape
    pitch = pitch or pad8(k)
    if split:
        hi, lo = split_f16s(w)
        oh, ol = torch.zeros(n, pitch, dtype=torch.float16), torch.zeros(n, pitch, dtype=torch.float16)
        oh[:, :k], ol[:, :k] = hi, lo
        return Split(oh.to(device), ol.to(device))
    out = torch.zeros(n, pitch, dtype=dtype)
    out[:, :k] = w.to(dtype)
    return out.to(device)


def _vec(v: torch.Tensor, device):
    return v.float().contiguous().to(device)


class PackedWeights:
    """All device-resident parameters of the path, keyed by stage."""

    def __init__(self, matcher_sd: Dict[str, torch.Tensor], dino_sd: Dict[str, torch.Tensor], device, dtype: torch.dtype, split: bool = False):
        self.device, self.dtype, self.split = device, dtype, split
        sd = {k: v.detach().cpu() for k, v in matcher_sd.items()}
        dd = {k: v.detach().cpu().float() for k, v in dino_sd.items()}
        self._check(sd, dd)
        self.vgg = self._pack_vgg(sd)
        self.proj = self._pack_proj(sd)
        self.vit = self._pack_blocks(dd, "blocks", arch.VIT_DEPTH, layerscale=True, qkv_bias=True)
        self.vit_patch_w = _mat(dd["patch_embed.proj.weight"].flatten(1), dtype, device, split=split)       # [1024, 588 -> 592]
        self.vit_patch_b = _vec(dd["patch_embed.proj.bias"], device)
        self.vit_cls = _vec(dd["cls_token"].reshape(-1), device)
        self.vit_pos_embed = dd["pos_embed"]                  # host fp32; interpolated per resolution by the engine
        self.vit_norm = (_vec(dd["norm.weight"], device), _vec(dd["norm.bias"], device))
        self.dec = self._pack_blocks(sd, "decoder.embedding_decoder.blocks", arch.DEC_DEPTH, layerscale=False, qkv_bias=False)
        self.to_out_w = _mat(sd["decoder.embedding_decoder.to_out.weight"].float(), dtype, device, split=split)
        self.to_out_b = _vec(sd["decoder.embedding_decoder.to_out.bias"], device)
        self.gp_pos_w = sd["decoder.gps.16.pos_conv.weight"].float()          # host: the basis is a per-resolution constant
        self.gp_pos_b = sd["decoder.gps.16.pos_conv.bias"].float()
        self.refiner = {s: self._pack_refiner(sd, s) for s in arch.SCALES}

    # ------------------------------------------------------------------
    @staticmethod
    def _check(sd, dd):
        want = {k: tuple(shape) for k, shape, _ in arch.matcher_param_specs()}
        missing = [k for k in want if k not in sd]
        if missing:
            raise RuntimeError(f"Error(s) in loading state_dict: missing keys {missing[:4]}... ({len(missing)} total)")
        for k, shape in want.items():
            if tuple(sd[k].shape) != shape:
                raise RuntimeError(f"size mismatch for {k}: {tuple(sd[k].shape)} vs {shape}")
        wantd = {k: tuple(shape) for k, shape, _ in arch.dinov2_param_specs()}
        for k, shape in wantd.items():
            if k not in dd:
                raise RuntimeError(f"Error(s) in loading state_dict for DinoVisionTransformer: missing key {k}")
            if tuple(dd[k].shape) != shape:
                raise RuntimeError(f"size mismatch for {k}: {tuple(dd[k].shape)} vs {shape}")

    def _pack_vgg(self, sd):
        layers = []
        for li, (idx, cin, cout) in enumerate(arch.VGG_CONVS):
            w, b = fold_bn(sd[f"encoder.cnn.layers.{idx}.weight"].float(), sd[f"encoder.cnn.layers.{idx}.bias"].float(),
                           sd, f"encoder.cnn.layers.{idx + 1}")
            if li == 0:
                layers.append(dict(w=w.reshape(cout, 27).contiguous().to(self.device), b=_vec(b, self.device), cin=cin, cout=cout))
            else:
                wm = w.permute(0, 2, 3, 1).reshape(cout, 9 * cin)        # K = (ky, kx, cin)
                layers.append(dict(w=_mat(wm, self.dtype, self.device, pitch=9 * cin, split=self.split), b=_vec(b, self.device), cin=cin, cout=cout))
        return layers

    def _pack_proj(self, sd):
        out = {}
        for s in arch.SCALES:
            w, b = fold_bn(sd[f"decoder.proj.{s}.0.weight"].float().flatten(1), sd[f"decoder.proj.{s}.0.bias"].float(),
                           sd, f"decoder.proj.{s}.1")
            out[s] = dict(w=_mat(w, self.dtype, self.device, split=self.split), b=_vec(b, self.device))
        return out

    def _pack_blocks(self, sd, prefix, depth, layerscale, qkv_bias):
        blocks = []
        for i in range(depth):
            p = f"{prefix}.{i}"
            blocks.append(dict(
                ln1=(_vec(sd[f"{p}.norm1.weight"], self.device), _vec(sd[f"{p}.norm1.bias"], self.device)),
                qkv_w=_mat(sd[f"{p}.attn.qkv.weight"].float(), self.dtype, self.device, split=self.split),
                qkv_b=_vec(sd[f"{p}.attn.qkv.bias"], self.device) if qkv_bias else None,
                proj_w=_mat(sd[f"{p}.attn.proj.weight"].float(), self.dtype, self.device, split=self.split),
                proj_b=_vec(sd[f"{p}.attn.proj.bias"], self.device),
                ls1=_vec(sd[f"{p}.ls1.gamma"], self.device) if layerscale else None,
                ln2=(_vec(sd[f"{p}.norm2.weight"], self.device), _vec(sd[f"{p}.norm2.bias"], self.device)),
                fc1_w=_mat(sd[f"{p}.mlp.fc1.weight"].float(), self.dtype, self.device, split=self.split),
                fc1_b=_vec(sd[f"{p}.mlp.fc1.bias"], self.device),
                fc2_w=_mat(sd[f"{p}.mlp.fc2.weight"].float(), self.dtype, self.device, split=self.split),
                fc2_b=_vec(sd[f"{p}.mlp.fc2.bias"], self.device),
                ls2=_vec(sd[f"{p}.ls2.gamma"], self.device) if layerscale else None,
            ))
        return blocks

    def _pack_refiner(self, sd, s):
        spec = arch.REFINERS[s]
        c, cp = spec.channels, pad8(spec.channels)
        p = f"decoder.conv_refiner.{s}"
        blocks = []
        for blk in ["block1"] + [f"hidden_blocks.{j}" for j in range(arch.REFINER_HIDDEN_BLOCKS)]:
            q = f"{p}.{blk}"
            dw, db = fold_bn(sd[f"{q}.0.weight"].float(), sd[f"{q}.0.bias"].float(), sd, f"{q}.1")
            dwt = torch.zeros(25, cp)
            dwt[:, :c] = dw.reshape(c, 25).t()
            pw = sd[f"{q}.3.weight"].float().flatten(1)
            blocks.append(dict(
                dw_w=dwt.to(self.device), dw_b=_vec(db, self.device),
                pw_w=_mat(pw, self.dtype, self.device, pitch=cp, split=self.split),
                pw_b=_vec(sd[f"{q}.3.bias"], self.device),
                # thin maps (C = 24) run the fused CUDA-core block: fp32 copy of the compute-dtype-rounded weights
                # thin maps: the fused block kernel takes its pointwise weights as launch parameters, i.e. from host memory
                pw_w_host=pw.to(self.dtype).float().contiguous().cpu() if c <= 32 else None,      # (fp32 modes: exact)
                pw_b_host=sd[f"{q}.3.bias"].float().contiguous().cpu() if c <= 32 else None,
            ))
        ow = torch.zeros(3, cp)
        ow[:, :c] = sd[f"{p}.out_conv.weight"].float().flatten(1)
        return dict(
            blocks=blocks, out_w=ow.to(self.device), out_b=_vec(sd[f"{p}.out_conv.bias"], self.device),
            emb_w=_vec(sd[f"{p}.disp_emb.weight"].float().reshape(spec.emb, 2), self.device),
            emb_b=_vec(sd[f"{p}.disp_emb.bias"], self.device), c=c, cp=cp, spec=spec,
        )
