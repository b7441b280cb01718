"""CPU oracle for RoMa's dense `match()` / `sample()` path.  TEST INFRASTRUCTURE ONLY.

This file is a from-scratch, functional (no nn.Module) fp32 restatement of the reference's
algorithm for the hot path, written against `torch` CPU operators because the reference's
arithmetic *is* defined by those ATen operators (grid_sample, interpolate, SDPA, cholesky ...;
SURVEY.md §8c).  Every function cites the reference file:line it follows.  It exists so that
the CUDA path in `roma_b200/` can be checked on a box that has no copy of the reference.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s CPU-baseline legs may import it; the
product package never does (tests/test_host_logic.py::test_layout_product_never_imports_oracle enforces that).

Pinning: the reference has no tensor-level golden vectors (SURVEY.md §4), so the oracle is pinned
against outputs of the *unmodified reference itself*, imported from /root/reference in the build
container with the seeded synthetic weights of `roma_b200.synthetic`
(`tests/golden/make_golden.py` is the generating script, `tests/golden/*.npz` the fixtures,
`tests/test_oracle_golden.py` the check).  fused-local-corr 0.2.2 (PyPI wheel, binary only,
`uv.lock:541-553`) is absent, so the oracle follows the in-tree pure-torch local correlation
(`local_correlation.py:39-74`, `use_custom_corr=False`): parity at the wheel boundary is unpinned.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F

# ----------------------------------------------------------------------------------------------
# constants (roma_models.py:71-181)
# ----------------------------------------------------------------------------------------------
VGG_CONV_IDX = (0, 3, 7, 10, 14, 17, 20, 23, 27, 30, 33, 36)
VGG_POOL_IDX = (6, 13, 26, 39)
REFINER = {16: (128, 7), 8: (64, 3), 4: (32, 2), 2: (16, 0), 1: (6, 0)}   # scale -> (emb dim, radius)
SCALES = (16, 8, 4, 2, 1)


def pixel_centre_grid(b: int, h: int, w: int, device="cpu", dtype=torch.float32) -> torch.Tensor:
    """[b,2,h,w] normalised pixel-centre coordinates, channel 0 = x (matcher.py:365-377).  Always built in fp32 on the CPU (the
    values the fixtures were pinned with) and then moved: `device` only matters for the stock-PyTorch-CUDA timing leg, `dtype`
    for the fp64 oracle."""
    ys = torch.linspace(-1 + 1 / h, 1 - 1 / h, h)
    xs = torch.linspace(-1 + 1 / w, 1 - 1 / w, w)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    return torch.stack((gx, gy))[None].expand(b, 2, h, w).to(device, dtype)


class RomaOracle:
    """Functional fp32 restatement of `RegressionMatcher` (matcher.py:550-934) for tensor inputs."""

    def __init__(self, matcher_weights: Dict[str, torch.Tensor], dinov2_weights: Dict[str, torch.Tensor],
                 coarse_res=560, upsample_res=864, symmetric=True, upsample_preds=True,
                 attenuate_cert=True, sample_thresh=0.05, sample_mode="threshold_balanced", device="cpu", dtype=torch.float32):
        # device != "cpu" is the stock-PyTorch-on-GPU timing leg of bench.py (`--impl torch_cuda`): the same torch.nn.functional
        # graph on cuDNN / cuBLAS / SDPA kernels; every parity check uses the CPU default.  dtype=torch.float64 runs the same
        # graph in double precision (weights, activations and the fp32-built grids cast up): the reference stage checks of the
        # parity mode compare against, whose own fp32 rounding would be of the size of the errors they bound
        self.device = torch.device(device)
        self.dtype = dtype
        self.w = {k: (v.to(dtype) if v.is_floating_point() else v).to(self.device) for k, v in matcher_weights.items()}
        self.d = {k: v.to(dtype).to(self.device) for k, v in dinov2_weights.items()}
        cr = (coarse_res, coarse_res) if isinstance(coarse_res, int) else tuple(coarse_res)
        ur = (upsample_res, upsample_res) if isinstance(upsample_res, int) else upsample_res
        self.h_resized, self.w_resized = cr
        self.upsample_res = ur
        self.symmetric = symmetric
        self.upsample_preds = upsample_preds
        self.attenuate_cert = attenuate_cert
        self.sample_thresh = sample_thresh
        self.sample_mode = sample_mode
        self.trace: Optional[dict] = None      # set to {} to record stage outputs

    # ------------------------------------------------------------------ helpers
    def _rec(self, name, value):
        if self.trace is not None:
            self.trace[name] = value

    def _bn(self, x, prefix):
        w = self.w
        return F.batch_norm(x, w[f"{prefix}.running_mean"], w[f"{prefix}.running_var"],
                            w[f"{prefix}.weight"], w[f"{prefix}.bias"], False, 0.0, 1e-5)

    # ------------------------------------------------------------------ encoders
    def vgg(self, x):
        """VGG19-BN features[:40]; taps are the inputs of the four max-pools (encoders.py:17-27)."""
        feats = {}
        for s in (1, 2, 4, 8):
            if s > 1:
                x = F.max_pool2d(x, 2, 2)
            x = feats[s] = self.vgg_stage(s, x)
        return feats

    def vgg_stage(self, s, x):
        """The conv + BN + ReLU layers of VGG stage `s` (1, 2, 4, 8): the image (s = 1) or the max-pooled tap of the stage before
        -> the tap at stride s."""
        k = (1, 2, 4, 8).index(s)
        for idx in range(VGG_POOL_IDX[k - 1] + 1 if k else 0, VGG_POOL_IDX[k]):
            if idx in VGG_CONV_IDX:
                p = f"encoder.cnn.layers.{idx}"
                x = F.conv2d(x, self.w[f"{p}.weight"], self.w[f"{p}.bias"], padding=1)
                x = F.relu(self._bn(x, f"encoder.cnn.layers.{idx + 1}"))
        return x

    def dinov2_pos_embed(self, hp, wp):
        """Bicubic resize of the 37x37 positional grid with the `+0.1` scale-factor quirk
        (dinov2.py:166-190); `size=` would give different values (SURVEY Appendix A)."""
        pe = self.d["pos_embed"]
        n = pe.shape[1] - 1
        side = int(math.sqrt(n))
        if hp * wp == n and hp == wp:
            return pe
        grid = pe[:, 1:].reshape(1, side, side, -1).permute(0, 3, 1, 2)
        grid = F.interpolate(grid, scale_factor=((hp + 0.1) / side, (wp + 0.1) / side), mode="bicubic")
        assert grid.shape[-2:] == (hp, wp)
        grid = grid.permute(0, 2, 3, 1).reshape(1, hp * wp, -1)
        return torch.cat((pe[:, :1], grid), dim=1)

    def _vit_block(self, x, p, w, heads, eps, layerscale):
        """pre-LN block: x += ls1(attn(LN(x))); x += ls2(mlp(LN(x))) (block.py:82-107, attention.py:50-63)."""
        b, n, c = x.shape
        y = F.layer_norm(x, (c,), w[f"{p}.norm1.weight"], w[f"{p}.norm1.bias"], eps)
        qkv = F.linear(y, w[f"{p}.attn.qkv.weight"], w.get(f"{p}.attn.qkv.bias"))
        q, k, v = qkv.reshape(b, n, 3, heads, c // heads).unbind(2)
        a = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2))
        a = F.linear(a.transpose(1, 2).reshape(b, n, c), w[f"{p}.attn.proj.weight"], w[f"{p}.attn.proj.bias"])
        x = x + (a * w[f"{p}.ls1.gamma"] if layerscale else a)
        y = F.layer_norm(x, (c,), w[f"{p}.norm2.weight"], w[f"{p}.norm2.bias"], eps)
        y = F.linear(F.gelu(F.linear(y, w[f"{p}.mlp.fc1.weight"], w[f"{p}.mlp.fc1.bias"])),
                     w[f"{p}.mlp.fc2.weight"], w[f"{p}.mlp.fc2.bias"])
        return x + (y * w[f"{p}.ls2.gamma"] if layerscale else y)

    def dinov2(self, x):
        """DINOv2 ViT-L/14 patch tokens as a [B,1024,H/14,W/14] map (encoders.py:60-67, dinov2.py:192-237)."""
        d = self.d
        b, _, hh, ww = x.shape
        t = F.conv2d(x, d["patch_embed.proj.weight"], d["patch_embed.proj.bias"], stride=14)
        hp, wp = t.shape[-2:]
        t = t.flatten(2).transpose(1, 2)
        t = torch.cat((d["cls_token"].expand(b, -1, -1), t), dim=1) + self.dinov2_pos_embed(hp, wp)
        for i in range(24):
            t = self._vit_block(t, f"blocks.{i}", d, 16, 1e-6, True)
        t = F.layer_norm(t, (1024,), d["norm.weight"], d["norm.bias"], 1e-6)
        return t[:, 1:].permute(0, 2, 1).reshape(b, 1024, hp, wp)

    def encoder(self, x, upsample=False):
        pyramid = self.vgg(x)
        if not upsample:
            pyramid[16] = self.dinov2(x)
        return pyramid

    # ------------------------------------------------------------------ coarse matcher
    def proj(self, s, f):
        """1x1 conv + BN (roma_models.py:156-169; applied matcher.py:441-450)."""
        p = f"decoder.proj.{s}"
        return self._bn(F.conv2d(f, self.w[f"{p}.0.weight"], self.w[f"{p}.0.bias"]), f"{p}.1")

    @staticmethod
    def cos_kernel(x, y, T=0.2, eps=1e-6):
        """K = exp((cos(x,y) - 1)/T), eps added to the product of norms (matcher.py:191-200)."""
        c = torch.einsum("bnd,bmd->bnm", x, y) / (x.norm(dim=-1)[..., None] * y.norm(dim=-1)[:, None] + eps)
        return ((c - 1.0) / torch.tensor(T)).exp()

    def gp(self, x, y):
        """GP posterior mean of the Fourier positional basis (matcher.py:291-323)."""
        b, c, h1, w1 = x.shape
        _, _, h2, w2 = y.shape
        w = self.w
        f = torch.cos(8 * math.pi * F.conv2d(pixel_centre_grid(b, h2, w2, x.device, self.dtype),
                                              w["decoder.gps.16.pos_conv.weight"], w["decoder.gps.16.pos_conv.bias"]))
        flat = lambda t: t.flatten(2).transpose(1, 2)
        x, y, f = flat(x.to(self.dtype)), flat(y.to(self.dtype)), flat(f)
        k_yy = self.cos_kernel(y, y)
        k_xy = self.cos_kernel(x, y)
        noise = 0.1 * torch.eye(h2 * w2, dtype=self.dtype)[None].to(x.device)
        chol = torch.linalg.cholesky(k_yy + noise)
        alpha = torch.cholesky_solve(f, chol, upper=False)
        mu = k_xy @ alpha
        self._rec("gp.k_xy", k_xy), self._rec("gp.alpha", alpha)
        return mu.transpose(1, 2).reshape(b, -1, h1, w1)

    def embedding_decoder(self, gp_post, feats):
        """5 pre-LN blocks (8 heads, eps 1e-5, no qkv bias, no LayerScale) + Linear -> 64*64+1
        (transformer/__init__.py:30-46)."""
        b, _, h, wd = gp_post.shape
        t = torch.cat((gp_post, feats), dim=1).flatten(2).transpose(1, 2)
        for i in range(5):
            t = self._vit_block(t, f"decoder.embedding_decoder.blocks.{i}", self.w, 8, 1e-5, False)
        out = F.linear(t, self.w["decoder.embedding_decoder.to_out.weight"],
                       self.w["decoder.embedding_decoder.to_out.bias"])
        out = out.transpose(1, 2).reshape(b, -1, h, wd)
        return out[:, :-1], out[:, -1:]

    @staticmethod
    def cls_to_flow_refine(cls):
        """softmax -> argmax -> 5-neighbour soft-argmax over the 64x64 anchor grid, with the
        reference's clamp/wrap behaviour (utils.py:300-322). Returns [B,H,W,2]."""
        b, c, h, w = cls.shape
        res = round(math.sqrt(c))
        lin = torch.linspace(-1 + 1 / res, 1 - 1 / res, res)
        gy, gx = torch.meshgrid(lin, lin, indexing="ij")
        anchors = torch.stack((gx, gy), dim=-1).reshape(c, 2).to(cls.device, cls.dtype)
        p = cls.softmax(dim=1)
        mode = p.max(dim=1).indices
        idx = torch.stack((mode - 1, mode, mode + 1, mode - res, mode + res), dim=1).clamp(0, c - 1)
        nb = torch.gather(p, 1, idx)[..., None]
        num = sum(nb[:, j] * anchors[idx[:, j]] for j in range(5))
        return num / nb.sum(dim=1)

    # ------------------------------------------------------------------ refinement
    @staticmethod
    def local_correlation(f0, f1, r, flow):
        """(2r+1)^2 window of bilinear samples of f1 around `flow`, dotted with f0/sqrt(c)
        (local_correlation.py:77-142 with the pure-torch body :39-74). flow is [B,2,H,W]."""
        b, c, h, w = f0.shape
        k = (2 * r + 1) ** 2
        wy = torch.linspace(-2 * r / h, 2 * r / h, 2 * r + 1)
        wx = torch.linspace(-2 * r / w, 2 * r / w, 2 * r + 1)
        oy, ox = torch.meshgrid(wy, wx, indexing="ij")
        window = torch.stack((ox, oy), dim=-1).reshape(1, k, 2).to(f0.device, f0.dtype)
        flow = flow.permute(0, 2, 3, 1)
        corr = torch.empty(b, k, h, w, device=f0.device, dtype=f0.dtype)
        band = max(1, (1 << 27) // (c * w * k * f0.element_size()))      # rows per grid_sample: bounds the [c, rows, w, k] samples
        for i in range(b):
            for y0 in range(0, h, band):
                y1 = min(h, y0 + band)
                coords = (flow[i, y0:y1, :, None] + window[:, None, None]).reshape(1, y1 - y0, w * k, 2)
                samp = F.grid_sample(f1[i:i + 1], coords, padding_mode="zeros", align_corners=False,
                                     mode="bilinear").reshape(c, y1 - y0, w, k)
                corr[i, :, y0:y1] = (f0[i, :, y0:y1, :, None] / (c ** 0.5) * samp).sum(dim=0).permute(2, 0, 1)
        return corr

    def refiner_input(self, s, x, y, flow, scale_factor):
        """d = cat(x, x_hat, disp_emb, local_corr) (matcher.py:132-168)."""
        b, c, hs, ws = x.shape
        emb_dim, r = REFINER[s]
        p = f"decoder.conv_refiner.{s}"
        x_hat = F.grid_sample(y, flow.permute(0, 2, 3, 1), align_corners=False, mode="bilinear")
        disp = flow - pixel_centre_grid(b, hs, ws, flow.device, self.dtype)
        emb = F.conv2d(40 / 32 * scale_factor * disp, self.w[f"{p}.disp_emb.weight"], self.w[f"{p}.disp_emb.bias"])
        parts = [x, x_hat, emb]
        if r:
            parts.append(self.local_correlation(x, y, r, flow))
        return torch.cat(parts, dim=1)

    def refiner_blocks(self, s, d):
        """block1 + 8 hidden blocks of DW5x5 + BN + ReLU + PW1x1, then the fp32 1x1 head
        (matcher.py:92-122,175-179)."""
        p = f"decoder.conv_refiner.{s}"
        c = d.shape[1]
        for blk in ["block1"] + [f"hidden_blocks.{j}" for j in range(8)]:
            q = f"{p}.{blk}"
            d = F.conv2d(d, self.w[f"{q}.0.weight"], self.w[f"{q}.0.bias"], padding=2, groups=c)
            d = F.relu(self._bn(d, f"{q}.1"))
            d = F.conv2d(d, self.w[f"{q}.3.weight"], self.w[f"{q}.3.bias"])
            self._rec(f"refiner{s}.{blk}", d)
        return F.conv2d(d, self.w[f"{p}.out_conv.weight"], self.w[f"{p}.out_conv.bias"])

    def conv_refiner(self, s, x, y, flow, scale_factor):
        d = self.refiner_input(s, x, y, flow, scale_factor)
        self._rec(f"refiner{s}.input", d)
        out = self.refiner_blocks(s, d)
        return out[:, :-1], out[:, -1:]

    def decoder(self, f1, f2, upsample=False, flow=None, certainty=None, scale_factor=1.0):
        """Coarse-to-fine loop (matcher.py:395-527)."""
        scales = SCALES if not upsample else SCALES[1:]
        sizes = {s: f1[s].shape[-2:] for s in f1}
        h, w = sizes[1]
        b = f1[1].shape[0]
        tag = "up" if upsample else "lo"
        if not upsample:
            flow, certainty = pixel_centre_grid(b, *sizes[16], device=f1[1].device, dtype=self.dtype), 0.0
        else:
            flow = F.interpolate(flow, size=sizes[8], align_corners=False, mode="bilinear")
            certainty = F.interpolate(certainty, size=sizes[8], align_corners=False, mode="bilinear")
        corresps = {}
        for s in scales:
            x, y = self.proj(s, f1[s].to(self.dtype)), self.proj(s, f2[s].to(self.dtype))
            self._rec(f"{tag}.proj{s}.x", x)
            if s == 16:
                post = self.gp(x, y)
                self._rec("gp.mu", post)
                cls, certainty = self.embedding_decoder(post, x)
                self._rec("cls", cls)
                flow = self.cls_to_flow_refine(cls).permute(0, 3, 1, 2)
                self._rec("coarse_flow", flow)
            self._rec(f"{tag}.flow_in{s}", flow)
            delta, dcert = self.conv_refiner(s, x, y, flow, scale_factor)
            self._rec(f"{tag}.delta{s}", torch.cat((delta, dcert), 1))
            disp = s * torch.stack((delta[:, 0] / (4 * w), delta[:, 1] / (4 * h)), dim=1)
            flow = flow + disp
            certainty = certainty + dcert
            corresps[s] = {"flow": flow, "certainty": certainty}
            if s != 1:
                flow = F.interpolate(flow, size=sizes[s // 2], mode="bilinear")
                certainty = F.interpolate(certainty, size=sizes[s // 2], mode="bilinear")
        return corresps

    def forward(self, im_a, im_b, upsample=False, scale_factor=1.0, corresps=None):
        """forward_symmetric / forward (matcher.py:631-670)."""
        pyr = self.encoder(torch.cat((im_a, im_b)), upsample=upsample)
        if self.trace is not None:
            tag = "up" if upsample else "lo"
            for s, f in pyr.items():
                self._rec(f"{tag}.feat{s}", f)
        if self.symmetric:
            f_q = pyr
            f_s = {s: torch.cat((f.chunk(2)[1], f.chunk(2)[0])) for s, f in pyr.items()}
        else:
            f_q = {s: f.chunk(2)[0] for s, f in pyr.items()}
            f_s = {s: f.chunk(2)[1] for s, f in pyr.items()}
        return self.decoder(f_q, f_s, upsample=upsample, scale_factor=scale_factor, **(corresps or {}))

    # ------------------------------------------------------------------ API
    @torch.inference_mode()
    def match(self, im_a, im_b, im_a_high=None, im_b_high=None):
        """Tensor-input `match` (matcher.py:779-934): returns (warp [b,H,W(*2),4], certainty [b,H,W(*2)])."""
        scale_factor = math.sqrt(self.h_resized * self.w_resized / 560 ** 2)
        corresps = self.forward(im_a, im_b, scale_factor=scale_factor)
        coarse_certainty = corresps[16]["certainty"] if self.attenuate_cert else None
        if self.upsample_preds:
            scale_factor = math.sqrt(self.upsample_res[0] * self.upsample_res[1] / 560 ** 2)
            corresps = self.forward(im_a_high, im_b_high, upsample=True, scale_factor=scale_factor,
                                    corresps=corresps[1])
        return self.epilogue(corresps[1]["flow"], corresps[1]["certainty"], coarse_certainty)

    def epilogue(self, flow, certainty, coarse_certainty=None):
        """The end of `match` (matcher.py:868-934): final flow [D,2,H,W] and certainty logit [D,1,H,W], attenuated by the coarse
        pass's stride-16 certainty [D,1,h,w] unless it is None -> (warp [b,H,W(*2),4], certainty [b,H,W(*2)])."""
        hs, ws = flow.shape[-2:]
        b = flow.shape[0] // (2 if self.symmetric else 1)
        low = 0
        if coarse_certainty is not None:
            low = F.interpolate(coarse_certainty, size=(hs, ws), align_corners=False, mode="bilinear")
            low = 0.5 * low * (low < 0)
        flow = flow.permute(0, 2, 3, 1)
        cert = (certainty - low).sigmoid()
        self._rec("final.flow", flow), self._rec("final.logit", certainty - low)
        grid = pixel_centre_grid(b, hs, ws, flow.device, self.dtype).permute(0, 2, 3, 1)
        if (flow.abs() > 1).any():
            wrong = (flow.abs() > 1).sum(dim=-1) > 0
            cert[wrong[:, None]] = 0
        flow = flow.clamp(-1, 1)
        if self.symmetric:
            a2b, b2a = flow.chunk(2)
            warp = torch.cat((torch.cat((grid, a2b), dim=-1), torch.cat((b2a, grid), dim=-1)), dim=2)
            cert = torch.cat(cert.chunk(2), dim=3)
        else:
            warp = torch.cat((grid, flow), dim=-1)
        return warp, cert[:, 0]

    @staticmethod
    def kde(x, std=0.1):
        """fp16 Gaussian KDE (kde.py:4-12)."""
        x = x.half()
        return (-torch.cdist(x, x) ** 2 / (2 * std ** 2)).exp().sum(dim=-1)

    def sample(self, matches, certainty, num=10000):
        """threshold-balanced sampling (matcher.py:598-629); RNG = torch global generator."""
        if "threshold" in self.sample_mode:
            certainty = certainty.clone()
            certainty[certainty > self.sample_thresh] = 1
        matches, certainty = matches.reshape(-1, 4), certainty.reshape(-1)
        factor = 4 if "balanced" in self.sample_mode else 1
        good = torch.multinomial(certainty, num_samples=min(factor * num, len(certainty)), replacement=False)
        gm, gc = matches[good], certainty[good]
        if "balanced" not in self.sample_mode:
            return gm, gc
        density = self.kde(gm, std=0.1)
        p = 1 / (density + 1)
        p[density < 10] = 1e-7
        pick = torch.multinomial(p, num_samples=min(num, len(gc)), replacement=False)
        return gm[pick], gc[pick]
