"""CPU fp32 restatement of TinyRoMa's inference path (`romatch/models/tiny.py`: forward_single, corr_volume, pos_embed, forward,
match, sample) in plain torch.nn.functional — test infrastructure for `roma_b200.tiny`, checked against the reference's goldens.

The backbone is the caller's XFeat module itself (loaded with the checkpoint's `xfeat.0.*` entries, eval mode), run part by part
in the order tiny.py:81-97 uses; the matcher heads are restated from the checkpoint tensors.  `device` other than "cpu" is the
stock-PyTorch-on-GPU leg of scripts/bench_tiny.py.
"""
from __future__ import annotations

import copy
import math

import torch
import torch.nn.functional as F

from oracle.roma_oracle import RomaOracle

XFEAT_DELETED = ("heatmap_head", "keypoint_head", "fine_matcher")


class TinyOracle:
    def __init__(self, weights, xfeat, exact_softmax=False, sample_thresh=0.05, sample_mode="threshold_balanced", device="cpu"):
        self.device = torch.device(device)
        xf = copy.deepcopy(xfeat)
        for name in XFEAT_DELETED:
            if hasattr(xf, name):
                delattr(xf, name)
        xf.load_state_dict({k[len("xfeat.0."):]: v for k, v in weights.items() if k.startswith("xfeat.0.")}, strict=True)
        self.xfeat = xf.to(self.device).eval()
        self.sd = {k: v.to(self.device) for k, v in weights.items() if not k.startswith("xfeat.")}
        self.exact_softmax = exact_softmax
        self.sample_thresh, self.sample_mode = sample_thresh, sample_mode
        self.trace = None                      # set to {} to record stage outputs

    def _keep(self, key, t):
        if self.trace is not None:
            self.trace.setdefault(key, []).append(t.detach().clone())

    @staticmethod
    def preprocess(x):
        H, W = x.shape[-2:]
        return F.interpolate(x, (H // 32 * 32, W // 32 * 32), mode="bilinear", align_corners=False)

    def backbone(self, x):
        xf = self.xfeat
        x = xf.norm(x.mean(dim=1, keepdim=True))
        x1 = xf.block1(x)
        x2 = xf.block2(x1 + xf.skip1(x))
        x3 = xf.block3(x2)
        x4 = xf.block4(x3)
        x5 = xf.block5(x4)
        x4 = F.interpolate(x4, x3.shape[-2:], mode="bilinear", align_corners=False)
        x5 = F.interpolate(x5, x3.shape[-2:], mode="bilinear", align_corners=False)
        return x2, xf.block_fusion(x3 + x4 + x5)

    def head(self, name, x):
        for i in range(4):
            p = f"{name}.{i}.layer"
            x = F.conv2d(x, self.sd[f"{p}.0.weight"], padding=1)
            x = F.relu(F.batch_norm(x, self.sd[f"{p}.1.running_mean"], self.sd[f"{p}.1.running_var"], None, None, False, 0.0, 1e-5))
        return F.conv2d(x, self.sd[f"{name}.4.weight"], self.sd[f"{name}.4.bias"])

    @staticmethod
    def corr(f0, f1):
        """s[b, j, i] = <f1[b,:,j], f0[b,:,i]> / sqrt(C): [B, h1*w1, h0*w0]."""
        B, C = f0.shape[:2]
        return torch.einsum("bci,bcj->bji", f0.reshape(B, C, -1), f1.reshape(B, C, -1)) / math.sqrt(C)

    @staticmethod
    def pos_embed(f0, f1, exact=False):
        """pos_embed(corr_volume(f0, f1)) -> [B, 2, h0, w0]; also returns the argmax index and the top-2 score gap per pixel."""
        B, C, h0, w0 = f0.shape
        h1, w1 = f1.shape[-2:]
        cv = TinyOracle.corr(f0, f1)                                        # [B, h1*w1, h0*w0]
        gx = torch.linspace(-1 + 1 / w1, 1 - 1 / w1, w1)
        gy = torch.linspace(-1 + 1 / h1, 1 - 1 / h1, h1)
        grid = torch.stack(torch.meshgrid(gx, gy, indexing="xy"), -1).reshape(h1 * w1, 2).to(cv)
        top2 = cv.topk(2, dim=1).values
        gap = (top2[:, 0] - top2[:, 1]).reshape(B, h0, w0)
        best = cv.argmax(dim=1)                                              # first index on ties
        if exact:
            P = cv.softmax(dim=1)
            pos = torch.einsum("bji,jd->bdi", P, grid)
        else:
            d = 4
            lx = torch.linspace(-1 + d / w1, 1 - d / w1, w1 // d)
            ly = torch.linspace(-1 + d / h1, 1 - d / h1, h1 // d)
            grid_lr = torch.stack(torch.meshgrid(lx, ly, indexing="xy"), -1).reshape(-1, 2).to(cv)
            sub = cv.reshape(B, h1, w1, -1)[:, ::d, ::d].reshape(B, -1, h0 * w0)
            P = torch.cat((sub, best[:, None].to(cv.dtype)), 1).softmax(dim=1)     # the extra logit is the argmax INDEX
            pos = torch.einsum("bki,kd->bdi", P[:, :-1], grid_lr) + P[:, -1:] * grid[best].permute(0, 2, 1)
        return pos.reshape(B, 2, h0, w0), best.reshape(B, h0, w0), gap

    def forward(self, im0, im1):
        im0, im1 = self.preprocess(im0.to(self.device).float()), self.preprocess(im1.to(self.device).float())
        H1, W1 = im1.shape[-2:]
        to_normalized = torch.tensor((2 / W1, 2 / H1, 1)).to(im0.device)[None, :, None, None]
        if im0.shape[-2:] == im1.shape[-2:]:
            x2, feats = self.backbone(torch.cat((im0, im1)))
            x2_0, x2_1 = x2.chunk(2)
            f0, f1 = feats.chunk(2)
        else:
            (x2_0, f0), (x2_1, f1) = self.backbone(im0), self.backbone(im1)
        self._keep("x2", torch.cat((x2_0, x2_1)) if x2_0.shape == x2_1.shape else x2_0)
        self._keep("feats", torch.cat((f0, f1)) if f0.shape == f1.shape else f0)
        coarse, best, gap = self.pos_embed(f0, f1, self.exact_softmax)
        self._keep("pos_embed", coarse)
        self._keep("gap", gap)
        state = torch.cat((coarse, torch.zeros_like(coarse[:, -1:])), 1)
        warped = F.grid_sample(f1, state.permute(0, 2, 3, 1)[..., :2], mode="bilinear", align_corners=False)
        state = state + self.head("coarse_matcher", torch.cat((f0, warped, coarse), 1)) * to_normalized
        out = {8: {"flow": state[:, :2], "certainty": state[:, 2:]}}
        up = F.interpolate(state, size=x2_0.shape[-2:], mode="bilinear", align_corners=False)
        warped = F.grid_sample(x2_1, up.permute(0, 2, 3, 1)[..., :2], mode="bilinear", align_corners=False)
        fine = up + self.head("fine_matcher", torch.cat((x2_0, warped, up[:, :2]), 1)) * to_normalized
        out[4] = {"flow": fine[:, :2], "certainty": fine[:, 2:]}
        self._keep("corresps8", state)
        self._keep("corresps4", fine)
        return out

    @torch.no_grad()
    def match(self, im0, im1):
        B, _, H0, W0 = im0.shape
        c = self.forward(im0, im1)
        flow = F.interpolate(c[4]["flow"], size=(H0, W0), mode="bilinear", align_corners=False).permute(0, 2, 3, 1)
        gx = torch.linspace(-1 + 1 / W0, 1 - 1 / W0, W0)
        gy = torch.linspace(-1 + 1 / H0, 1 - 1 / H0, H0)
        grid = torch.stack(torch.meshgrid(gx, gy, indexing="xy"), -1).float().to(flow.device).expand(B, H0, W0, 2)
        cert = F.interpolate(c[4]["certainty"], size=(H0, W0), mode="bilinear", align_corners=False)[:, 0].sigmoid()
        return torch.cat((grid, flow), -1), cert

    # the CUDA-path sampler of the reference's tiny model (fp16 KDE, no down-sampling) is RoMa's sample() with num=5000
    kde = staticmethod(RomaOracle.kde)

    def sample(self, matches, certainty, num=5000):
        return RomaOracle.sample(self, matches, certainty, num)
