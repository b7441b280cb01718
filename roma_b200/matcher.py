"""`RegressionMatcher`: the reference's public matcher API on top of the H100 engine.

Mirrors `romatch.models.matcher.RegressionMatcher` (`romatch/models/matcher.py:550-986`): same
constructor-level attributes (mutable, as the reference's README documents), same method names,
argument meaning, return shapes/dtypes and error behaviour, so that callers (`demo/*.py`,
`romatch/benchmarks/*`) can switch implementation without edits.  The heavy lifting (`match`, `forward`,
the KDE inside `sample`) runs in the hand-written CUDA kernels behind `roma_b200.engine.Engine`; the small
geometry helpers are plain tensor arithmetic on whatever device their inputs live on.
"""
from __future__ import annotations

import math
import operator
import os
from warnings import warn

import torch
import torch.nn.functional as F
from PIL import Image

from . import cabi
from .cache import GraphCache
from .engine import Engine
from .preprocess import DeviceImage, DevicePreprocessor, open_inputs
from . import sampling
from .sampling import sample_device


class RegressionMatcher:
    def __init__(self, engine: Engine, h=448, w=448, sample_mode="threshold_balanced", upsample_preds=False,
                 symmetric=False, sample_thresh=0.05, name=None, attenuate_cert=None, upsample_res=None):
        self.engine = engine
        self.attenuate_cert = attenuate_cert
        self.name = name
        self.w_resized = w
        self.h_resized = h
        self.sample_mode = sample_mode
        self.upsample_preds = upsample_preds
        self.upsample_res = upsample_res or (14 * 16 * 6, 14 * 16 * 6)      # matcher.py:575
        self.symmetric = symmetric
        self.sample_thresh = sample_thresh
        self.training = False
        self.device_sampler = True      # sample(): weighted sampling without replacement in one kernel per draw (False: torch.multinomial)
        self.use_cuda_graph = True      # replay the whole device side of match() as one CUDA graph per input shape
        self._graphs = GraphCache()
        self._pre = None
        self._sample_graphs = GraphCache()      # static buffers + CUDA graph of the device sampler, per (n, num, mode)
        self._pair_graphs = GraphCache()        # match_pairs: encode batches and decode chunks, per size
        self._bank_version = 0                  # the engine's feature bank the match_pairs graphs were recorded over

    # ---- nn.Module-ish conveniences callers rely on ------------------------------------------------
    def train(self, mode: bool = True):
        self.training = False      # inference-only implementation; match() forces eval (matcher.py:790)
        return self

    def eval(self):
        return self.train(False)

    def to(self, *args, **kwargs):
        return self

    def _get_device(self):
        return self.engine.device

    @property
    def graph_launches(self):
        """Kernels launched through replays of the match() graphs (cabi.kernel_launches() counts eager ones)."""
        return self._graphs.launches

    def free_buffers(self):
        """Release every cached activation buffer and the CUDA graphs recorded over them."""
        self._graphs.clear()
        self._sample_graphs.clear()
        self._pair_graphs.clear()
        self.engine.free_buffers()

    def get_output_resolution(self):
        if not self.upsample_preds:
            return self.h_resized, self.w_resized
        return self.upsample_res

    # ---- dense matching -----------------------------------------------------------------------------
    def _states_to_corresps(self, states):
        return {s: {"flow": st[..., :2].permute(0, 3, 1, 2), "certainty": st[..., 2:3].permute(0, 3, 1, 2)}
                for s, st in states.items()}

    @torch.inference_mode()
    def forward(self, batch, batched=True, upsample=False, scale_factor=1):
        """{scale: {"flow" [B,2,h,w], "certainty" [B,1,h,w]}} like `RegressionMatcher.forward` (matcher.py:631-652)."""
        return self._forward(batch, False, upsample, scale_factor)

    @torch.inference_mode()
    def forward_symmetric(self, batch, batched=True, upsample=False, scale_factor=1):
        return self._forward(batch, True, upsample, scale_factor)

    def _forward(self, batch, symmetric, upsample, scale_factor):
        eng = self.engine
        im_a = batch["im_A"].to(eng.device, torch.float32)
        im_b = batch["im_B"].to(eng.device, torch.float32)
        images = torch.cat((im_a, im_b)).contiguous()
        b, scale_factor = im_a.shape[0], float(scale_factor)
        with torch.cuda.device(eng.device):
            if upsample:
                c = batch["corresps"]
                state = torch.cat((c["flow"], c["certainty"]), dim=1).permute(0, 2, 3, 1).contiguous().float()
                _, states = eng.upsample_pass(state, eng.encode_cnn(images, "up"), b, symmetric, scale_factor, keep_states=True)
            else:
                _, states = eng.coarse_pass(eng.image_stage(images), b, symmetric, scale_factor, keep_states=True)
        return self._states_to_corresps(states)

    def _preprocessor(self) -> DevicePreprocessor:
        if self._pre is None:
            self._pre = DevicePreprocessor(self.engine.device)
        return self._pre

    @torch.inference_mode()
    def match(self, im_A_input, im_B_input, *args, im_A_high_res=None, im_B_high_res=None, batched=True, device=None):
        """Dense warp and certainty (matcher.py:779-934).  Returns (warp [b,H,W*(2 if symmetric),4] fp32 in
        [-1,1], certainty [b,H,W*(2)] fp32 in [0,1]); extra positional args are ignored like the reference."""
        if not batched:
            raise ValueError("batched must be True, non-batched inference is no longer supported.")
        eng = self.engine
        if device is None:
            device = eng.device
        if torch.device(device).type != "cuda":
            raise RuntimeError("roma_b200 computes on CUDA only; device=%r" % (device,))
        ws, hs = self.w_resized, self.h_resized
        scale_factor = math.sqrt(hs * ws / (560 ** 2))
        (a_t, b_t), hi = self._device_inputs([im_A_input, im_B_input], [im_A_high_res, im_B_high_res], ("im_A", "im_B"))
        a_h, b_h = hi if hi is not None else (None, None)
        with torch.cuda.device(eng.device):
            return self._match_device(a_t, b_t, a_h, b_h, b_t.shape[0], self.symmetric, scale_factor)

    def _device_inputs(self, inputs, high_res, names):
        """The input rules `match` and `match_pairs` share.  `inputs`: paths / PIL images, or tensors [b, 3, h, w] of one size (not a
        mix); `high_res`: the caller's upsample-resolution tensors, one per input (all None, or all given); `names` name the inputs
        in error messages.  Returns ([coarse-resolution tensor [b, 3, h, w] per input], [upsample-resolution tensor per input] when
        upsample_preds, else None).  JPEG paths are decoded on the device in one launch set; path and PIL inputs are resized
        there (Pillow-exact bicubic, csrc/preprocess.cu) to (h_resized, w_resized) and to upsample_res."""
        opened = open_inputs(inputs, self.engine.device)
        hs, ws = self.h_resized, self.w_resized
        pil_route = all(isinstance(im, (Image.Image, DeviceImage)) for im in opened)
        if pil_route:
            # raw RGB bytes go up once per image (or were decoded there)
            pre = self._preprocessor()
            raws = [im.raw if isinstance(im, DeviceImage) else pre.upload(im) for im in opened]
            lo = [pre.resize_normalize(raw, (hs, ws))[None] for raw in raws]
        elif all(isinstance(im, torch.Tensor) for im in opened):
            h, w = opened[0].shape[-2:]
            assert all(im.shape[-2:] == (h, w) for im in opened), "For batched images we assume same size"
            if h != self.h_resized or self.w_resized != w:
                warn("Model resolution and batch resolution differ, may produce unexpected results")
            lo = list(opened)
        else:
            raise ValueError("Unsupported input type: " + " and ".join(f"type({nm})={type(im)!r}" for nm, im in zip(names, opened)))
        if not self.upsample_preds:
            return lo, None
        hs, ws = self.upsample_res
        if all(h is None for h in high_res):
            # the reference re-opens / re-uses the same images here (matcher.py:855-866): same bytes, already on the device
            if not isinstance(inputs[0], (str, os.PathLike)):
                for nm, x in zip(names, inputs):
                    assert isinstance(x, Image.Image), f"Unsupported input type: type({nm}_input)={type(x)!r}"
            assert pil_route, "upsample_preds without high-res tensors needs path or PIL inputs"
            return lo, [pre.resize_normalize(raw, (hs, ws))[None] for raw in raws]
        if all(h is not None for h in high_res):
            return lo, list(high_res)
        parts = [p for nm, im, h in zip(names, opened, high_res) for p in (f"{nm}={im!r}", f"{nm}_high_res={h!r}")]
        raise ValueError(f"Invalid upsample_preds and high_res inputs with {','.join(parts[:-1])} and {parts[-1]}")

    @torch.inference_mode()
    def match_pairs(self, images, pairs, images_high_res=None, *, max_batch=8, on_batch=None):
        """Dense warps of many pairs drawn from one image set, each image encoded once.

        images: a sequence of paths / PIL images (decoded and resized on the device as in `match`), or a tensor [N, 3, h, w]
        (then `images_high_res` [N, 3, H, W] is required when upsample_preds).  pairs: a [P, 2] integer tensor or a sequence of
        (i, j); pair k matches im_A = images[i_k] with im_B = images[j_k] (any order, repeats and i == j allowed).

        Returns (warp [P, H, W*(2 if symmetric), 4], certainty [P, H, W*(2)]) in pair order: pair k holds what
        match(images[i_k], images[j_k]) returns.  With `on_batch`, calls on_batch(first_pair_index, warp, certainty) for consecutive
        chunks of at most `max_batch` pairs instead and returns None; those tensors are reused by the next chunk, so they stay valid
        until the callback returns and a caller that keeps them clones them.

        Only the images some pair references are encoded, each once, in batches of at most `max_batch` (which also bounds the
        decode chunk of path inputs) into a per-image feature bank of the engine (about 0.24 GB per image at 560 -> 864 with fp32
        maps, computed from the buffer shapes); the bank is kept for later calls until free_buffers()."""
        eng = self.engine
        if int(max_batch) < 1:
            raise ValueError(f"max_batch must be positive, got {max_batch}")
        max_batch = int(max_batch)
        if isinstance(images, torch.Tensor):
            if images.dim() != 4:
                raise ValueError(f"images must be [N, 3, h, w], got shape {tuple(images.shape)}")
            n_images = images.shape[0]
        else:
            images = list(images)
            bad = [type(x) for x in images if not isinstance(x, (str, os.PathLike, Image.Image))]
            if bad:
                raise ValueError(f"Unsupported input type: images mixes paths / PIL images with {bad[0]!r}")
            n_images = len(images)
        pairs = pair_tensor(pairs, n_images)
        hi_given = images_high_res is not None
        if hi_given and (images_high_res.dim() != 4 or images_high_res.shape[0] != n_images):
            raise ValueError(f"images_high_res must be [{n_images}, 3, H, W], got shape {tuple(images_high_res.shape)}")
        if isinstance(images, torch.Tensor):
            self._device_inputs([images], [images_high_res], ("images",))      # match()'s checks of tensor inputs; no device work
            hs, ws = images.shape[-2:]
        else:
            hs, ws = self.h_resized, self.w_resized
        hu, wu = (0, 0)
        if self.upsample_preds:
            hu, wu = images_high_res.shape[-2:] if hi_given else self.upsample_res
        P = pairs.shape[0]
        ho, wo = (hu, wu) if self.upsample_preds else (hs, ws)
        wout = 2 * wo if self.symmetric else wo
        if P == 0:
            if on_batch is not None:
                return None
            return (torch.empty(0, ho, wout, 4, dtype=torch.float32, device=eng.device),
                    torch.empty(0, ho, wout, dtype=torch.float32, device=eng.device))
        plan = plan_pairs(pairs, max_batch)
        with torch.cuda.device(eng.device):
            return self._match_pairs_device(images, images_high_res, plan, (hs, ws), (hu, wu), (ho, wout), on_batch)

    def _match_pairs_device(self, images, images_high_res, plan, lo_res, hi_res, out_res, on_batch):
        eng = self.engine
        dev = eng.device
        (hs, ws), (hu, wu), (ho, wout) = lo_res, hi_res, out_res
        used, index = plan["used"], plan["index"].to(dev)
        symmetric, attenuate = self.symmetric, bool(self.attenuate_cert)
        scale_lo = math.sqrt(self.h_resized * self.w_resized / (560 ** 2))
        scale_hi = math.sqrt(self.upsample_res[0] * self.upsample_res[1] / (560 ** 2))
        use_graph = self.use_cuda_graph and eng.debug is None and eng.profile is None and eng.gemm_profile is None
        bank = eng.feature_bank(len(used), hs, ws, hu, wu)
        if eng.bank_version != self._bank_version:
            self._pair_graphs.clear()           # graphs recorded over a bank that is gone
            self._bank_version = eng.bank_version
        cap = bank["p16"].shape[0]
        slots = torch.arange(len(used), dtype=torch.int32, device=dev)
        for e0 in range(0, len(used), plan["max_batch"]):
            sel = used[e0:e0 + plan["max_batch"]]
            E = len(sel)
            key = ("encode", E, hs, ws, hu, wu, cap, eng.bank_version)
            entry = self._pair_graphs.entry(key, lambda: dict(
                images=torch.empty(E, 3, hs, ws, dtype=torch.float32, device=dev),
                images_hi=torch.empty(E, 3, hu, wu, dtype=torch.float32, device=dev) if hu else None,
                slots=torch.empty(E, dtype=torch.int32, device=dev)), use_graph, eng.generation)
            bufs = entry["bufs"]
            if isinstance(images, torch.Tensor):
                lo = [images[sel]]
                hi = [images_high_res[sel]] if hu else None
            else:
                lo, hi = self._device_inputs([images[i] for i in sel], [None] * E if images_high_res is None else
                                             [images_high_res[i:i + 1] for i in sel], [f"images[{i}]" for i in sel])
            for name, parts in (("images", lo), ("images_hi", hi if hu else [])):
                k = 0
                for t in parts:
                    bufs[name][k:k + t.shape[0]].copy_(t, non_blocking=True)
                    k += t.shape[0]
            bufs["slots"].copy_(slots[e0:e0 + E], non_blocking=True)
            self._pair_graphs.run(entry, lambda: eng.encode_images(bufs["images"], bufs["images_hi"], bufs["slots"], bank))
        n_pairs = plan["chunks"][-1][1]
        outs = None if on_batch is not None else (torch.empty(n_pairs, ho, wout, 4, dtype=torch.float32, device=dev),
                                                  torch.empty(n_pairs, ho, wout, dtype=torch.float32, device=dev))
        for k0, k1, i0, i1 in plan["chunks"]:
            P = k1 - k0
            key = ("decode", P, hs, ws, hu, wu, symmetric, attenuate, scale_lo, scale_hi, cap, eng.bank_version)
            entry = self._pair_graphs.entry(key, lambda: dict(
                index=torch.empty(2 * P, dtype=torch.int32, device=dev),
                warp=torch.empty(P, ho, wout, 4, dtype=torch.float32, device=dev),
                cert=torch.empty(P, ho, wout, dtype=torch.float32, device=dev)), use_graph, eng.generation)
            bufs = entry["bufs"]
            bufs["index"].copy_(index[i0:i1], non_blocking=True)
            self._pair_graphs.run(entry, lambda: eng.decode_pairs(bank, bufs["index"], P, symmetric, scale_lo, scale_hi, attenuate,
                                                                  bufs["warp"], bufs["cert"]))
            if on_batch is not None:
                on_batch(k0, bufs["warp"], bufs["cert"])
            else:
                outs[0][k0:k1].copy_(bufs["warp"])
                outs[1][k0:k1].copy_(bufs["cert"])
        return outs

    def _match_device(self, a_t, b_t, a_h, b_h, b, symmetric, scale_factor):
        eng = self.engine
        dev = eng.device
        hs, ws = a_t.shape[-2:]
        ho, wo = (a_h.shape[-2:] if a_h is not None else (hs, ws))
        wout = 2 * wo if symmetric else wo
        attenuate = bool(self.attenuate_cert)
        use_graph = self.use_cuda_graph and eng.debug is None and eng.profile is None and eng.gemm_profile is None
        key = (b, hs, ws, ho if a_h is not None else 0, wo if a_h is not None else 0, symmetric, attenuate, float(scale_factor),
               tuple(self.upsample_res))
        entry = self._graphs.entry(key, lambda: dict(
            images=torch.empty(2 * b, 3, hs, ws, dtype=torch.float32, device=dev),
            images_hi=torch.empty(2 * b, 3, ho, wo, dtype=torch.float32, device=dev) if a_h is not None else None,
            warp=torch.empty(b, ho, wout, 4, dtype=torch.float32, device=dev), cert=torch.empty(b, ho, wout, dtype=torch.float32, device=dev)),
            use_graph, eng.generation)
        bufs = entry["bufs"]
        bufs["images"][:b].copy_(a_t, non_blocking=True)
        bufs["images"][b:].copy_(b_t, non_blocking=True)
        if a_h is not None:
            bufs["images_hi"][:b].copy_(a_h, non_blocking=True)
            bufs["images_hi"][b:].copy_(b_h, non_blocking=True)
        sf_hi = math.sqrt(self.upsample_res[0] * self.upsample_res[1] / (560 ** 2))
        self._graphs.run(entry, lambda: eng.run_match(bufs["images"], bufs["images_hi"], b, symmetric, scale_factor, sf_hi, attenuate,
                                                      bufs["warp"], bufs["cert"]))
        if not use_graph:
            return bufs["warp"], bufs["cert"]
        return bufs["warp"].clone(), bufs["cert"].clone()

    # ---- sampling (matcher.py:598-629) ----------------------------------------------------------------
    def sample(self, matches, certainty, num=10000):
        """Certainty-thresholded, density-balanced match sampling (matcher.py:598-629).  Both weighted draws without
        replacement run on the device (`romab200_weighted_sample`: exponential race + radix select, the certainty
        thresholding and the density balancing fused into the key computation) and the 4*num x 4*num Gaussian KDE in
        `romab200_kde_density` without materialising the matrix; the seeds of the two draws come from torch's CPU generator,
        so `torch.manual_seed` makes the result reproducible.  With `device_sampler = False` the two `torch.multinomial`
        calls of the reference are used instead (same distribution, torch's RNG stream)."""
        if self.device_sampler and matches.is_cuda:
            return self._sample_device(matches, certainty, num)
        if "threshold" in self.sample_mode:
            upper_thresh = self.sample_thresh
            certainty = certainty.clone()
            certainty[certainty > upper_thresh] = 1
        matches, certainty = matches.reshape(-1, 4), certainty.reshape(-1)
        expansion_factor = 4 if "balanced" in self.sample_mode else 1
        good_samples = torch.multinomial(certainty, num_samples=min(expansion_factor * num, len(certainty)), replacement=False)
        good_matches, good_certainty = matches[good_samples], certainty[good_samples]
        if "balanced" not in self.sample_mode:
            return good_matches, good_certainty
        if good_matches.device.type != "cuda":
            raise RuntimeError("roma_b200.sample needs CUDA tensors (no CPU fallback)")
        with torch.cuda.device(good_matches.device):
            density = self.engine.kde(good_matches, std=0.1, half=True).to(torch.float16)   # kde.py: x.half()
        p = 1 / (density + 1)
        p[density < 10] = 1e-7      # at least ~10 perfect neighbours, as in the reference
        balanced_samples = torch.multinomial(p, num_samples=min(num, len(good_certainty)), replacement=False)
        return good_matches[balanced_samples], good_certainty[balanced_samples]

    def _sample_device(self, matches, certainty, num):
        return sample_device(self._sample_graphs, self.engine.kde, matches, certainty, num, self.sample_mode, self.sample_thresh,
                             self.use_cuda_graph)

    def sample_batched(self, matches, certainty, num=10000, *, repeats=1, chunk_bytes=sampling.SAMPLE_CHUNK_BYTES):
        """`repeats` samples of every pair of a batched warp in one call: matches [B, ..., 4] and certainty [B, ...] (fp32, as `match()`
        returns them) -> (m [B, repeats, k, 4], c [B, repeats, k]), k being what one `sample(matches[b], certainty[b], num)` returns.
        After the same `torch.manual_seed` the result equals, element for element, `sample(matches[b], certainty[b], num)` called for
        b in range(B), r in range(repeats) in that order (the seeds of call b * repeats + r are row b * repeats + r of one CPU
        `torch.randint(0, 2**62, (B * repeats, 2))`).  The device chain reads the caller's tensors in place, in chunks of whole pairs
        whose workspace fits `chunk_bytes`, and launches the same kernels for any B and repeats.  With `device_sampler = False` or
        CPU tensors it is that `sample()` loop."""
        B = sampling.check_batched(matches, certainty, num, repeats)
        if not (self.device_sampler and matches.is_cuda):
            outs = [self.sample(matches[b], certainty[b], num) for b in range(B) for _ in range(repeats)]
            return (torch.stack([m for m, _ in outs]).view(B, repeats, -1, 4), torch.stack([c for _, c in outs]).view(B, repeats, -1))
        return sampling.sample_batched(self._sample_graphs, self.engine.kde, matches, certainty, num, repeats, self.sample_mode,
                                       self.sample_thresh, self.use_cuda_graph, chunk_bytes)

    # ---- small geometry helpers (matcher.py:672-773) ---------------------------------------------------
    def _to_pixel_coordinates(self, coords, H, W):
        return torch.stack((W / 2 * (coords[..., 0] + 1), H / 2 * (coords[..., 1] + 1)), dim=-1)

    def to_pixel_coordinates(self, coords, H_A, W_A, H_B=None, W_B=None):
        if coords.shape[-1] == 2:
            return self._to_pixel_coordinates(coords, H_A, W_A)
        if isinstance(coords, (list, tuple)):
            kpts_A, kpts_B = coords[0], coords[1]
        else:
            kpts_A, kpts_B = coords[..., :2], coords[..., 2:]
        return self._to_pixel_coordinates(kpts_A, H_A, W_A), self._to_pixel_coordinates(kpts_B, H_B, W_B)

    def to_normalized_coordinates(self, coords, H_A, W_A, H_B, W_B):
        if isinstance(coords, (list, tuple)):
            kpts_A, kpts_B = coords[0], coords[1]
        else:
            kpts_A, kpts_B = coords[..., :2], coords[..., 2:]
        kpts_A = torch.stack((2 / W_A * kpts_A[..., 0] - 1, 2 / H_A * kpts_A[..., 1] - 1), dim=-1)
        kpts_B = torch.stack((2 / W_B * kpts_B[..., 0] - 1, 2 / H_B * kpts_B[..., 1] - 1), dim=-1)
        return kpts_A, kpts_B

    def conf_from_fb_consistency(self, flow_forward, flow_backward, th=2):
        has_batch = flow_forward.dim() != 3
        if not has_batch:
            flow_forward, flow_backward = flow_forward[None], flow_backward[None]
        H, W = flow_forward.shape[-3:-1]
        th_n = 2 * th / max(H, W)
        xs = torch.linspace(-1 + 1 / W, 1 - 1 / W, W)
        ys = torch.linspace(-1 + 1 / H, 1 - 1 / H, H)
        coords = torch.stack(torch.meshgrid(xs, ys, indexing="xy"), dim=-1).to(flow_forward.device)
        coords_fb = F.grid_sample(flow_backward.permute(0, 3, 1, 2), flow_forward, align_corners=False,
                                  mode="bilinear").permute(0, 2, 3, 1)
        in_th = ((coords - coords_fb).norm(dim=-1) < th_n).float()
        return in_th if has_batch else in_th[0]

    def match_keypoints(self, x_A, x_B, warp, certainty, return_tuple=True, return_inds=False, max_dist=0.005, cert_th=0):
        """Mutual nearest neighbours of the keypoints x_A carried through the warp and the keypoints x_B (matcher.py:732-773).
        fp32 CUDA inputs of the expected shapes run on the device (`romab200_keypoints_*`) in O(N_A + N_B) memory, with the
        exact-difference distance sqrt(dx² + dy²) where `torch.cdist` expands ‖a‖² + ‖b‖² − 2a·b; everything else runs the
        reference's torch statement."""
        if _keypoints_on_device(x_A, x_B, warp, certainty):
            inds_A, inds_B = _match_keypoints_device(x_A, x_B, warp, certainty, max_dist, cert_th)
        else:
            x_A_to_B = F.grid_sample(warp[..., -2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False,
                                     mode="bilinear")[0, :, 0].mT
            cert_A_to_B = F.grid_sample(certainty[None, None, ...], x_A[None, None], align_corners=False,
                                        mode="bilinear")[0, 0, 0]
            D = torch.cdist(x_A_to_B, x_B)
            mutual = (D == D.min(dim=-1, keepdim=True).values) * (D == D.min(dim=-2, keepdim=True).values)
            inds_A, inds_B = torch.nonzero(mutual * (cert_A_to_B[:, None] > cert_th) * (D < max_dist), as_tuple=True)
        if return_tuple:
            return (inds_A, inds_B) if return_inds else (x_A[inds_A], x_B[inds_B])
        if return_inds:
            return torch.cat((inds_A, inds_B), dim=-1)
        return torch.cat((x_A[inds_A], x_B[inds_B]), dim=-1)

    def visualize_warp(self, warp, certainty, im_A=None, im_B=None, im_A_path=None, im_B_path=None, device="cuda",
                       symmetric=True, save_path=None, unnormalize=False):
        import numpy as np
        H, W2, _ = warp.shape
        W = W2 // 2 if symmetric else W2
        if im_A is None:
            im_A, im_B = Image.open(im_A_path).convert("RGB"), Image.open(im_B_path).convert("RGB")
        if not isinstance(im_A, torch.Tensor):
            im_A, im_B = im_A.resize((W, H)), im_B.resize((W, H))
            x_B = (torch.tensor(np.array(im_B)) / 255).to(device).permute(2, 0, 1)
            x_A = (torch.tensor(np.array(im_A)) / 255).to(device).permute(2, 0, 1) if symmetric else None
        else:
            x_A, x_B = (im_A if symmetric else None), im_B
        im_A_transfer = F.grid_sample(x_B[None], warp[:, :W, 2:][None], mode="bilinear", align_corners=False)[0]
        if symmetric:
            im_B_transfer = F.grid_sample(x_A[None], warp[:, W:, :2][None], mode="bilinear", align_corners=False)[0]
            warp_im = torch.cat((im_A_transfer, im_B_transfer), dim=2)
            white_im = torch.ones((H, 2 * W), device=device)
        else:
            warp_im, white_im = im_A_transfer, torch.ones((H, W), device=device)
        vis_im = certainty * warp_im + (1 - certainty) * white_im
        if save_path is not None:
            arr = vis_im
            if unnormalize:
                mean = torch.tensor([0.485, 0.456, 0.406], device=arr.device)[:, None, None]
                std = torch.tensor([0.229, 0.224, 0.225], device=arr.device)[:, None, None]
                arr = arr * std + mean
            arr = (arr.clamp(0, 1) * 255).byte().permute(1, 2, 0).cpu().numpy()
            Image.fromarray(arr).save(save_path)
        return vis_im


def pair_tensor(pairs, n_images: int) -> torch.Tensor:
    """`pairs` of match_pairs as an int64 [P, 2] CPU tensor.  ValueError for anything but a [P, 2] integer tensor or a sequence of
    (i, j) integers, IndexError for an index outside [0, n_images)."""
    if isinstance(pairs, torch.Tensor):
        if pairs.dtype.is_floating_point or pairs.dtype.is_complex or pairs.dtype == torch.bool:
            raise ValueError(f"pairs must hold integers, got {pairs.dtype}")
        t = pairs.detach().to("cpu", torch.int64)
    else:
        rows = []
        for p in pairs:
            try:
                i, j = p
                rows.append((operator.index(i), operator.index(j)))
            except (TypeError, ValueError):
                raise ValueError(f"pairs must be (i, j) pairs of integers, got {p!r}") from None
        t = torch.tensor(rows, dtype=torch.int64).reshape(-1, 2)
    if t.dim() != 2 or t.shape[1] != 2:
        raise ValueError(f"pairs must be [P, 2], got shape {tuple(t.shape)}")
    if t.numel() and (int(t.min()) < 0 or int(t.max()) >= n_images):
        bad = t[(t < 0) | (t >= n_images)][0].item()
        raise IndexError(f"pairs holds image index {bad}, outside [0, {n_images})")
    return t


def plan_pairs(pairs: torch.Tensor, max_batch: int) -> dict:
    """Schedule of match_pairs for [P, 2] pairs (P > 0): `used`, the referenced images in ascending order (bank row k holds image
    used[k]; they are encoded in batches of max_batch in that order); `chunks`, (first pair, end pair, first and end entry of
    `index`) of the decode chunks of at most max_batch pairs; `index`, int32, the bank rows of every chunk's images in
    [A_1..A_P | B_1..B_P] order, chunk after chunk."""
    used, rows = torch.unique(pairs.flatten(), return_inverse=True)
    rows = rows.view(-1, 2).to(torch.int32)
    index, chunks = [], []
    for k0 in range(0, pairs.shape[0], max_batch):
        k1 = min(pairs.shape[0], k0 + max_batch)
        index += [rows[k0:k1, 0], rows[k0:k1, 1]]
        chunks.append((k0, k1, 2 * k0, 2 * k1))
    return dict(used=used.tolist(), index=torch.cat(index), chunks=chunks, max_batch=max_batch)


def _keypoints_on_device(x_A, x_B, warp, certainty) -> bool:
    """The inputs `match_keypoints` runs on the device: fp32 CUDA tensors on one device, points [N, 2], warp [H, W, >= 2],
    certainty [H', W'] (non-empty maps)."""
    ts = (x_A, x_B, warp, certainty)
    if not all(isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 for t in ts):
        return False
    if len({t.device for t in ts}) != 1:
        return False
    return (x_A.dim() == 2 and x_A.shape[1] == 2 and x_B.dim() == 2 and x_B.shape[1] == 2 and warp.dim() == 3 and warp.shape[-1] >= 2
            and warp.numel() > 0 and certainty.dim() == 2 and certainty.numel() > 0)


def _match_keypoints_device(x_A, x_B, warp, certainty, max_dist, cert_th):
    """(inds_A, inds_B) int64 of the mutual nearest neighbours, row-major like torch.nonzero.  One host read: the match count."""
    if x_A.shape[0] == 0 or x_B.shape[0] == 0:
        raise IndexError("min(): Expected reduction dim to have non-zero size.")      # what the torch statement's D.min raises
    x_A_to_B, cert_A = _keypoints_sample_device(x_A, warp, certainty)
    return _mutual_nn_device(x_A_to_B, cert_A, x_B, max_dist, cert_th)


def _keypoints_sample_device(x_A, warp, certainty):
    """(x_A_to_B [N, 2], cert_A [N]): the two grid samples of match_keypoints (matcher.py:743-754) in one kernel; warp and
    certainty are read in place through their strides."""
    n_a, dev = x_A.shape[0], x_A.device
    with torch.cuda.device(dev):
        x_A = x_A.contiguous()
        w2 = warp[..., -2:]
        x_A_to_B = torch.empty(n_a, 2, dtype=torch.float32, device=dev)
        cert_A = torch.empty(n_a, dtype=torch.float32, device=dev)
        cabi.call("romab200_keypoints_sample", "rb_keypoints_sample_args", x=x_A, n=n_a,
                  warp=w2, warp_h=w2.shape[0], warp_w=w2.shape[1], warp_ld_row=w2.stride(0), warp_ld_px=w2.stride(1), warp_ld_ch=w2.stride(2),
                  cert=certainty, cert_h=certainty.shape[0], cert_w=certainty.shape[1], cert_ld_row=certainty.stride(0),
                  cert_ld_px=certainty.stride(1), x_to_B=x_A_to_B, cert_out=cert_A)
    return x_A_to_B, cert_A


def _mutual_nn_device(x_A_to_B, cert_A, x_B, max_dist, cert_th):
    """(inds_A, inds_B) of the mutual nearest neighbours under the exact-difference distance (include/romab200.h)."""
    n_a, n_b, dev = x_A_to_B.shape[0], x_B.shape[0], x_B.device
    with torch.cuda.device(dev):
        x_B = x_B.contiguous()
        workspace = torch.empty(17 * (n_a + n_b), dtype=torch.float32, device=dev)
        offsets = torch.empty(n_a + 1, dtype=torch.int64, device=dev)
        kw = dict(x_A_to_B=x_A_to_B, cert_A=cert_A, x_B=x_B, n_a=n_a, n_b=n_b, cert_th=float(cert_th), max_dist=float(max_dist),
                  workspace=workspace, workspace_floats=workspace.numel(), offsets=offsets)
        cabi.call("romab200_keypoints_mnn_count", "rb_keypoints_mnn_args", **kw)
        total = int(offsets[n_a].item())
        inds = torch.empty(2, total, dtype=torch.int64, device=dev)
        if total:
            cabi.call("romab200_keypoints_mnn_emit", "rb_keypoints_mnn_args", inds_A=inds[0], inds_B=inds[1], **kw)
    return inds[0], inds[1]
