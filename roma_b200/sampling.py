"""Device sampler behind `sample()` of both matchers (RoMa `matcher.py:598-629`, TinyRoMa `tiny.py:234-266`: the same algorithm,
certainty thresholding + two weighted draws without replacement around the fp16 Gaussian KDE)."""
from __future__ import annotations

import torch

from . import cabi
from .cache import GraphCache


def sample_device(cache: GraphCache, kde, matches, certainty, num, sample_mode, sample_thresh, use_cuda_graph=True):
    """Device sampler; from the third call with the same sizes on, the whole chain (two draws, sort, gathers, KDE) is one
    CUDA-graph replay fed through static buffers, with the two seeds of a call written to a device word.  `cache` holds those
    buffers and graphs per (n, num, mode) for the owning matcher; `kde(x, std, half)` is the density kernel's wrapper."""
    balanced = "balanced" in sample_mode
    thresholded = "threshold" in sample_mode
    dev = matches.device
    with torch.cuda.device(dev):
        n = certainty.numel()
        key = (n, num, sample_mode, float(sample_thresh), dev.index)
        k1 = min((4 if balanced else 1) * num, n)
        entry = cache.entry(key, lambda: dict(
            m=torch.empty(n, 4, device=dev), c=torch.empty(n, device=dev), seeds=torch.zeros(2, dtype=torch.int64, device=dev),
            seeds_host=torch.zeros(2, dtype=torch.int64).pin_memory(), idx1=torch.empty(k1, dtype=torch.int32, device=dev),
            idx2=torch.empty(min(num, k1), dtype=torch.int32, device=dev), keys=torch.empty(n, device=dev),
            scratch=torch.empty(2056, dtype=torch.int32, device=dev)), use_cuda_graph)
        st = entry["bufs"]
        st["m"].copy_(matches.reshape(-1, 4), non_blocking=True)
        st["c"].copy_(certainty.reshape(-1), non_blocking=True)
        st["seeds_host"].copy_(torch.randint(0, 2 ** 62, (2,), dtype=torch.int64))       # CPU generator: follows torch.manual_seed
        st["seeds"].copy_(st["seeds_host"], non_blocking=True)

        def chain():
            m, c = st["m"], st["c"]
            cabi.call("romab200_weighted_sample", "rb_sample_args", values=c, n=n, k=k1, batch=1, stride=n, seed=0, seed_dev=st["seeds"],
                      transform=cabi.SAMPLE_THRESHOLD if thresholded else cabi.SAMPLE_IDENTITY, param=float(sample_thresh),
                      out_idx=st["idx1"], out_weights=None, keys=st["keys"], scratch=st["scratch"])
            sel1 = st["idx1"].long().sort().values           # the compaction order is not deterministic; the drawn SET is
            good_matches = m[sel1]
            w1 = torch.where(c[sel1] > sample_thresh, torch.ones((), device=dev), c[sel1]) if thresholded else c[sel1]
            if not balanced:
                return good_matches, w1
            density = kde(good_matches, std=0.1, half=True).to(torch.float16).float().contiguous()     # kde.py: x.half()
            cabi.call("romab200_weighted_sample", "rb_sample_args", values=density, n=k1, k=st["idx2"].numel(), batch=1, stride=k1, seed=0,
                      seed_dev=st["seeds"][1:], transform=cabi.SAMPLE_BALANCE, param=0.0, out_idx=st["idx2"], out_weights=None, keys=st["keys"],
                      scratch=st["scratch"])
            sel = st["idx2"].long().sort().values
            return good_matches[sel], w1[sel]

        out, replayed = cache.run(entry, chain)
        return (out[0].clone(), out[1].clone()) if replayed else out


def kde(x: torch.Tensor, std: float = 0.1, half: bool = True, symmetric: bool = True):
    """Gaussian KDE density of every row of x [n, 4] (`romab200_kde_density`, kde.py:4-12)."""
    x = x.contiguous().float()
    n = x.shape[0]
    out = torch.empty(n, dtype=torch.float32, device=x.device)
    splits = 16 if n >= 8192 else 1
    sym = bool(half) and splits > 1 and symmetric      # every pair once: (splits + blocks of 256) * n floats of workspace
    nws = (splits + (n + 255) // 256) * n if sym else splits * n
    ws = torch.empty(nws, dtype=torch.float32, device=x.device) if splits > 1 else None
    cabi.call("romab200_kde_density", "rb_kde_args", x=x, density=out, n=n, std=std, half=int(half), workspace=ws, splits=splits,
              symmetric=int(sym), workspace_floats=nws if ws is not None else 0)
    return out
