"""Device sampler behind `sample()` and `sample_batched()` of both matchers (RoMa `matcher.py:598-629`, TinyRoMa `tiny.py:234-266`: the
same algorithm, certainty thresholding + two weighted draws without replacement around the fp16 Gaussian KDE)."""
from __future__ import annotations

import torch

from . import cabi
from .cache import GraphCache
from .packing import at

# Device workspace one chunk of a batched draw may take (keys, KDE workspace, intermediate draws); chunks are whole pairs, at least one
SAMPLE_CHUNK_BYTES = 2 << 30


def _draw(kde, m, c, seeds, n, repeats, num, sample_mode, sample_thresh, out=None):
    """The sampling chain for items = seeds.shape[0] draws of `repeats` per pair: m [pairs, n, 4] and c [pairs, n] are read in place,
    item i draws from pair i // repeats with the seeds of row i of `seeds` [items, 2] (int64, device).  Every item draws exactly what
    a one-item chain with its seeds draws.  Returns (m [items, k, 4], c [items, k]), written into `out` when given."""
    balanced = "balanced" in sample_mode
    thresholded = "threshold" in sample_mode
    items, dev = seeds.shape[0], c.device
    k1 = min((4 if balanced else 1) * num, n)
    k2 = min(num, k1)
    keys = torch.empty(items * n, device=dev)
    scratch = torch.empty(items * 2056, dtype=torch.int32, device=dev)
    idx1 = torch.empty(items, k1, dtype=torch.int32, device=dev)
    cabi.call("romab200_weighted_sample", "rb_sample_args", values=c, n=n, k=k1, batch=items, stride=n, seed=0, seed_dev=seeds, seed_stride=2,
              repeats=repeats, transform=cabi.SAMPLE_THRESHOLD if thresholded else cabi.SAMPLE_IDENTITY, param=float(sample_thresh),
              out_idx=idx1, out_weights=None, keys=keys, scratch=scratch)
    sel1 = idx1.sort(dim=1).values                    # the compaction order is not deterministic; the drawn SET is
    if balanced or out is None:
        good_m, w1 = torch.empty(items, k1, 4, device=dev), torch.empty(items, k1, device=dev)
    else:
        good_m, w1 = out
    cabi.call("romab200_sample_gather", "rb_sample_gather_args", matches=m, certainty=c, n=n, idx=sel1, items=items, k=k1, repeats=repeats,
              threshold=int(thresholded), thresh=float(sample_thresh), out_matches=good_m, out_certainty=w1)
    if not balanced:
        return good_m, w1
    density = kde(good_m, std=0.1, half=True).to(torch.float16).float().contiguous()     # kde.py: x.half()
    idx2 = torch.empty(items, k2, dtype=torch.int32, device=dev)
    cabi.call("romab200_weighted_sample", "rb_sample_args", values=density, n=k1, k=k2, batch=items, stride=k1, seed=0, seed_dev=at(seeds, 1),
              seed_stride=2, transform=cabi.SAMPLE_BALANCE, param=0.0, out_idx=idx2, out_weights=None, keys=keys, scratch=scratch)
    sel = idx2.sort(dim=1).values
    out_m, out_c = out if out is not None else (torch.empty(items, k2, 4, device=dev), torch.empty(items, k2, device=dev))
    cabi.call("romab200_sample_gather", "rb_sample_gather_args", matches=good_m, certainty=w1, n=k1, idx=sel, items=items, k=k2, repeats=1,
              threshold=0, thresh=0.0, out_matches=out_m, out_certainty=out_c)
    return out_m, out_c


def sample_device(cache: GraphCache, kde, matches, certainty, num, sample_mode, sample_thresh, use_cuda_graph=True):
    """Device sampler of one pair; from the third call with the same sizes on, the whole chain (two draws, sorts, gathers, KDE) is one
    CUDA-graph replay fed through static buffers, with the two seeds of a call copied to device words.  `cache` holds those
    buffers and graphs per (n, num, mode) for the owning matcher; `kde(x, std, half)` is the density kernel's wrapper."""
    dev = matches.device
    with torch.cuda.device(dev):
        n = certainty.numel()
        key = (n, num, sample_mode, float(sample_thresh), dev.index)
        entry = cache.entry(key, lambda: dict(
            m=torch.empty(1, n, 4, device=dev), c=torch.empty(1, n, device=dev), seeds=torch.zeros(1, 2, dtype=torch.int64, device=dev)),
            use_cuda_graph)
        st = entry["bufs"]
        st["m"].view(-1, 4).copy_(matches.reshape(-1, 4), non_blocking=True)
        st["c"].view(-1).copy_(certainty.reshape(-1), non_blocking=True)
        # CPU generator: follows torch.manual_seed.  A fresh pinned tensor per call: the asynchronous copy of one call must not read a
        # staging buffer that the next call has already overwritten (the caching host allocator holds it until the copy has run)
        st["seeds"].copy_(torch.randint(0, 2 ** 62, (1, 2), dtype=torch.int64).pin_memory(), non_blocking=True)
        out, replayed = cache.run(entry, lambda: _draw(kde, st["m"], st["c"], st["seeds"], n, 1, num, sample_mode, sample_thresh))
        return (out[0][0].clone(), out[1][0].clone()) if replayed else (out[0][0], out[1][0])


def check_batched(matches, certainty, num, repeats):
    """Argument rules of `sample_batched`, checked before any device work; returns the number of pairs."""
    if not isinstance(num, int) or num < 1:
        raise ValueError(f"sample_batched: num must be a positive int, got {num!r}")
    if not isinstance(repeats, int) or repeats < 1:
        raise ValueError(f"sample_batched: repeats must be a positive int, got {repeats!r}")
    if matches.dim() < 2 or matches.shape[-1] != 4 or tuple(matches.shape[:-1]) != tuple(certainty.shape):
        raise ValueError(f"sample_batched: matches [B, ..., 4] and certainty [B, ...] must share their leading shape, got "
                         f"{tuple(matches.shape)} and {tuple(certainty.shape)}")
    if certainty.numel() == 0:
        raise ValueError(f"sample_batched: empty batch or warp {tuple(certainty.shape)}")
    if matches.device != certainty.device:
        raise ValueError(f"sample_batched: matches on {matches.device} and certainty on {certainty.device}")
    if matches.dtype != torch.float32 or certainty.dtype != torch.float32:
        raise ValueError(f"sample_batched: fp32 matches and certainty expected, got {matches.dtype} and {certainty.dtype}")
    return certainty.shape[0]


def _item_bytes(n, num, balanced):
    """Device bytes one item of a batched draw allocates (keys, selection scratch, draws, gathers and the KDE workspace)."""
    k1 = min((4 if balanced else 1) * num, n)
    total = 4 * n + 4 * 2056 + k1 * (2 * 4 + 16 + 4)
    if balanced:
        splits = 16 if k1 >= 8192 else 1
        kde_ws = (splits + (k1 + 255) // 256) * k1 if splits > 1 else 0
        total += 4 * kde_ws + k1 * (4 + 2 + 4) + min(num, k1) * 2 * 4
    return total


def sample_batched(cache: GraphCache, kde, matches, certainty, num, repeats, sample_mode, sample_thresh, use_cuda_graph=True,
                   chunk_bytes=SAMPLE_CHUNK_BYTES):
    """`repeats` draws of `num` matches from each pair of matches [B, ..., 4] / certainty [B, ...] (CUDA, fp32): (m [B, repeats, k, 4],
    c [B, repeats, k]), item (b, r) bit-equal to the (b * repeats + r)-th call of a `sample_device` loop after the same seed.  One pair
    drawn once is `sample_device` itself; otherwise the chain reads the caller's tensors in place, with the launches of one chain per
    chunk of whole pairs whose workspace fits `chunk_bytes`."""
    B = certainty.shape[0]
    if B * repeats == 1:
        m, c = sample_device(cache, kde, matches[0], certainty[0], num, sample_mode, sample_thresh, use_cuda_graph)
        return m.view(1, 1, -1, 4), c.view(1, 1, -1)
    dev = matches.device
    with torch.cuda.device(dev):
        m, c = matches.contiguous().view(B, -1, 4), certainty.contiguous().view(B, -1)
        n = c.shape[1]
        k = min(num, min((4 if "balanced" in sample_mode else 1) * num, n))
        seeds = torch.randint(0, 2 ** 62, (B * repeats, 2), dtype=torch.int64).pin_memory().to(dev, non_blocking=True)
        out_m, out_c = torch.empty(B * repeats, k, 4, device=dev), torch.empty(B * repeats, k, device=dev)
        per_chunk = max(1, chunk_bytes // (repeats * _item_bytes(n, num, "balanced" in sample_mode)))
        for p0 in range(0, B, per_chunk):
            i0, i1 = p0 * repeats, min(B, p0 + per_chunk) * repeats
            _draw(kde, m[p0:p0 + per_chunk], c[p0:p0 + per_chunk], seeds[i0:i1], n, repeats, num, sample_mode, sample_thresh,
                  out=(out_m[i0:i1], out_c[i0:i1]))
        return out_m.view(B, repeats, k, 4), out_c.view(B, repeats, k)


def kde(x: torch.Tensor, std: float = 0.1, half: bool = True, symmetric: bool = True):
    """Gaussian KDE density of every row of x [n, 4] (`romab200_kde_density`, kde.py:4-12), or of each item of x [items, n, 4] on its
    own (density [items, n], every item bit-equal to a call on it alone)."""
    x = x.contiguous().float()
    items, n = (x.shape[0] if x.dim() == 3 else 1), x.shape[-2]
    out = torch.empty(x.shape[:-1], dtype=torch.float32, device=x.device)
    splits = 16 if n >= 8192 else 1
    sym = bool(half) and splits > 1 and symmetric      # every pair once: (splits + blocks of 256) * n floats of workspace
    nws = items * ((splits + (n + 255) // 256) * n if sym else splits * n)
    ws = torch.empty(nws, dtype=torch.float32, device=x.device) if splits > 1 else None
    cabi.call("romab200_kde_density", "rb_kde_args", x=x, density=out, n=n, std=std, half=int(half), workspace=ws, splits=splits,
              symmetric=int(sym), workspace_floats=nws if ws is not None else 0, batch=items)
    return out
