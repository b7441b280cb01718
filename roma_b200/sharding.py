"""Multi-GPU sharding of independent image pairs (SURVEY §8e).

`match()` has no cross-pair dependency (BatchNorm is in eval mode, `matcher.py:790`), so a batch of pairs shards
contiguously over ranks with replicated weights and no collective on the data path.  The only communication a caller
may want is distribution of inputs that live on one rank and collection of the results — plain NCCL
scatter / gather over NVLink (25.4 MB in, 29.9 MB out per pair: ~0.07 ms at 770 GB/s against >= 25 ms of compute per
pair, so nothing is fused with compute).  One process per GPU; works with any `torch.distributed` backend (the CPU tests
use gloo with world size 2).
"""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch
import torch.distributed as dist


def shard_bounds(n_pairs: int, world: int) -> List[Tuple[int, int]]:
    """Contiguous [start, end) slice of the pair batch for every rank; the first `n % world` ranks get one more."""
    base, extra = divmod(n_pairs, world)
    out, start = [], 0
    for r in range(world):
        size = base + (1 if r < extra else 0)
        out.append((start, start + size))
        start += size
    return out


def _exchange(ops):
    """One grouped launch of point-to-point operations (ncclGroupStart/End under NCCL) and wait for all of them."""
    if ops:
        for req in dist.batch_isend_irecv(ops):
            req.wait()


def scatter_pairs(tensors: Optional[List[torch.Tensor]], n_pairs: int, shape_tail: List[Tuple[int, ...]], device, src: int = 0,
                  group=None) -> List[torch.Tensor]:
    """Rank `src` holds `tensors` (each [n_pairs, ...]); every rank receives its contiguous shard of each of them.
    `shape_tail` gives the per-pair shape of each tensor so that receivers can allocate without a metadata exchange.
    All sends / receives of a call travel as ONE grouped collective-like launch (`dist.batch_isend_irecv`)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bounds = shard_bounds(n_pairs, world)
    lo, hi = bounds[rank]
    out, ops, keep = [], [], []
    for i, tail in enumerate(shape_tail):
        if rank == src:
            full = tensors[i].to(device=device, dtype=torch.float32)
            out.append(full[lo:hi])                       # the source's own shard: a view, no copy
            for r, (a, b) in enumerate(bounds):
                if r != src and b > a:
                    piece = full[a:b].contiguous()
                    keep.append(piece)
                    ops.append(dist.P2POp(dist.isend, piece, r, group))
        else:
            recv = torch.empty((hi - lo,) + tuple(tail), dtype=torch.float32, device=device)
            if hi > lo:
                ops.append(dist.P2POp(dist.irecv, recv, src, group))
            out.append(recv)
    _exchange(ops)
    return out


def gather_results(local: List[torch.Tensor], n_pairs: int, dst: int = 0, group=None) -> Optional[List[torch.Tensor]]:
    """Inverse of `scatter_pairs` for the per-pair results (warp, certainty): returns the full tensors on `dst`."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    bounds = shard_bounds(n_pairs, world)
    if rank != dst:
        _exchange([dist.P2POp(dist.isend, t.contiguous(), dst, group) for t in local if t.shape[0] > 0])
        return None
    out, ops = [], []
    for t in local:
        full = torch.empty((n_pairs,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        for r, (a, b) in enumerate(bounds):
            if r == dst:
                full[a:b].copy_(t)
            elif b > a:
                ops.append(dist.P2POp(dist.irecv, full[a:b], r, group))
        out.append(full)
    _exchange(ops)
    return out


def wire_bytes(n_pairs: int, world: int, in_bytes_per_pair: int, out_bytes_per_pair: int, src: int = 0) -> Tuple[int, int]:
    """(scatter, gather) bytes that cross the interconnect for one sharded batch (the source keeps its own shard)."""
    lo, hi = shard_bounds(n_pairs, world)[src]
    remote = n_pairs - (hi - lo)
    return remote * in_bytes_per_pair, remote * out_bytes_per_pair


def match_sharded(model, im_A, im_B, im_A_high_res=None, im_B_high_res=None, n_pairs: Optional[int] = None, src: int = 0,
                  group=None, max_batch: Optional[int] = None, on_batch=None, pair_shapes=None):
    """`model.match` over a pair batch sharded across the process group.  Rank `src` passes the full tensors (other ranks
    pass None and `n_pairs`); returns (warp, certainty) on `src`, None elsewhere.  The per-pair input shapes the other ranks
    allocate for are the model's configured resolutions, or `pair_shapes` = ((C, H, W) of im_A, (C, H, W) of im_B) when given —
    needed for models without a configured resolution (TinyRoMa matches at the input size).  `on_batch(warp, certainty)` is
    called on every rank after each local sub-batch (e.g. to run `sample`)."""
    rank = dist.get_rank(group)
    device = model._get_device() if hasattr(model, "_get_device") else model.device
    if pair_shapes is not None:
        tails = [tuple(pair_shapes[0]), tuple(pair_shapes[1])]
    else:
        h, w = model.h_resized, model.w_resized
        tails = [(3, h, w), (3, h, w)]
    tensors = [im_A, im_B]
    if getattr(model, "upsample_preds", False):
        hu, wu = model.upsample_res
        tails += [(3, hu, wu), (3, hu, wu)]
        tensors += [im_A_high_res, im_B_high_res]
    if rank == src:
        n_pairs = im_A.shape[0]
    assert n_pairs is not None, "non-source ranks must pass n_pairs"
    shards = scatter_pairs(tensors if rank == src else None, n_pairs, tails, device, src, group)
    if shards[0].shape[0] > 0:
        # the local shard runs in sub-batches of `max_batch` pairs (bounded activation memory, one CUDA graph per shape)
        mb = max_batch or shards[0].shape[0]
        outs = []
        for a in range(0, shards[0].shape[0], mb):
            kw = dict(im_A_high_res=shards[2][a:a + mb], im_B_high_res=shards[3][a:a + mb]) if len(shards) == 4 else {}
            outs.append(model.match(shards[0][a:a + mb], shards[1][a:a + mb], **kw))
            if on_batch is not None:
                on_batch(*outs[-1])
        warp = outs[0][0] if len(outs) == 1 else torch.cat([o[0] for o in outs])
        cert = outs[0][1] if len(outs) == 1 else torch.cat([o[1] for o in outs])
    elif not hasattr(model, "get_output_resolution"):        # TinyRoMa: one warp per pixel of im_A
        warp = torch.empty((0,) + tuple(tails[0][1:]) + (4,), device=device)
        cert = torch.empty((0,) + tuple(tails[0][1:]), device=device)
    else:
        ho, wo = model.get_output_resolution()
        wout = 2 * wo if model.symmetric else wo
        warp = torch.empty(0, ho, wout, 4, device=device)
        cert = torch.empty(0, ho, wout, device=device)
    return gather_results([warp, cert], n_pairs, src, group)
