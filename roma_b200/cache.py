"""The activation-buffer arena and the CUDA-graph replay cache shared by RoMa's engine, TinyRoMa and the device sampler."""
from __future__ import annotations

import torch

from . import cabi


class BufferArena:
    """Activation buffers keyed by (name, shape, dtype), allocated on first use and reused, and constants keyed by the caller.
    `free()` drops the buffers and bumps `generation`: a graph recorded over them holds their raw pointers and must not replay."""

    def __init__(self, device):
        self.device, self._buf, self._const, self.generation = torch.device(device), {}, {}, 0

    def buf(self, name, shape, dtype, zero=False):
        key = (name, tuple(shape), dtype)
        if key not in self._buf:
            self._buf[key] = (torch.zeros if zero else torch.empty)(key[1], dtype=dtype, device=self.device)
        return self._buf[key]

    def const(self, key, make):
        if key not in self._const:
            self._const[key] = make().to(self.device)
        return self._const[key]

    def free(self):
        self._buf.clear()
        self.generation += 1


class GraphCache(dict):
    """Entries keyed by the caller's key, one CUDA graph each: the first call with a key runs eagerly (and allocates what its
    work allocates on first use), the second runs eagerly and then captures the same work, later calls replay the capture.
    `launches` counts the kernels launched by replays (`cabi.kernel_launches()` counts the eager ones)."""

    def __init__(self):
        super().__init__()
        self.launches = 0

    def entry(self, key, make, enabled=True, generation=0) -> dict:
        """The entry of `key`: its static buffers "bufs" from `make()` (the caller copies its inputs in, its work reads and writes
        them) and its "graph".  Made again when it was recorded under another arena `generation`; with `enabled` False made
        fresh, not kept and run eagerly."""
        e = self.get(key) if enabled else None
        if e is None or e["generation"] != generation:
            e = dict(bufs=make(), generation=generation, capture=enabled, calls=0, graph=None, out=None, launches=0)
            if enabled:
                self[key] = e
        return e

    def run(self, e: dict, fn):
        """Run `fn` (work on the current device's current stream, no host sync) or replay its capture.  Returns (what `fn`
        returned, on a replay what the captured call returned; whether this call was a replay)."""
        e["calls"] += 1
        if e["graph"] is not None:
            e["graph"].replay()
            self.launches += e["launches"]
            return e["out"], True
        out = fn()
        if e["capture"] and e["calls"] >= 2:
            torch.cuda.synchronize()
            e["graph"], launches0 = torch.cuda.CUDAGraph(), cabi.kernel_launches()
            with torch.cuda.graph(e["graph"]):
                e["out"] = fn()
            e["launches"] = cabi.kernel_launches() - launches0
        return out, False
