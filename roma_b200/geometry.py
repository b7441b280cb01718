"""Relative pose on the device: a drop-in for `romatch.utils.estimate_pose` (romatch/utils/utils.py:30-51).

The reference normalises the keypoints with the intrinsics, runs `cv2.findEssentialMat` (plain RANSAC over the five-point
solver) and `cv2.recoverPose` on one host core.  Here the same estimator runs in `csrc/pose.cu`: the same E error, threshold
test, sequential best-model replay and stopping rule, and the same chirality test.  The one intended difference is the random
stream of minimal samples (Philox4x32-10 keyed by `seed`, counter (hypothesis, pair, block); include/romab200.h), so a result
is deterministic for a given seed.  There is no CPU fallback and cv2 is never called.

    from roma_b200 import estimate_pose
    R, t, mask = estimate_pose(kpts0, kpts1, K0, K1, norm_thresh)
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import cabi

# include/romab200.h: RB_POSE_ROUND, RB_POSE_MAX_SOL, RB_POSE_MAX_SPLITS, RB_POSE_STATE
ROUND, MAX_SOL, MAX_SPLITS, STATE = 1024, 10, 16, 8


def _device():
    if not torch.cuda.is_available():
        raise RuntimeError("estimate_pose runs on the GPU only (there is no CPU fallback): no CUDA device is available")
    return torch.device("cuda", torch.cuda.current_device())


def _points(k, dev):
    t = torch.as_tensor(k) if not isinstance(k, torch.Tensor) else k
    if t.dim() != 2 or t.shape[1] != 2:
        raise ValueError(f"keypoints must be [N, 2], got {tuple(t.shape)}")
    if t.dtype not in (torch.float32, torch.float64):
        raise TypeError(f"keypoints must be float32 or float64, got {t.dtype}")
    return t.to(dev, torch.float64).contiguous()


def _intrinsics(K, batch, dev):
    t = torch.as_tensor(np.asarray(K, dtype=np.float64)) if not isinstance(K, torch.Tensor) else K.detach()
    t = t.to(dev, torch.float64)
    if t.shape == (3, 3):
        t = t.expand(batch, 3, 3)
    if tuple(t.shape) != (batch, 3, 3):
        raise ValueError(f"intrinsics must be [3, 3] or [{batch}, 3, 3], got {tuple(t.shape)}")
    return t


def _launch(x0, x1, offsets, K, max_n, norm_thresh, conf, max_iters, seed):
    """Enqueues the whole estimate on the current stream.  x0, x1: float64 [total, 2] device tensors, offsets: int64 [B + 1],
    K: float64 [B, 2, 3, 3].  With max_iters <= ROUND this is one round and reads nothing back, so it can be captured in a CUDA
    graph; each further round costs one 4-byte read of the `running` flag.  Returns the buffers (R, t, ok, mask, state,
    best_E, sample, E, nsol)."""
    dev = x0.device
    B = offsets.numel() - 1
    total = x0.shape[0]
    f64, i32 = dict(device=dev, dtype=torch.float64), dict(device=dev, dtype=torch.int32)
    buf = dict(
        xn=torch.empty(max(total, 1), 4, **f64), sample=torch.empty(B, ROUND, 5, **i32), E=torch.empty(B, ROUND, MAX_SOL, 9, **f64),
        nsol=torch.empty(B, ROUND, **i32), counts=torch.empty(B, MAX_SPLITS, MAX_SOL, ROUND, **i32), state=torch.zeros(B, STATE, **i32),
        best_E=torch.zeros(B, MAX_SOL, 9, **f64), running=torch.zeros(1, **i32), R=torch.empty(B, 3, 3, **f64), t=torch.empty(B, 3, **f64),
        ok=torch.empty(B, device=dev, dtype=torch.uint8), mask=torch.empty(max(total, 1), device=dev, dtype=torch.uint8))
    kw = dict(batch=B, x0=x0, x1=x1, offsets=offsets, K=K, max_n=int(max_n), thresh=float(norm_thresh), conf=float(conf),
              max_iters=int(max_iters), seed=int(seed) & (2 ** 64 - 1), **buf)
    rounds = (int(max_iters) + ROUND - 1) // ROUND
    for r in range(rounds):
        kw["round"] = r
        cabi.call("romab200_pose_hypotheses", "rb_pose_args", **kw)
        cabi.call("romab200_pose_score", "rb_pose_args", **kw)
        cabi.call("romab200_pose_select", "rb_pose_args", **kw)
        if r + 1 < rounds and int(buf["running"].item()) == 0:
            break
    cabi.call("romab200_pose_recover", "rb_pose_args", **kw)
    return buf


def _check_args(norm_thresh, conf, max_iters):
    if not max_iters >= 1:
        raise ValueError(f"max_iters must be >= 1, got {max_iters}")
    if not (math.isfinite(norm_thresh) and norm_thresh > 0):
        raise ValueError(f"norm_thresh must be positive, got {norm_thresh}")


def estimate_pose_batched(kpts0_list, kpts1_list, K0, K1, norm_thresh, conf=0.99999, *, max_iters=1000, seed=0):
    """`estimate_pose` for B pairs in one launch set.  kpts*_list: B arrays / tensors [N_b, 2] (ragged N); K0, K1: one [3, 3]
    for every pair or [B, 3, 3].  Pair b draws its samples from the stream keyed by (seed, b), so the result of pair b is
    bit-identical to `estimate_pose` of that pair alone when b == 0, and to the pair-b stream otherwise.
    Returns (R [B, 3, 3] float64, t [B, 3, 1] float64, ok [B] bool, masks: list of bool [N_b]); numpy keypoints give numpy
    outputs, CUDA tensors give device tensors.  ok[b] is False where `estimate_pose` returns None."""
    if len(kpts0_list) != len(kpts1_list) or len(kpts0_list) == 0:
        raise ValueError("kpts0_list and kpts1_list must be non-empty and of the same length")
    _check_args(norm_thresh, conf, max_iters)
    dev = _device()
    as_numpy = not isinstance(kpts0_list[0], torch.Tensor)
    p0 = [_points(k, dev) for k in kpts0_list]
    p1 = [_points(k, dev) for k in kpts1_list]
    for a, b in zip(p0, p1):
        if a.shape != b.shape:
            raise ValueError(f"kpts0 and kpts1 differ in shape: {tuple(a.shape)} vs {tuple(b.shape)}")
    B = len(p0)
    ns = [a.shape[0] for a in p0]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(ns)]), dtype=torch.int64, device=dev)
    K = torch.stack([_intrinsics(K0, B, dev), _intrinsics(K1, B, dev)], dim=1).contiguous()
    x0 = torch.cat(p0) if sum(ns) else torch.zeros(1, 2, dtype=torch.float64, device=dev)
    x1 = torch.cat(p1) if sum(ns) else torch.zeros(1, 2, dtype=torch.float64, device=dev)
    buf = _launch(x0, x1, offsets, K, max(ns), norm_thresh, conf, max_iters, seed)
    ok = buf["ok"].bool()
    masks = list(buf["mask"][:sum(ns)].bool().split(ns))
    R, t = buf["R"], buf["t"].view(B, 3, 1)
    if as_numpy:
        return R.cpu().numpy(), t.cpu().numpy(), ok.cpu().numpy(), [m.cpu().numpy() for m in masks]
    return R, t, ok, masks


def estimate_pose(kpts0, kpts1, K0, K1, norm_thresh, conf=0.99999, *, max_iters=1000, seed=0):
    """Drop-in for `romatch.utils.estimate_pose`: essential matrix by five-point RANSAC at threshold `norm_thresh` on the
    normalised points (OpenCV's E error, `conf`, at most `max_iters` hypotheses), then recoverPose.  Returns None when
    len(kpts0) < 5 or no model is found, otherwise (R float64 [3, 3], t float64 [3, 1], mask bool [N]) where mask holds the
    RANSAC inliers that pass the chirality test.  numpy in gives numpy out; CUDA tensors give device tensors."""
    if len(kpts0) < 5:
        return None
    R, t, ok, masks = estimate_pose_batched([kpts0], [kpts1], K0, K1, norm_thresh, conf, max_iters=max_iters, seed=seed)
    if not bool(ok[0]):
        return None
    return R[0], t[0], masks[0]
