"""Two-view geometry on the device: relative pose, a drop-in for `romatch.utils.estimate_pose` (romatch/utils/utils.py:30-51),
and homographies, a drop-in for the `cv2.findHomography` call of the HPatches harness.

The reference normalises the keypoints with the intrinsics, runs `cv2.findEssentialMat` (plain RANSAC over the five-point
solver) and `cv2.recoverPose` on one host core.  Here the same estimator runs in `csrc/pose.cu`: the same E error, threshold
test, sequential best-model replay and stopping rule, and the same chirality test.  The one intended difference is the random
stream of minimal samples (Philox4x32-10 keyed by `seed`, counter (hypothesis, pair, block); include/romab200.h), so a result
is deterministic for a given seed.  There is no CPU fallback and cv2 is never called.

    from roma_b200 import estimate_pose
    R, t, mask = estimate_pose(kpts0, kpts1, K0, K1, norm_thresh)

`find_homography` runs OpenCV 4.13's `findHomography(..., RANSAC)` in `csrc/homography.cu`: the same subset checks, normalised
four-point solver, float32 reprojection error, sequential best-model replay and stopping rule, and least-squares refinement of
the final model.  Again only the stream of minimal samples differs (Philox4x32-10 keyed by `seed`; include/romab200.h).

    from roma_b200 import find_homography, RANSAC
    H, mask = find_homography(pos_a, pos_b, RANSAC, 3.0, confidence=0.99999)

`find_fundamental` replaces the `cv2.findFundamentalMat(..., cv2.USAC_MAGSAC, ...)` call of the reference's usage example with
MAGSAC++ over seven-point samples in `csrc/fundamental.cu`.  OpenCV's USAC internals are not restated; the estimator is defined
in include/romab200.h and DESIGN.md and agrees with cv2 statistically.

    from roma_b200 import find_fundamental, USAC_MAGSAC
    F, mask = find_fundamental(kptsA, kptsB, ransacReprojThreshold=0.2, method=USAC_MAGSAC, confidence=0.999999, maxIters=10000)
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import cabi

# include/romab200.h: RB_POSE_ROUND, RB_POSE_MAX_SOL, RB_POSE_MAX_SPLITS, RB_POSE_STATE
ROUND, MAX_SOL, MAX_SPLITS, STATE = 1024, 10, 16, 8


def _device(what="estimate_pose"):
    if not torch.cuda.is_available():
        raise RuntimeError(f"{what} runs on the GPU only (there is no CPU fallback): no CUDA device is available")
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
              max_iters=int(max_iters), seed=int(seed) & (2 ** 64 - 1), round=0, **buf)
    _ransac_rounds("pose", "rb_pose_args", kw, ROUND)
    cabi.call("romab200_pose_recover", "rb_pose_args", **kw)
    return buf


def _ransac_rounds(prefix, struct, kw, round_size):
    """Enqueues the hypotheses -> score -> select rounds of `romab200_<prefix>_*`.  A round after the first runs only when the
    previous select left the `running` flag set, which costs one 4-byte read."""
    rounds = (kw["max_iters"] + round_size - 1) // round_size
    for r in range(rounds):
        for stage in ("hypotheses", "score", "select"):
            cabi.call(f"romab200_{prefix}_{stage}", struct, **{**kw, "round": r})
        if r + 1 < rounds and int(kw["running"].item()) == 0:
            break


def _pack_pairs(a_list, b_list, to_points, what, list_names, point_names):
    """Validates two lists of per-pair point sets and packs them for the device: returns (a, b, offsets int64 [B + 1], ns) with
    a and b the concatenated points of every pair (one zero row when there are none, so the buffers are never empty)."""
    if len(a_list) != len(b_list) or len(a_list) == 0:
        raise ValueError(f"{list_names[0]} and {list_names[1]} must be non-empty and of the same length")
    dev = _device(what)
    pa = [to_points(p, dev) for p in a_list]
    pb = [to_points(p, dev) for p in b_list]
    for a, b in zip(pa, pb):
        if a.shape != b.shape:
            raise ValueError(f"{point_names[0]} and {point_names[1]} differ in shape: {tuple(a.shape)} vs {tuple(b.shape)}")
    ns = [a.shape[0] for a in pa]
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(ns)]), dtype=torch.int64, device=dev)
    if not sum(ns):
        pa = pb = [torch.zeros(1, 2, dtype=pa[0].dtype, device=dev)]
    return torch.cat(pa), torch.cat(pb), offsets, ns


def _outputs(as_numpy, *outs):
    """The estimators' return: device tensors as they are, or (for numpy inputs) host arrays; a list is converted item by item."""
    if not as_numpy:
        return outs
    return tuple([m.cpu().numpy() for m in o] if isinstance(o, list) else o.cpu().numpy() for o in outs)


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
    _check_args(norm_thresh, conf, max_iters)
    x0, x1, offsets, ns = _pack_pairs(kpts0_list, kpts1_list, _points, "estimate_pose", ("kpts0_list", "kpts1_list"), ("kpts0", "kpts1"))
    B, dev = len(ns), offsets.device
    K = torch.stack([_intrinsics(K0, B, dev), _intrinsics(K1, B, dev)], dim=1).contiguous()
    buf = _launch(x0, x1, offsets, K, max(ns), norm_thresh, conf, max_iters, seed)
    masks = list(buf["mask"][:sum(ns)].bool().split(ns))
    return _outputs(not isinstance(kpts0_list[0], torch.Tensor), buf["R"], buf["t"].view(B, 3, 1), buf["ok"].bool(), masks)


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


# ---- homographies --------------------------------------------------------------------------------------------------------
RANSAC = 8                      # cv2.RANSAC
# include/romab200.h: RB_HOMOG_ROUND, RB_HOMOG_MAX_SPLITS, RB_HOMOG_STATE
HOMOG_ROUND, HOMOG_MAX_SPLITS, HOMOG_STATE = 2048, 32, 8
# cv2's other findHomography methods, which are not restated here
_HOMOG_UNSUPPORTED = {4: "LMEDS", 16: "RHO", 32: "USAC_DEFAULT", 33: "USAC_PARALLEL", 34: "USAC_FM_8PTS", 35: "USAC_FAST",
                      36: "USAC_ACCURATE", 37: "USAC_PROSAC", 38: "USAC_MAGSAC"}


def _homog_points(p, dev):
    """[N, 2] or [N, 1, 2] points -> float32 [N, 2] on `dev`, rounded to float32 first as cv2 does."""
    t = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p))
    if t.dim() == 3 and t.shape[1] == 1:
        t = t[:, 0]
    if t.dim() != 2 or t.shape[1] != 2:
        raise ValueError(f"points must be [N, 2] or [N, 1, 2], got {tuple(t.shape)}")
    if t.dtype.is_complex or t.dtype == torch.bool:
        raise TypeError(f"points must be real numbers, got {t.dtype}")
    return t.to(torch.float32).to(dev).contiguous()


def _homog_args(method, thr, conf, max_iters):
    """Mirrors cv2.findHomography's argument handling; returns (method, threshold, confidence, maxIters) as the estimator uses them."""
    method = int(method)
    if method in _HOMOG_UNSUPPORTED:
        raise NotImplementedError(f"find_homography implements method 0 and RANSAC only, not {_HOMOG_UNSUPPORTED[method]}")
    if method not in (0, RANSAC):
        raise ValueError(f"unknown estimation method {method}")
    thr = float(thr)
    if thr <= 0:                # OpenCV substitutes its default threshold
        thr = 3.0
    conf = float(conf)
    if method == RANSAC and not 0 < conf < 1:
        raise ValueError(f"confidence must lie in (0, 1), got {conf}")
    return method, thr, conf, max(int(max_iters), 1)


def _homog_launch(src, dst, offsets, max_n, method, thr, conf, max_iters, seed):
    """Enqueues the whole estimate on the current stream.  src, dst: float32 [total, 2] device tensors, offsets: int64 [B + 1].
    With max_iters <= HOMOG_ROUND this is one round and reads nothing back, so it can be captured in a CUDA graph; each further
    round costs one 4-byte read of the `running` flag.  Returns the buffers (out_H, ok, mask, state, best_H, sample, attempts,
    status, H, counts)."""
    dev = src.device
    B = offsets.numel() - 1
    total = src.shape[0]
    f64, i32 = dict(device=dev, dtype=torch.float64), dict(device=dev, dtype=torch.int32)
    ransac = method == RANSAC
    R = HOMOG_ROUND if ransac else 1
    buf = dict(
        sample=torch.empty(B, R, 4, **i32), attempts=torch.empty(B, R, **i32), status=torch.empty(B, R, **i32),
        H=torch.empty(B, R, 9, **f64), counts=torch.empty(B, HOMOG_MAX_SPLITS if ransac else 1, R, **i32),
        state=torch.zeros(B, HOMOG_STATE, **i32), best_H=torch.zeros(B, 9, **f64), running=torch.zeros(1, **i32),
        out_H=torch.empty(B, 9, **f64), ok=torch.empty(B, device=dev, dtype=torch.uint8),
        mask=torch.empty(max(total, 1), device=dev, dtype=torch.uint8))
    kw = dict(batch=B, src=src, dst=dst, offsets=offsets, max_n=int(max_n), thresh=float(thr), conf=float(conf), max_iters=int(max_iters),
              method=int(method), seed=int(seed) & (2 ** 64 - 1), round=0, **buf)
    if ransac:
        _ransac_rounds("homography", "rb_homography_args", kw, HOMOG_ROUND)
    cabi.call("romab200_homography_refine", "rb_homography_args", **kw)
    return buf


def find_homography_batched(src_list, dst_list, method=RANSAC, ransacReprojThreshold=3, maxIters=2000, confidence=0.995, *, seed=0):
    """`find_homography` for B pairs in one launch set.  src_list, dst_list: B arrays / tensors [N_b, 2] or [N_b, 1, 2] (ragged N).
    Pair b draws its samples from the stream keyed by (seed, b), so pair 0 is bit-identical to `find_homography` of that pair alone.
    Returns (H [B, 3, 3] float64, ok [B] bool, masks: list of uint8 [N_b, 1]); numpy inputs give numpy outputs, tensors give
    device tensors.  ok[b] is False where `find_homography` returns None, and for pairs of fewer than 4 points (mask all zero);
    H[b] is zero there."""
    method, thr, conf, max_iters = _homog_args(method, ransacReprojThreshold, confidence, maxIters)
    src, dst, offsets, ns = _pack_pairs(src_list, dst_list, _homog_points, "find_homography", ("src_list", "dst_list"),
                                        ("srcPoints", "dstPoints"))
    buf = _homog_launch(src, dst, offsets, max(ns), method, thr, conf, max_iters, seed)
    masks = [m.view(-1, 1) for m in buf["mask"][:sum(ns)].split(ns)]
    return _outputs(not isinstance(src_list[0], torch.Tensor), buf["out_H"].view(len(ns), 3, 3), buf["ok"].bool(), masks)


def find_homography(srcPoints, dstPoints, method=0, ransacReprojThreshold=3, mask=None, maxIters=2000, confidence=0.995, *, seed=0):
    """Drop-in for `cv2.findHomography` with method 0 (least squares over all points) or RANSAC: the same signature, defaults and
    return form.  Returns (H float64 [3, 3], mask uint8 [N, 1]): H is refined (normalised DLT, then Levenberg-Marquardt) on the
    inliers of the best RANSAC hypothesis, and mask holds the inliers of the refined H, as cv2 4.13 returns them (all ones for 4
    points); (None, zeros) when no model is found.  `mask` is accepted and
    ignored, as in cv2's Python binding.  numpy in gives numpy out; tensors give device tensors.  Raises ValueError for fewer
    than 4 points and NotImplementedError for LMEDS, RHO and the USAC methods."""
    del mask
    method, thr, conf, max_iters = _homog_args(method, ransacReprojThreshold, confidence, maxIters)
    n = len(srcPoints)
    if n < 4 or len(dstPoints) != n:
        raise ValueError(f"find_homography needs the same number (>= 4) of source and destination points, got {n} and {len(dstPoints)}")
    H, ok, masks = find_homography_batched([srcPoints], [dstPoints], method, thr, max_iters, conf, seed=seed)
    if not bool(ok[0]):
        return None, masks[0]
    return H[0], masks[0]


# ---- fundamental matrices ------------------------------------------------------------------------------------------------
USAC_MAGSAC = 38                # cv2.USAC_MAGSAC
# include/romab200.h: RB_FUND_ROUND, RB_FUND_MODELS, RB_FUND_SLICE, RB_FUND_TABLE, RB_FUND_STATE
FUND_ROUND, FUND_MODELS, FUND_SLICE, FUND_TABLE, FUND_STATE = 1024, 3, 512, 1024, 8
# cv2's other findFundamentalMat methods, which are not restated here
_FUND_UNSUPPORTED = {1: "FM_7POINT", 2: "FM_8POINT", 4: "FM_LMEDS", 8: "FM_RANSAC", 32: "USAC_DEFAULT", 33: "USAC_PARALLEL",
                     34: "USAC_FM_8PTS", 35: "USAC_FAST", 36: "USAC_ACCURATE", 37: "USAC_PROSAC"}
# MAGSAC++ with 4 degrees of freedom (a point correspondence) and sigma_max = ransacReprojThreshold: the loss reaches its outlier
# value at k sigma_max, k^2 the 0.99 quantile of chi^2 with 4 degrees of freedom (include/romab200.h: RB_FUND_K2)
MAGSAC_K2 = 13.276704135987622


def _gamma_upper_3_2(x):
    """Gamma(3/2, x), the upper incomplete gamma function (not regularised)."""
    return math.sqrt(x) * math.exp(-x) + 0.5 * math.sqrt(math.pi) * math.erfc(math.sqrt(x))


def _gamma_lower_5_2(x):
    """gamma(5/2, x), the lower incomplete gamma function (not regularised)."""
    return 0.75 * math.sqrt(math.pi) - (1.5 * _gamma_upper_3_2(x) + x * math.sqrt(x) * math.exp(-x))


def magsac_tables():
    """The MAGSAC++ loss and weight of a residual r at q = r^2 / (k sigma_max)^2 = i / FUND_TABLE, i = 0 .. FUND_TABLE: float64
    [2, FUND_TABLE + 1].  With x = r^2 / (2 sigma_max^2) = q k^2 / 2 and x_k = k^2 / 2 (DESIGN.md):
        loss(q)   = (gamma(5/2, x) + x (Gamma(3/2, x) - Gamma(3/2, x_k))) / gamma(5/2, x_k)     0 at r = 0, 1 at r = k sigma_max
        weight(q) = (Gamma(3/2, x) - Gamma(3/2, x_k)) / (Gamma(3/2, 0) - Gamma(3/2, x_k))        1 at r = 0, 0 at r = k sigma_max
    which are the paper's sigma-marginalised loss and weight, each divided by its value at the end of its range."""
    xk = 0.5 * MAGSAC_K2
    gk, lk = _gamma_upper_3_2(xk), _gamma_lower_5_2(xk)
    g0 = 0.5 * math.sqrt(math.pi)
    out = np.empty((2, FUND_TABLE + 1))
    for i in range(FUND_TABLE + 1):
        x = xk * i / FUND_TABLE
        g = _gamma_upper_3_2(x)
        out[0, i] = (_gamma_lower_5_2(x) + x * (g - gk)) / lk
        out[1, i] = (g - gk) / (g0 - gk)
    out[:, 0] = (0.0, 1.0)
    out[:, -1] = (1.0, 0.0)
    return out


_TABLES = {}


def _magsac_tables_on(dev):
    """magsac_tables() on `dev`, uploaded once per device (so that a CUDA graph can capture the estimate)."""
    if dev not in _TABLES:
        _TABLES[dev] = torch.tensor(magsac_tables(), dtype=torch.float64, device=dev)
    return _TABLES[dev]


def _fund_points(p, dev):
    """[N, 2] or [N, 1, 2] real points -> float64 [N, 2] on `dev`."""
    t = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p))
    if t.dim() == 3 and t.shape[1] == 1:
        t = t[:, 0]
    if t.dim() != 2 or t.shape[1] != 2:
        raise ValueError(f"points must be [N, 2] or [N, 1, 2], got {tuple(t.shape)}")
    if t.dtype.is_complex or t.dtype == torch.bool:
        raise TypeError(f"points must be real numbers, got {t.dtype}")
    return t.to(torch.float64).to(dev).contiguous()


def _fund_args(method, thr, conf, max_iters):
    """Mirrors cv2.findFundamentalMat's argument checks for USAC_MAGSAC; returns (threshold, confidence, maxIters)."""
    method = int(method)
    if method in _FUND_UNSUPPORTED:
        raise NotImplementedError(f"find_fundamental implements USAC_MAGSAC only, not {_FUND_UNSUPPORTED[method]}")
    if method != USAC_MAGSAC:
        raise ValueError(f"unknown estimation method {method}")
    thr, conf = float(thr), float(conf)
    if not (math.isfinite(thr) and thr > 0):
        raise ValueError(f"ransacReprojThreshold must be positive, got {thr}")
    if not 0 < conf < 1:
        raise ValueError(f"confidence must lie in (0, 1), got {conf}")
    if int(max_iters) < 1:
        raise ValueError(f"maxIters must be >= 1, got {max_iters}")
    return thr, conf, int(max_iters)


def _fund_launch(x0, x1, offsets, max_n, thr, conf, max_iters, seed):
    """Enqueues the whole estimate on the current stream.  x0, x1: float64 [total, 2] device tensors, offsets: int64 [B + 1].
    With max_iters <= FUND_ROUND this is one round and reads nothing back, so it can be captured in a CUDA graph; each further
    round costs one 4-byte read of the `running` flag.  Returns the buffers (out_F, ok, mask, state, best_F, best_loss, norm, xn,
    sample, nmod, F, counts, losses)."""
    dev = x0.device
    B = offsets.numel() - 1
    total = x0.shape[0]
    S = max(1, -(-int(max_n) // FUND_SLICE))
    f64, i32 = dict(device=dev, dtype=torch.float64), dict(device=dev, dtype=torch.int32)
    buf = dict(
        norm=torch.empty(B, 6, **f64), xn=torch.empty(max(total, 1), 4, **f64), sample=torch.empty(B, FUND_ROUND, 7, **i32),
        nmod=torch.empty(B, FUND_ROUND, **i32), F=torch.empty(B, FUND_ROUND, FUND_MODELS, 9, **f64),
        counts=torch.empty(B, S, FUND_ROUND * FUND_MODELS, **i32), losses=torch.empty(B, S, FUND_ROUND * FUND_MODELS, **f64),
        state=torch.zeros(B, FUND_STATE, **i32), best_F=torch.zeros(B, 9, **f64), best_loss=torch.zeros(B, **f64),
        running=torch.zeros(1, **i32), out_F=torch.empty(B, 9, **f64), ok=torch.empty(B, device=dev, dtype=torch.uint8),
        mask=torch.empty(max(total, 1), device=dev, dtype=torch.uint8))
    kw = dict(batch=B, x0=x0, x1=x1, offsets=offsets, max_n=int(max_n), thresh=float(thr), conf=float(conf), max_iters=int(max_iters),
              seed=int(seed) & (2 ** 64 - 1), round=0, table=_magsac_tables_on(dev), **buf)
    _ransac_rounds("fund", "rb_fund_args", kw, FUND_ROUND)
    cabi.call("romab200_fund_refine", "rb_fund_args", **kw)
    return buf


def find_fundamental_batched(points1_list, points2_list, method=USAC_MAGSAC, ransacReprojThreshold=3, confidence=0.99, maxIters=1000,
                             *, seed=0):
    """`find_fundamental` for B pairs in one launch set.  points*_list: B arrays / tensors [N_b, 2] or [N_b, 1, 2] (ragged N).
    Every pair draws from the stream keyed by `seed` alone and nothing of pair b depends on the other pairs, so pair b is
    bit-identical to `find_fundamental` of that pair alone.  Returns (F [B, 3, 3] float64, ok [B] bool, masks: list of uint8
    [N_b, 1]); numpy inputs give numpy outputs, tensors give device tensors.  ok[b] is False, F[b] zero and the mask all zero
    where `find_fundamental` returns None, and for pairs of fewer than 7 points."""
    thr, conf, max_iters = _fund_args(method, ransacReprojThreshold, confidence, maxIters)
    x0, x1, offsets, ns = _pack_pairs(points1_list, points2_list, _fund_points, "find_fundamental", ("points1_list", "points2_list"),
                                      ("points1", "points2"))
    buf = _fund_launch(x0, x1, offsets, max(ns), thr, conf, max_iters, seed)
    masks = [m.view(-1, 1) for m in buf["mask"][:sum(ns)].split(ns)]
    return _outputs(not isinstance(points1_list[0], torch.Tensor), buf["out_F"].view(len(ns), 3, 3), buf["ok"].bool(), masks)


def find_fundamental(points1, points2, method=USAC_MAGSAC, ransacReprojThreshold=3, confidence=0.99, maxIters=1000, mask=None, *, seed=0):
    """Drop-in for `cv2.findFundamentalMat` with method USAC_MAGSAC: the same keywords and return form.  points2^T F points1 = 0.
    MAGSAC++ over seven-point samples (csrc/fundamental.cu, DESIGN.md): the best model by the sigma-marginalised loss with
    sigma_max = ransacReprojThreshold, at most maxIters hypotheses (fewer as `confidence` allows, from the inlier ratio at
    the threshold), then sigma-consensus++.  Returns (F float64 [3, 3], mask uint8 [N, 1]): F has unit Frobenius norm and its
    largest-magnitude entry positive (cv2 fixes neither, so compare up to scale and sign); the mask holds the points whose Sampson
    distance to F is below ransacReprojThreshold.  `mask` is accepted and ignored, as in cv2's Python binding.  numpy in gives
    numpy out (float32 points are accepted); tensors give device tensors.
    Rows with a NaN or infinite coordinate are never inliers and do not enter the normalisation; a sample that draws one gives no
    model.  When no sample gives a model (all points identical, all on one line in both images, ...) the result is (None, all-zero
    mask).  Raises ValueError for fewer than 7 points and NotImplementedError for every other cv2 method."""
    del mask
    thr, conf, max_iters = _fund_args(method, ransacReprojThreshold, confidence, maxIters)
    n = len(points1)
    if n < 7 or len(points2) != n:
        raise ValueError(f"find_fundamental needs the same number (>= 7) of points in both images, got {n} and {len(points2)}")
    F, ok, masks = find_fundamental_batched([points1], [points2], USAC_MAGSAC, thr, conf, max_iters, seed=seed)
    if not bool(ok[0]):
        return None, masks[0]
    return F[0], masks[0]


# ---- absolute pose -------------------------------------------------------------------------------------------------------
# include/romab200.h: RB_ABS_ROUND, RB_ABS_MAX_SOL, RB_ABS_STATE, RB_ABS_MAX_BATCH
ABS_ROUND, ABS_MAX_SOL, ABS_STATE, ABS_MAX_BATCH = cabi.RB_ABS_ROUND, cabi.RB_ABS_MAX_SOL, cabi.RB_ABS_STATE, cabi.RB_ABS_MAX_BATCH


def _abs_points(p, dev, width, name):
    """[n, width] real points of any float dtype -> float64 [n, width] on `dev`."""
    t = p if isinstance(p, torch.Tensor) else torch.as_tensor(np.asarray(p))
    if t.dim() != 2 or t.shape[1] != width:
        raise ValueError(f"{name} must be [n, {width}], got {tuple(t.shape)}")
    if not t.dtype.is_floating_point:
        raise TypeError(f"{name} must have a float dtype, got {t.dtype}")
    return t.to(dev, torch.float64).contiguous()


def _abs_args(max_error, confidence, max_iters, seed):
    """Checks the estimator's scalar arguments; returns (max_error^2, confidence, max_iters, seed)."""
    max_error, confidence = float(max_error), float(confidence)
    if not (math.isfinite(max_error) and max_error > 0):
        raise ValueError(f"max_error must be finite and > 0, got {max_error!r}")
    if not 0 < confidence < 1:
        raise ValueError(f"confidence must lie in (0, 1), got {confidence!r}")
    if isinstance(max_iters, bool) or not 1 <= int(max_iters) < 1 << 31 or int(max_iters) != max_iters:
        raise ValueError(f"max_iters must be an int in [1, 2^31), got {max_iters!r}")
    if isinstance(seed, bool) or int(seed) != seed or not 0 <= int(seed) < 1 << 64:
        raise ValueError(f"seed must be an int in [0, 2^64), got {seed!r}")
    return max_error * max_error, confidence, int(max_iters), int(seed)


def _abs_launch(x, X, offsets, K, max_n, max_error2, conf, max_iters, seed):
    """Enqueues the whole absolute-pose estimate on the current stream.  x: float64 [total, 2], X: float64 [total, 3] device tensors
    (total >= 1), offsets: int64 [B + 1], K: float64 [B, 3, 3].  With max_iters <= ABS_ROUND this is one round and reads nothing
    back; each further round costs one 4-byte read of the `running` flag.  Returns the buffers (R, t, ok, num_inliers, mask, ...);
    their bytes are include/romab200.h's per-chunk formula of image registration, less the gathered points and image list."""
    dev = x.device
    B = offsets.numel() - 1
    total = x.shape[0]
    S = cabi.abspose_splits(max_n)
    f64, i32 = dict(device=dev, dtype=torch.float64), dict(device=dev, dtype=torch.int32)
    buf = dict(sample=torch.empty(B, ABS_ROUND, 3, **i32), models=torch.empty(B, ABS_ROUND, ABS_MAX_SOL, 12, **f64),
               nsol=torch.empty(B, ABS_ROUND, **i32), counts=torch.empty(B, S, ABS_MAX_SOL, ABS_ROUND, **i32),
               state=torch.zeros(B, ABS_STATE, **i32), best=torch.zeros(B, 12, **f64), running=torch.zeros(1, **i32),
               R=torch.empty(B, 3, 3, **f64), t=torch.empty(B, 3, **f64), ok=torch.empty(B, device=dev, dtype=torch.uint8),
               num_inliers=torch.empty(B, device=dev, dtype=torch.int64), mask=torch.empty(total, device=dev, dtype=torch.uint8))
    kw = dict(batch=B, x=x, X=X, offsets=offsets, K=K, max_n=int(max_n), max_error2=float(max_error2), conf=float(conf),
              max_iters=int(max_iters), seed=int(seed) & (2 ** 64 - 1), round=0, **buf)
    _ransac_rounds("abspose", "rb_abspose_args", kw, ABS_ROUND)
    cabi.call("romab200_abspose_refine", "rb_abspose_args", **kw)
    return buf


def estimate_absolute_pose_batched(points2D_list, points3D_list, K, *, max_error=12.0, confidence=0.9999, max_iters=10000, seed=0):
    """Absolute pose of B cameras x ~ K (R X + t) from ragged sets of pixels points2D_list[b] [n_b, 2] and world points
    points3D_list[b] [n_b, 3] of any float dtype (widened to float64); K is one [3, 3] for every item or [B, 3, 3].  COLMAP's
    EstimateAbsolutePose + RefineAbsolutePose on the device (csrc/absolute_pose.cu, the rules in include/romab200.h): Lambda Twist
    P3P on Philox-drawn samples, the model with the most points within `max_error` px and in front of the camera (OpenCV's RANSAC
    loop and stopping rule at `confidence`, at most `max_iters` hypotheses), then Gauss-Newton on its inliers and the inliers
    recomputed once.  Every item draws the stream keyed by `seed` alone, so item b is bit-identical to a call on that item alone.
    Returns (R [B, 3, 3] float64, t [B, 3] float64, ok [B] bool, num_inliers [B] int64, masks: list of bool [n_b]); numpy inputs give
    numpy outputs, tensors give device tensors.  ok[b] is False, and R, t, the mask zero, where no model was found or n_b < 3.
    Host reads: the `running` flag once per round of RB_ABS_ROUND hypotheses before the last."""
    max_error2, conf, max_iters, seed = _abs_args(max_error, confidence, max_iters, seed)
    if len(points2D_list) != len(points3D_list) or len(points2D_list) == 0:
        raise ValueError("points2D_list and points3D_list must be non-empty and of the same length")
    if len(points2D_list) > ABS_MAX_BATCH:
        raise ValueError(f"at most {ABS_MAX_BATCH} items per call, got {len(points2D_list)}")
    dev = _device("estimate_absolute_pose")
    xs = [_abs_points(p, dev, 2, "points2D") for p in points2D_list]
    Xs = [_abs_points(p, dev, 3, "points3D") for p in points3D_list]
    for a, b in zip(xs, Xs):
        if a.shape[0] != b.shape[0]:
            raise ValueError(f"points2D and points3D differ in length: {a.shape[0]} vs {b.shape[0]}")
    ns = [a.shape[0] for a in xs]
    B = len(ns)
    offsets = torch.tensor(np.concatenate([[0], np.cumsum(ns)]), dtype=torch.int64, device=dev)
    if not sum(ns):
        xs, Xs = [torch.zeros(1, 2, dtype=torch.float64, device=dev)], [torch.zeros(1, 3, dtype=torch.float64, device=dev)]
    Kt = _intrinsics(K, B, dev).contiguous()
    buf = _abs_launch(torch.cat(xs), torch.cat(Xs), offsets, Kt, max(ns), max_error2, conf, max_iters, seed)
    masks = list(buf["mask"][:sum(ns)].bool().split(ns))
    return _outputs(not isinstance(points2D_list[0], torch.Tensor), buf["R"], buf["t"], buf["ok"].bool(), buf["num_inliers"], masks)


def estimate_absolute_pose(points2D, points3D, K, *, max_error=12.0, confidence=0.9999, max_iters=10000, seed=0):
    """`estimate_absolute_pose_batched` for one camera: None when no model is found (or fewer than 3 points), otherwise
    (R float64 [3, 3], t float64 [3], mask bool [n]) with x ~ K (R X + t).  numpy in gives numpy out; tensors give device tensors."""
    R, t, ok, _, masks = estimate_absolute_pose_batched([points2D], [points3D], K, max_error=max_error, confidence=confidence,
                                                        max_iters=max_iters, seed=seed)
    if not bool(ok[0]):
        return None
    return R[0], t[0], masks[0]
