"""Bundle adjustment of cameras and track points on the device (`bundle_adjust`): Levenberg-Marquardt over the poses of the free
cameras and the points of the ok tracks, minimising the (optionally Cauchy-robust) reprojection error of the inlier observations
that `triangulate_tracks` marked.  The normal equations are reduced to the cameras by the Schur complement and factored by dense
Cholesky on the device; the host only drives the loop.  The exact rules are in include/romab200.h and INTEGRATION.md;
`oracle/bundle.py` restates them in numpy."""
from __future__ import annotations

import math
import operator
from dataclasses import dataclass

import numpy as np
import torch

from . import cabi
from . import triangulate as _tri
from .match_graph import WORKSPACE_BYTES, MatchGraph
from .tracks import Tracks
from .triangulate import Points3D

LAMBDA0, NU0, MIN_RELATIVE_DECREASE, MAX_LAMBDA = 1e-4, 2.0, 1e-3, 1e32


@dataclass
class BundleResult:
    """R float64 [N, 3, 3] and t [N, 3] on the graph's device; points: X refined for ok tracks, ok, num_inliers and inlier as given,
    error recomputed at the final X, R, t (the given points unchanged when no step was kept).  cost: host float64 [n + 1], the
    cost before the first trial and after each (a rejected trial repeats it); accepted: host bool [n]; pred: host float64 [n], each
    trial's predicted decrease 1/2 d^T (lambda D d - g); termination:
    "function_tolerance", "max_iterations", "no_progress" or "nothing_to_adjust"."""
    R: torch.Tensor
    t: torch.Tensor
    points: Points3D
    cost: np.ndarray
    accepted: np.ndarray
    pred: np.ndarray
    termination: str


def workspace_bytes(num_images: int, num_free: int, num_tracks: int, num_elements: int) -> int:
    """Device bytes of one call (include/romab200.h): every buffer `_buffers` allocates."""
    tiles = -(-num_elements // cabi.RB_TRACKS_TILE)
    return (cabi.RB_BA_ELEMENT_BYTES * num_elements + cabi.RB_BA_TRACK_BYTES * num_tracks + cabi.RB_BA_IMAGE_BYTES * num_images
            + cabi.RB_BA_FREE_BYTES * num_free + 288 * num_free * num_free + 1024 * tiles + cabi.RB_BA_ONCE_BYTES)


def _buffers(dev, N, F, T, E) -> dict:
    """The call's device buffers, named by their rb_ba_args fields (uninitialised; the kernels write them before reading)."""
    f64, i32, i64, u8 = torch.float64, torch.int32, torch.int64, torch.uint8
    tiles = -(-E // cabi.RB_TRACKS_TILE)
    shapes = dict(kp_offsets=(N + 1, i64), track_offsets=(T + 1, i64), track_ok=(T, u8), inlier=(E, u8),
                  free_index=(N, i32), free_cams=(F, i32), fixed_tx=(F, u8), info=(2, i64), elem_track=(E, i32), keys=(E, i64),
                  keys_alt=(E, i64), hist=(256 * tiles + 1, i32), obs_offsets=(N + 1, i64), obs=(E, i32), cams=(N * cabi.RB_BA_CAM, f64),
                  X=(3 * T, f64), cams_trial=(N * cabi.RB_BA_CAM, f64), X_trial=(3 * T, f64), W=(18 * E, f64),
                  track_sys=(T * cabi.RB_BA_TRACK, f64), cam_sys=(12 * F, f64), S=(36 * F * F, f64), rhs=(6 * F, f64), cam_pred=(N, f64),
                  track_part=(3 * T, f64), result=(cabi.RB_BA_RESULT, f64), error=(T, f64))
    return {k: torch.empty(n, dtype=d, device=dev) for k, (n, d) in shapes.items()}


def _indices(name, v, N):
    try:
        out = [operator.index(i) for i in v]
    except TypeError:
        raise ValueError(f"bundle_adjust: {name} must be a sequence of ints, got {v!r}") from None
    if any(isinstance(i, bool) for i in v) or not all(0 <= i < N for i in out):
        raise ValueError(f"bundle_adjust: {name} must hold camera indices in [0, {N}), got {v!r}")
    return sorted(set(out))


def _check(graph, tracks, points, K, R, t, fixed_poses, fixed_tx, loss_scale, max_iterations, function_tolerance, workspace_bytes_):
    """Argument rules, checked before any device work.  Returns (kp_offsets, track_offsets, K, R, t as float64 arrays, fixed
    poses, fixed_tx, c^2, max_iterations, function_tolerance)."""
    kp_off, tr_off, *_ = _tri._check(graph, tracks, K, R, t, 1.0, 0.0, 1, 0, what="bundle_adjust", device=False)
    N, T, E = len(kp_off) - 1, len(tr_off) - 1, tr_off[-1]
    K, R, t = (_tri._float64(n, v, s, "bundle_adjust") for n, v, s in (("K", K, (N, 3, 3)), ("R", R, (N, 3, 3)), ("t", t, (N, 3))))
    if not isinstance(points, Points3D):
        raise ValueError(f"bundle_adjust: points must be Points3D, got {type(points).__name__}")
    for name, v, dt, shape in (("points.X", points.X, torch.float64, (T, 3)), ("points.ok", points.ok, torch.bool, (T,)),
                               ("points.inlier", points.inlier, torch.bool, (E,))):
        if not isinstance(v, torch.Tensor) or v.dtype != dt or tuple(v.shape) != shape:
            raise ValueError(f"bundle_adjust: {name} must be {dt} {list(shape)}, got {getattr(v, 'dtype', type(v).__name__)} "
                             f"{tuple(getattr(v, 'shape', ()))}")
    fixed_poses = _indices("fixed_poses", fixed_poses, N)
    if N == 1 and isinstance(fixed_tx, (tuple, list)) and tuple(fixed_tx) == (1,):
        fixed_tx = ()                                     # the default names the second camera
    fixed_tx = _indices("fixed_tx", fixed_tx, N)
    if loss_scale is not None:
        if isinstance(loss_scale, bool) or not isinstance(loss_scale, (int, float)) or not (math.isfinite(loss_scale) and loss_scale > 0):
            raise ValueError(f"bundle_adjust: loss_scale must be None or finite and > 0, got {loss_scale!r}")
    if isinstance(max_iterations, bool) or not isinstance(max_iterations, int) or max_iterations < 0:
        raise ValueError(f"bundle_adjust: max_iterations must be an int >= 0, got {max_iterations!r}")
    if isinstance(function_tolerance, bool) or not isinstance(function_tolerance, (int, float)) or not (function_tolerance >= 0):
        raise ValueError(f"bundle_adjust: function_tolerance must be a number >= 0, got {function_tolerance!r}")
    if isinstance(workspace_bytes_, bool) or not isinstance(workspace_bytes_, int):
        raise ValueError(f"bundle_adjust: workspace_bytes must be an int, got {workspace_bytes_!r}")
    need = workspace_bytes(N, N - len(fixed_poses), T, E)
    if need > workspace_bytes_:
        raise ValueError(f"bundle_adjust: the call needs {need} bytes of device memory ({N - len(fixed_poses)} free cameras, {T} tracks, "
                         f"{E} elements), more than workspace_bytes = {workspace_bytes_}")
    _tri._check_device([graph.kp_offsets, graph.keypoints, tracks.track_offsets, tracks.elements, points.X, points.ok, points.inlier],
                       "bundle_adjust")
    if not bool(torch.isfinite(points.X).all()):
        raise ValueError("bundle_adjust: points.X has values that are not finite")
    c2 = 0.0 if loss_scale is None else float(loss_scale) ** 2
    return kp_off, tr_off, K, R, t, fixed_poses, fixed_tx, c2, max_iterations, float(function_tolerance)


def bundle_adjust(graph: MatchGraph, tracks: Tracks, points: Points3D, K, R, t, *, fixed_poses=(0,), fixed_tx=(1,), loss_scale=None,
                  max_iterations=50, function_tolerance=1e-6, workspace_bytes=WORKSPACE_BYTES) -> BundleResult:
    """Refines the cameras x ~ K[i] (R[i] X + t[i]) (the convention of `triangulate_tracks`; K stays fixed) and the points of the ok
    tracks of `points` (from `triangulate_tracks` on the same graph and tracks) to minimise 1/2 sum rho(|r_e|^2) over the inlier
    observations: rho(s) = s, or the Cauchy c^2 log(1 + s / c^2) with c = `loss_scale` px.  K, R [N, 3, 3] and t [N, 3] are tensors or
    arrays of any float dtype, widened to float64 on the host.

    Gauge: the cameras in `fixed_poses` keep their pose, and those in `fixed_tx` keep their x-translation (COLMAP's default: the
    first pose and the second camera's t_x; with one camera, the default fixed_tx is dropped).  Levenberg-Marquardt from
    lambda = 1e-4, every trial counting against `max_iterations`; the run stops after a kept step that lowered the cost by at most
    `function_tolerance` times the cost, or when lambda exceeds 1e32.  A track whose inlier observations repeat an image (tracks
    built with drop_conflicts=False) raises ValueError, as does an element id outside its image's keypoints.

    Bit-identical from run to run.  Arguments are checked before any device work; `workspace_bytes` bounds the device memory of
    the call (`workspace_bytes()` gives it).  Host reads: the offsets, a finiteness flag of X, the setup status and cost, and four
    numbers per trial."""
    kp_off, tr_off, K, R, t, fixed, ftx, c2, max_iterations, ftol = _check(graph, tracks, points, K, R, t, fixed_poses, fixed_tx,
                                                                           loss_scale, max_iterations, function_tolerance, workspace_bytes)
    N, T, E = len(kp_off) - 1, len(tr_off) - 1, tr_off[-1]
    dev = graph.kp_offsets.device
    with torch.cuda.device(dev):
        R0, t0 = torch.from_numpy(R).to(dev), torch.from_numpy(t).to(dev)
        inputs = BundleResult(R0, t0, points, np.zeros(1), np.zeros(0, bool), np.zeros(0), "nothing_to_adjust")
        if T == 0 or E == 0:
            return inputs
        free_cams = [i for i in range(N) if i not in set(fixed)]
        F = len(free_cams)
        b = _buffers(dev, N, F, T, E)
        free_index = np.full(N, -1, np.int32)
        free_index[free_cams] = np.arange(F, dtype=np.int32)
        cams = np.concatenate((R.reshape(N, 9), t, K.reshape(N, 9)), 1)
        # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
        for name, v in (("kp_offsets", np.asarray(kp_off, np.int64)), ("track_offsets", np.asarray(tr_off, np.int64)),
                        ("free_index", free_index), ("free_cams", np.asarray(free_cams, np.int32)),
                        ("fixed_tx", np.asarray([i in set(ftx) for i in free_cams], np.uint8)), ("cams", cams.reshape(-1))):
            b[name].copy_(torch.from_numpy(v))
        b["track_ok"].copy_(points.ok)
        b["inlier"].copy_(points.inlier)
        b["X"].copy_(points.X.reshape(-1))
        if F == 0:
            for name in ("free_cams", "fixed_tx", "cam_sys", "S", "rhs"):
                b[name] = None
        args = dict(num_tracks=T, num_images=N, num_free=F, elements=tracks.elements.contiguous(), num_elements=E,
                    keypoints=graph.keypoints.contiguous(), num_rows=kp_off[-1], loss_scale2=c2, **b)

        def call(fn, lam):
            cabi.call(f"romab200_ba_{fn}", "rb_ba_args", **args, **{"lambda": lam})

        lam, nu = LAMBDA0, NU0
        call("setup", lam)
        # the status is read before any kernel that indexes with the element ids
        status, used = b["info"].tolist()
        if status & cabi.RB_BA_BAD_ID:
            raise ValueError("bundle_adjust: a track element lies outside its image's keypoints")
        if status & cabi.RB_BA_REPEATED:
            raise ValueError("bundle_adjust: a track's inlier observations repeat an image (tracks built with drop_conflicts=False)")
        if used == 0:
            return inputs
        call("linearize", lam)
        call("cost", lam)
        F_cur = float(b["result"][0].item())
        cost, accepted, preds, termination, fresh = [F_cur], [], [], "max_iterations", True
        for _ in range(max_iterations):
            if not fresh:
                call("linearize", lam)
            fresh = False
            if F > 0:
                call("cameras", lam)
                call("cholesky", lam)
            call("step", lam)
            F_new, pred, bad_depth, pivot = b["result"].tolist()
            with np.errstate(divide="ignore", invalid="ignore"):
                rho = float(np.float64(F_cur - F_new) / np.float64(pred))
            keep = pivot == 0 and math.isfinite(F_new) and bad_depth == 0 and rho > MIN_RELATIVE_DECREASE
            accepted.append(keep)
            preds.append(pred)
            if keep:
                args["cams"], args["cams_trial"] = args["cams_trial"], args["cams"]
                args["X"], args["X_trial"] = args["X_trial"], args["X"]
                decrease, F_cur = F_cur - F_new, F_new
                cost.append(F_cur)
                lam *= max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3)
                nu = NU0
                if decrease <= ftol * (F_cur + decrease):
                    termination = "function_tolerance"
                    break
            else:
                cost.append(F_cur)
                lam *= nu
                nu *= 2.0
                if lam > MAX_LAMBDA:
                    termination = "no_progress"
                    break
        cost, accepted, preds = np.asarray(cost, np.float64), np.asarray(accepted, bool), np.asarray(preds, np.float64)
        if not accepted.any():
            return BundleResult(R0, t0, points, cost, accepted, preds, termination)
        call("error", lam)
        cams_d = args["cams"].view(N, cabi.RB_BA_CAM)
        out = Points3D(args["X"].view(T, 3).clone(), points.ok, points.num_inliers, args["error"].clone(), points.inlier)
        return BundleResult(cams_d[:, :9].reshape(N, 3, 3).clone(), cams_d[:, 9:12].clone(), out, cost, accepted, preds, termination)
