"""Reconstruction without known cameras on the device: the two-view initialisation of COLMAP's incremental mapper
(`initialize_reconstruction`: FindInitialImagePair + EstimateInitialTwoViewGeometry), the register -> triangulate -> adjust loop
that grows it to every image it can (`reconstruct`), and COLMAP's text model of the result (`write_colmap_text`).  The
initialisation's statistics run in `csrc/twoview.cu`; the loop only calls the existing device stages.  The exact rules are in
include/romab200.h and INTEGRATION.md; `oracle/mapper.py` restates them in numpy."""
from __future__ import annotations

import math
import operator
import os
from dataclasses import dataclass

import numpy as np
import torch

from . import cabi, geometry
from . import triangulate as _tri
from . import verify as _verify
from .bundle import bundle_adjust
from .match_graph import WORKSPACE_BYTES, MatchGraph
from .register import register_images
from .tracks import Tracks
from .triangulate import Points3D, triangulate_tracks

MAX_CANDIDATES = 4096           # the relative-pose estimator's batch limit (romab200_pose_recover)


@dataclass
class TwoViewInit:
    """Per candidate c, in rank order, on the graph's device: pair_index[c] int64 (the row of `pairs`), images[c] int64 [2] (i, j as
    that row gives them), R[c] float64 [3, 3] and t[c] [3] (unit length; x_j ~ K_j (R x + t) for a point x of camera i's frame), ok[c]
    bool (a pose was found), num_inliers[c] int64 (matches that passed RANSAC and the chirality test), num_good[c] int64,
    median_angle[c] float64 degrees, forward[c] = |t_z| and accepted[c] bool.  mask bool [total] holds every candidate's per-match
    mask, candidate c at offsets[c]:offsets[c + 1] (int64 [C + 1]).  chosen is the host int index of the first accepted candidate, or
    -1."""
    pair_index: torch.Tensor
    images: torch.Tensor
    R: torch.Tensor
    t: torch.Tensor
    ok: torch.Tensor
    num_inliers: torch.Tensor
    num_good: torch.Tensor
    median_angle: torch.Tensor
    forward: torch.Tensor
    accepted: torch.Tensor
    mask: torch.Tensor
    offsets: torch.Tensor
    chosen: int


@dataclass
class Reconstruction:
    """registered bool [N]; R float64 [N, 3, 3] and t [N, 3] (x ~ K (R X + t); zero where an image is not registered); points: the
    final Points3D (triangulated with the registered cameras); init: the TwoViewInit; rounds: one host dict per round (registered:
    the images registered when it started, ba_termination, ba_cost: the cost before and after its bundle adjustment, ok_tracks after
    its re-triangulation, added: the images registration added); termination: "all_registered", "no_image_added" or
    "no_initial_pair"."""
    registered: torch.Tensor
    R: torch.Tensor
    t: torch.Tensor
    points: Points3D
    init: TwoViewInit
    rounds: list
    termination: str


def rank_candidates(match_offsets, min_num_inliers, num_candidates) -> list:
    """The candidate pairs: every k with n_k = match_offsets[k + 1] - match_offsets[k] >= min_num_inliers, by n_k descending, then
    k ascending, the first num_candidates of them."""
    ns = np.diff(np.asarray(match_offsets, np.int64))
    ks = np.flatnonzero(ns >= min_num_inliers)
    order = np.lexsort((ks, -ns[ks]))
    return ks[order][:num_candidates].tolist()


def _int(what, name, v, lo, hi=None):
    ok = not isinstance(v, (bool, np.bool_))
    try:
        v = operator.index(v)
    except TypeError:
        ok = False
    if not ok or v < lo or (hi is not None and v > hi):
        raise ValueError(f"{what}: {name} must be an int in [{lo}, {'inf' if hi is None else hi}], got {v!r}")
    return v


def _float(what, name, v, lo, strict):
    try:
        f = float(v)
    except (TypeError, ValueError):
        f = math.nan
    if isinstance(v, bool) or not math.isfinite(f) or f < lo or (strict and f == lo):
        raise ValueError(f"{what}: {name} must be a finite number {'>' if strict else '>='} {lo}, got {v!r}")
    return f


def _check_init(pairs, graph, K, init_pair, num_candidates, min_num_inliers, max_error, min_tri_angle, max_forward_motion,
                confidence, max_iters, seed, what="initialize_reconstruction"):
    """Argument rules, checked before any device work.  Returns (pairs [P, 2] int64 CPU, K float64 [N, 3, 3], the ranked candidate
    pair indices, norm_thresh, and the checked scalars)."""
    num_candidates = _int(what, "num_candidates", num_candidates, 1, MAX_CANDIDATES)
    min_num_inliers = _int(what, "min_num_inliers", min_num_inliers, 0)
    max_error = _float(what, "max_error", max_error, 0.0, True)
    min_tri_angle = _float(what, "min_tri_angle", min_tri_angle, 0.0, False)
    if min_tri_angle >= 180:
        raise ValueError(f"{what}: min_tri_angle must lie in [0, 180) degrees, got {min_tri_angle!r}")
    max_forward_motion = _float(what, "max_forward_motion", max_forward_motion, 0.0, False)
    max_iters = _int(what, "max_iters", max_iters, 1, (1 << 31) - 1)
    seed = _int(what, "seed", seed, 0, (1 << 64) - 1)
    try:
        pairs, _, confidence, *_ = _verify._check(pairs, graph, max_error, confidence, max_iters, 0, seed, 1)
    except ValueError as e:
        raise ValueError(f"{what}: {str(e).split(': ', 1)[-1]}") from None
    N = len(graph._kp_off) - 1
    K = _tri._float64("K", K, (N, 3, 3), what)
    fbar = float(np.mean((K[:, 0, 0] + K[:, 1, 1]) / 2))
    if not fbar > 0:
        raise ValueError(f"{what}: the mean focal length of K must be > 0, got {fbar!r}")
    if init_pair is None:
        cand = rank_candidates(graph._m_off, min_num_inliers, num_candidates)
    else:
        try:
            i, j = init_pair
            i, j = operator.index(i), operator.index(j)
        except (TypeError, ValueError):
            raise ValueError(f"{what}: init_pair must be a pair of ints (i, j), got {init_pair!r}") from None
        p = pairs.numpy()
        rows = np.flatnonzero(((p[:, 0] == i) & (p[:, 1] == j)) | ((p[:, 0] == j) & (p[:, 1] == i)))
        if rows.size == 0:
            raise ValueError(f"{what}: init_pair {(i, j)} is not a row of pairs, in either order")
        cand = [int(rows[0])]
    return pairs, K, cand, max_error / fbar, dict(min_num_inliers=min_num_inliers, max_error=max_error, min_tri_angle=min_tri_angle,
                                                  max_forward_motion=max_forward_motion, confidence=confidence, max_iters=max_iters,
                                                  seed=seed)


def _gather(pairs, graph, cand):
    """The candidates' matched keypoints packed in rank order on the device (romab200_verify_gather with a pair_list): x0, x1
    float64 [max(total, 1), 2] and offsets int64 [C + 1].  Raises ValueError for a match id outside its image's keypoints."""
    kp_off, m_off = graph._kp_off, graph._m_off
    N, P, M, C = len(kp_off) - 1, len(m_off) - 1, m_off[-1], len(cand)
    dev = graph.kp_offsets.device
    total = sum(m_off[k + 1] - m_off[k] for k in cand)
    x0 = torch.zeros(max(total, 1), 2, dtype=torch.float64, device=dev)
    x1 = torch.zeros_like(x0)
    off = torch.zeros(C + 1, dtype=torch.int64, device=dev)
    if M == 0:
        return x0, x1, off, total
    # the offsets the host checked, not the tensors' current contents: the device indexes with exactly what was validated
    kw = dict(pairs=pairs.to(dev, non_blocking=True), num_pairs=P, num_images=N,
              kp_offsets=torch.tensor(kp_off, dtype=torch.int64).to(dev, non_blocking=True), keypoints=graph.keypoints.contiguous(),
              num_rows=kp_off[-1], match_offsets=torch.tensor(m_off, dtype=torch.int64).to(dev, non_blocking=True),
              matches=graph.matches.contiguous(), match_scores=graph.match_scores.contiguous(), num_matches=M,
              info=torch.empty(2, dtype=torch.int64, device=dev))
    cabi.call("romab200_verify_check", "rb_verify_args", **kw)
    if int(kw["info"][0].item()) & cabi.RB_VERIFY_BAD_ID:
        raise ValueError("initialize_reconstruction: a match id lies outside its image's keypoints")
    cabi.call("romab200_verify_gather", "rb_verify_args", pair_begin=0, pair_end=C, x0=x0, x1=x1, chunk_offsets=off,
              pair_list=torch.tensor(cand, dtype=torch.int32).to(dev), **kw)
    return x0, x1, off, total


def _score(x0, x1, off, Kc, buf, max_error):
    """romab200_twoview_score on the pose estimate `buf` (geometry._launch's buffers): (num_good, median_angle, forward)."""
    C, dev = off.numel() - 1, off.device
    out = dict(num_good=torch.empty(C, dtype=torch.int64, device=dev), median_angle=torch.empty(C, dtype=torch.float64, device=dev),
               forward=torch.empty(C, dtype=torch.float64, device=dev))
    cabi.call("romab200_twoview_score", "rb_twoview_args", batch=C, offsets=off, x0=x0, x1=x1, xn=buf["xn"], mask=buf["mask"], K=Kc,
              R=buf["R"], t=buf["t"], ok=buf["ok"], max_error2=max_error * max_error,
              angle=torch.empty(buf["mask"].numel(), dtype=torch.float64, device=dev), **out)
    return out["num_good"], out["median_angle"], out["forward"]


def initialize_reconstruction(pairs, graph: MatchGraph, K, *, init_pair=None, num_candidates=256, min_num_inliers=100, max_error=4.0,
                              min_tri_angle=16.0, max_forward_motion=0.95, confidence=0.999, max_iters=10000, seed=0) -> TwoViewInit:
    """The initial pair of a reconstruction and its relative pose, COLMAP's FindInitialImagePair + EstimateInitialTwoViewGeometry.
    `graph` is a verified MatchGraph (`verify_matches`) built from `pairs`; K [N, 3, 3] is a tensor or array of any float dtype.  The
    defaults are COLMAP's init_* mapper options.

    Candidates are the pairs with at least `min_num_inliers` matches, by match count descending, then pair index ascending, the first
    `num_candidates` (at most 4 096).  All of them are one batch of the relative-pose estimator: candidate c's R, t and mask are
    byte-identical to `estimate_pose_batched` over the ranked lists of keypoints, with K_i, K_j per candidate, norm_thresh =
    max_error / f (f the mean of (fx + fy) / 2 over all images), `confidence`, `max_iters` and `seed`.  romab200_twoview_score then
    triangulates every mask inlier and counts the good points (in front of both cameras, within `max_error` px in both images) and
    the median of their triangulation angles.  A candidate is accepted when a pose was found, num_good >= min_num_inliers,
    median_angle >= min_tri_angle degrees and |t_z| <= max_forward_motion; the first accepted one is chosen.  With `init_pair` =
    (i, j), a row of `pairs` in either order, that pair alone is candidate 0 (in its row's orientation) and is chosen only if
    accepted.

    Arguments are checked before any device work (ValueError).  Bit-identical from run to run.  Host reads: the status word of the
    id check, the estimator's `running` flag once per round of 1 024 hypotheses before the last, and the accepted flags."""
    pairs, K, cand, norm_thresh, o = _check_init(pairs, graph, K, init_pair, num_candidates, min_num_inliers, max_error, min_tri_angle,
                                                 max_forward_motion, confidence, max_iters, seed)
    C, dev = len(cand), graph.kp_offsets.device
    with torch.cuda.device(dev):
        pair_index = torch.tensor(cand, dtype=torch.int64)
        images = pairs[pair_index].to(dev)
        if C == 0:
            z = torch.zeros(0, dtype=torch.float64, device=dev)
            zi = torch.zeros(0, dtype=torch.int64, device=dev)
            zb = torch.zeros(0, dtype=torch.bool, device=dev)
            return TwoViewInit(zi, images, z.view(0, 3, 3), z.view(0, 3), zb, zi, zi, z, z, zb, zb,
                               torch.zeros(1, dtype=torch.int64, device=dev), -1)
        x0, x1, off, total = _gather(pairs, graph, cand)
        Kc = torch.from_numpy(np.stack((K[images[:, 0].cpu().numpy()], K[images[:, 1].cpu().numpy()]), 1)).to(dev).contiguous()
        ns = [graph._m_off[k + 1] - graph._m_off[k] for k in cand]
        buf = geometry._launch(x0, x1, off, Kc, max(ns), norm_thresh, o["confidence"], o["max_iters"], o["seed"])
        num_good, median_angle, forward = _score(x0, x1, off, Kc, buf, o["max_error"])
        mask = buf["mask"][:total].bool()
        csum = torch.cat((torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(mask.long(), 0)))
        num_inliers = csum[off[1:]] - csum[off[:-1]]
        ok = buf["ok"].bool()
        accepted = (ok & (num_good >= o["min_num_inliers"]) & (median_angle >= o["min_tri_angle"])
                    & (forward <= o["max_forward_motion"]))
        hits = np.flatnonzero(accepted.cpu().numpy())
    return TwoViewInit(pair_index.to(dev), images, buf["R"], buf["t"], ok, num_inliers, num_good, median_angle, forward, accepted, mask,
                       off, int(hits[0]) if hits.size else -1)


def reconstruct(pairs, graph: MatchGraph, tracks: Tracks, K, *, init_pair=None, init_num_candidates=256, init_min_num_inliers=100,
                init_max_error=4.0, init_min_tri_angle=16.0, init_max_forward_motion=0.95, tri_max_error=4.0, tri_min_angle=1.5,
                abs_max_error=12.0, abs_min_inliers=30, ba_loss_scale=None, ba_max_iterations=50, seed=0,
                workspace_bytes=WORKSPACE_BYTES) -> Reconstruction:
    """A reconstruction of the images of `graph` (verified, built from `pairs`) and `tracks` (built from it) with intrinsics K and no
    known camera.  `initialize_reconstruction` (the init_* arguments) chooses the pair (a, b); a gets [I | 0] and b the unit-baseline
    [R | t], and every other camera is zero.  Then each round:

        pts = triangulate_tracks(images=registered, max_error=tri_max_error, min_angle=tri_min_angle, seed=seed)
        ba = bundle_adjust(pts, fixed_poses=[a] + unregistered, fixed_tx=[b], loss_scale=ba_loss_scale,
                           max_iterations=ba_max_iterations, workspace_bytes=workspace_bytes);  R, t = ba.R, ba.t
        pts = triangulate_tracks(images=registered, ...)          # re-triangulated and re-filtered under the adjusted cameras
        stop ("all_registered") if every image is registered
        reg = register_images(pts, unregistered, max_error=abs_max_error, min_inliers=abs_min_inliers, seed=seed)
        stop ("no_image_added") if no image was accepted; otherwise the accepted images take their R, t and join the registered

    Every round adds an image, so there are at most N - 2.  The gauge is bundle_adjust's (COLMAP's): a's pose and b's x-translation
    are held.  Without an accepted initial pair nothing is registered and termination is "no_initial_pair" (no exception).  Every
    image that registration accepts is added in the same round (there is no next-best-view order and no local BA).

    Arguments are checked before any device work (ValueError).  Bit-identical from run to run.  Host reads: those of the stages, and
    the accepted flags of each registration."""
    what = "reconstruct"
    _float(what, "abs_max_error", abs_max_error, 0.0, True)
    _int(what, "abs_min_inliers", abs_min_inliers, 0)
    if ba_loss_scale is not None:
        _float(what, "ba_loss_scale", ba_loss_scale, 0.0, True)
    _int(what, "ba_max_iterations", ba_max_iterations, 0)
    _int(what, "workspace_bytes", workspace_bytes, 1)
    if not isinstance(graph, MatchGraph):
        raise ValueError(f"{what}: graph must be a MatchGraph, got {type(graph).__name__}")
    N = len(graph._kp_off) - 1
    _tri._check(graph, tracks, K, np.tile(np.eye(3), (max(N, 0), 1, 1)), np.zeros((max(N, 0), 3)), tri_max_error, tri_min_angle, 1,
                seed, what=what)
    _check_init(pairs, graph, K, init_pair, init_num_candidates, init_min_num_inliers, init_max_error, init_min_tri_angle,
                init_max_forward_motion, 0.999, 10000, seed, what=what)

    init = initialize_reconstruction(pairs, graph, K, init_pair=init_pair, num_candidates=init_num_candidates,
                                     min_num_inliers=init_min_num_inliers, max_error=init_max_error, min_tri_angle=init_min_tri_angle,
                                     max_forward_motion=init_max_forward_motion, seed=seed)
    dev = graph.kp_offsets.device
    with torch.cuda.device(dev):
        R = torch.zeros(N, 3, 3, dtype=torch.float64, device=dev)
        t = torch.zeros(N, 3, dtype=torch.float64, device=dev)
        tri = dict(max_error=tri_max_error, min_angle=tri_min_angle, seed=seed)
        if init.chosen < 0:
            pts = triangulate_tracks(graph, tracks, K, R, t, images=[], **tri)
            return Reconstruction(torch.zeros(N, dtype=torch.bool, device=dev), R, t, pts, init, [], "no_initial_pair")
        a, b = init.images[init.chosen].tolist()
        R[a] = torch.eye(3, dtype=torch.float64, device=dev)
        R[b], t[b] = init.R[init.chosen], init.t[init.chosen]
        registered, rounds = sorted((a, b)), []
        while True:
            rest = [i for i in range(N) if i not in registered]
            pts = triangulate_tracks(graph, tracks, K, R, t, images=registered, **tri)
            ba = bundle_adjust(graph, tracks, pts, K, R, t, fixed_poses=[a] + rest, fixed_tx=[b], loss_scale=ba_loss_scale,
                               max_iterations=ba_max_iterations, workspace_bytes=workspace_bytes)
            R, t = ba.R.clone(), ba.t.clone()
            pts = triangulate_tracks(graph, tracks, K, R, t, images=registered, **tri)
            rnd = dict(registered=list(registered), ba_termination=ba.termination, ba_cost=(float(ba.cost[0]), float(ba.cost[-1])),
                       ok_tracks=int(pts.ok.sum().item()), added=[])
            rounds.append(rnd)
            if not rest:
                termination = "all_registered"
                break
            reg = register_images(graph, tracks, pts, K, rest, max_error=abs_max_error, min_inliers=abs_min_inliers, seed=seed)
            acc = reg.accepted.tolist()
            rnd["added"] = [i for m, i in enumerate(rest) if acc[m]]
            if not rnd["added"]:
                termination = "no_image_added"
                break
            rows = torch.tensor([m for m in range(len(rest)) if acc[m]], device=dev)
            idx = torch.tensor(rnd["added"], device=dev)
            R[idx], t[idx] = reg.R[rows], reg.t[rows]
            registered = sorted(registered + rnd["added"])
        mask = torch.zeros(N, dtype=torch.bool, device=dev)
        mask[registered] = True
    return Reconstruction(mask, R, t, pts, init, rounds, termination)


# ---- COLMAP text model ---------------------------------------------------------------------------------------------------
def rotation_to_quaternion(R) -> np.ndarray:
    """Hamilton quaternions (qw, qx, qy, qz) with qw >= 0 of rotations R [..., 3, 3], by Shepperd's method: the largest of 1 + tr,
    1 + 2 R_00 - tr, ... chooses the component computed by a square root, so no division is by a small number."""
    R = np.asarray(R, np.float64)
    r = R.reshape(-1, 3, 3)
    tr = np.trace(r, axis1=1, axis2=2)
    d = np.stack((tr, r[:, 0, 0], r[:, 1, 1], r[:, 2, 2]), 1)
    which = np.argmax(d, 1)
    q = np.empty((r.shape[0], 4))
    for c in range(4):
        s = which == c
        m = r[s]
        if c == 0:
            w = 0.5 * np.sqrt(1.0 + tr[s])
            q[s] = np.stack((w, (m[:, 2, 1] - m[:, 1, 2]) / (4 * w), (m[:, 0, 2] - m[:, 2, 0]) / (4 * w), (m[:, 1, 0] - m[:, 0, 1]) / (4 * w)), 1)
        elif c == 1:
            x = 0.5 * np.sqrt(1.0 + m[:, 0, 0] - m[:, 1, 1] - m[:, 2, 2])
            q[s] = np.stack(((m[:, 2, 1] - m[:, 1, 2]) / (4 * x), x, (m[:, 0, 1] + m[:, 1, 0]) / (4 * x), (m[:, 0, 2] + m[:, 2, 0]) / (4 * x)), 1)
        elif c == 2:
            y = 0.5 * np.sqrt(1.0 - m[:, 0, 0] + m[:, 1, 1] - m[:, 2, 2])
            q[s] = np.stack(((m[:, 0, 2] - m[:, 2, 0]) / (4 * y), (m[:, 0, 1] + m[:, 1, 0]) / (4 * y), y, (m[:, 1, 2] + m[:, 2, 1]) / (4 * y)), 1)
        else:
            z = 0.5 * np.sqrt(1.0 - m[:, 0, 0] - m[:, 1, 1] + m[:, 2, 2])
            q[s] = np.stack(((m[:, 1, 0] - m[:, 0, 1]) / (4 * z), (m[:, 0, 2] + m[:, 2, 0]) / (4 * z), (m[:, 1, 2] + m[:, 2, 1]) / (4 * z), z), 1)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    q[q[:, 0] < 0] *= -1
    return q.reshape(R.shape[:-2] + (4,))


def _fmt(a) -> np.ndarray:
    """Every value of `a` as its shortest round-trip decimal string (vectorised)."""
    return np.char.mod("%.17g", np.asarray(a, np.float64))


def _join(*cols) -> np.ndarray:
    """The string columns joined row by row with single spaces (vectorised)."""
    out = np.asarray(cols[0]).astype(str)
    for c in cols[1:]:
        out = np.char.add(np.char.add(out, " "), np.asarray(c).astype(str))
    return out


def _host(v):
    return v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def write_colmap_text(path, recon: Reconstruction, graph: MatchGraph, tracks: Tracks, K, image_sizes, image_names=None) -> None:
    """Writes `recon` as COLMAP's text model into the directory `path` (created if needed): cameras.txt, images.txt and points3D.txt,
    with COLMAP's 1-based ids (image and camera i + 1, point k + 1 for track k).  One PINHOLE camera per image (fx fy cx cy of K[i],
    width and height from image_sizes [N, 2] = (H, W)); K with skew, or a last row other than (0, 0, 1), raises ValueError.  Keypoints
    and K are written as they are: the project's pixel frame has the top-left corner at (0, 0) and pixel centres at +0.5, as COLMAP's.
    images.txt lists the registered images: the Hamilton quaternion (QW >= 0) of R and t, then every keypoint of the image (so
    POINT2D_IDX is the keypoint id) with POINT3D_ID k + 1 when it is an inlier element of ok track k and -1 otherwise.  points3D.txt
    has one line per ok track: X, colour 128 128 128, ERROR = points.error and its inlier elements in element order.  image_names
    default to "image_<i>".  Values are written with 17 significant digits, so they read back exactly."""
    kp_off = np.asarray(graph._kp_off, np.int64)
    N = len(kp_off) - 1
    K = _tri._float64("K", K, (N, 3, 3), "write_colmap_text")
    if np.any(K[:, 0, 1] != 0) or np.any(K[:, 1, 0] != 0) or np.any(K[:, 2] != np.array([0.0, 0.0, 1.0])):
        raise ValueError("write_colmap_text: K must be a pinhole matrix [[fx, 0, cx], [0, fy, cy], [0, 0, 1]] (no skew)")
    sizes = _host(image_sizes).astype(np.int64).reshape(N, 2)
    names = [f"image_{i}" for i in range(N)] if image_names is None else [str(n) for n in image_names]
    if len(names) != N:
        raise ValueError(f"write_colmap_text: {len(names)} image names for {N} images")
    os.makedirs(path, exist_ok=True)
    reg = _host(recon.registered).astype(bool)
    R, t = _host(recon.R).astype(np.float64), _host(recon.t).astype(np.float64)
    kps = _host(graph.keypoints).astype(np.float64)
    tr_off = _host(tracks.track_offsets).astype(np.int64)
    el = _host(tracks.elements).astype(np.int64).reshape(-1, 2)
    ok, inl = _host(recon.points.ok).astype(bool), _host(recon.points.inlier).astype(bool)
    X, err = _host(recon.points.X).astype(np.float64), _host(recon.points.error).astype(np.float64)
    track = np.repeat(np.arange(len(tr_off) - 1), np.diff(tr_off))
    used = np.flatnonzero(inl & ok[track])                      # the inlier elements of ok tracks, in element order
    pid = np.full(kp_off[-1], -1, np.int64)
    pid[kp_off[el[used, 0]] + el[used, 1]] = track[used] + 1

    cam = _join(np.arange(1, N + 1), np.full(N, "PINHOLE"), sizes[:, 1], sizes[:, 0], _fmt(K[:, 0, 0]), _fmt(K[:, 1, 1]),
                _fmt(K[:, 0, 2]), _fmt(K[:, 1, 2]))
    with open(os.path.join(path, "cameras.txt"), "w") as f:
        f.write("# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n"
                f"# Number of cameras: {N}\n")
        f.write("\n".join(cam) + "\n")

    ids = np.flatnonzero(reg)
    q = rotation_to_quaternion(R[ids]) if ids.size else np.zeros((0, 4))
    with open(os.path.join(path, "images.txt"), "w") as f:
        f.write("# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n"
                f"#   POINTS2D[] as (X, Y, POINT3D_ID)\n# Number of images: {ids.size}\n")
        for m, i in enumerate(ids):
            head = " ".join([str(i + 1), *_fmt(q[m]), *_fmt(t[i]), str(i + 1), names[i]])
            b, e = kp_off[i], kp_off[i + 1]
            f.write(head + "\n" + " ".join(_join(_fmt(kps[b:e, 0]), _fmt(kps[b:e, 1]), pid[b:e])) + "\n")

    ks = np.flatnonzero(ok)
    with open(os.path.join(path, "points3D.txt"), "w") as f:
        f.write("# 3D point list with one line of data per point:\n"
                "#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n"
                f"# Number of points: {ks.size}\n")
        if ks.size:
            heads = np.char.add("\n", _join(ks + 1, _fmt(X[ks, 0]), _fmt(X[ks, 1]), _fmt(X[ks, 2]), np.full(ks.size, "128 128 128"),
                                            _fmt(err[ks])))
            elems = np.char.add(" ", _join(el[used, 0] + 1, el[used, 1]))
            starts = np.searchsorted(track[used], ks)            # the first inlier element of every ok track
            tokens = np.insert(elems.astype(object), starts, heads.astype(object))
            f.write("".join(tokens)[1:] + "\n")
