"""SHA-256 digests of `bundle_adjust` and `reconstruct` outputs, PINHOLE and per-image SIMPLE_RADIAL, on seeded `planted_cameras`
scenes.  The committed ba_digests.json was written on an H100 by the build before shared cameras (`camera_ids`) were added;
tests/test_shared_intrinsics_gpu.py recomputes the digests with the current build, so those paths stay byte-identical.

    python -m roma_b200.build && python tests/golden/make_golden_ba_digests.py [out.json]      (needs the GPU)
"""
import hashlib
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

DEV = "cuda"


def _sha(*vals) -> str:
    h = hashlib.sha256()
    for v in vals:
        if isinstance(v, torch.Tensor):
            v = v.detach().cpu().contiguous().numpy()
        h.update(np.ascontiguousarray(v).tobytes())
    return h.hexdigest()


def _ba_digest(res) -> str:
    vals = [res.R, res.t, res.points.X, res.points.error, res.cost, res.pred, res.accepted]
    if res.intrinsics is not None:
        vals.append(res.intrinsics)
    return _sha(*vals) + " " + res.termination


def _rec_digest(rec) -> str:
    vals = [rec.registered, rec.R, rec.t, rec.points.X, rec.points.ok, rec.points.error, rec.points.inlier]
    if rec.intrinsics is not None:
        vals.append(rec.intrinsics)
    return _sha(*vals) + " " + json.dumps(rec.rounds, sort_keys=True)


def digests() -> dict:
    from roma_b200 import build_tracks, bundle_adjust, consolidate_matches, reconstruct, synthetic, triangulate_tracks, verify_matches
    from roma_b200.camera import pinhole_K, undistort_graph

    out = {}
    thr = {1: 2.0, 4: 3.0}

    def graph(seed, N, points, cs, outlier_frac, radial, spread=False, verify=False):
        pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=(384, 512), cell_size=cs,
                                                                          outlier_frac=outlier_frac, radial=radial, spread=spread,
                                                                          device=DEV)
        g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
        if outlier_frac > 0 or verify:
            g = verify_matches(pairs, g, threshold=thr[cs])[0]
        return pairs, g, build_tracks(pairs, g), K, R, t

    for seed, N, cs, of, loss, points in [(0, 3, 1, 0.0, None, 500), (2, 8, 1, 0.2, None, 400), (3, 8, 4, 0.0, 2.0, 400),
                                          (5, 16, 4, 0.2, None, 300)]:
        pairs, g, tr, K, R, t = graph(seed, N, points, cs, of, None)
        R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
        pts = triangulate_tracks(g, tr, K, R1, t1, max_error=20.0)
        out[f"ba_pinhole_{seed}"] = _ba_digest(bundle_adjust(g, tr, pts, K, R1, t1, loss_scale=loss, max_iterations=100,
                                                             function_tolerance=1e-12))
        if seed == 2:
            out["ba_pinhole_gauge"] = _ba_digest(bundle_adjust(g, tr, pts, K, R1, t1, fixed_poses=(0, 3, 5), fixed_tx=(1, 6)))

    for seed, N, cs, of, loss, points in [(0, 3, 1, 0.0, None, 500), (1, 3, 4, 0.2, 1.0, 500), (2, 8, 1, 0.2, None, 400),
                                          (3, 8, 4, 0.0, 2.0, 400), (4, 16, 1, 0.0, 1.0, 300), (5, 16, 4, 0.2, None, 300)]:
        pairs, g, tr, intr, R, t = graph(seed, N, points, cs, of, (-0.05, 0.05))
        R1, t1 = synthetic.perturb_cameras(seed, R, t, 0.3, 0.05)
        rng = np.random.default_rng(seed)
        prior = intr.cpu().numpy().copy()
        prior[:, 0] *= 1 + rng.choice([-1.0, 1.0], N) * rng.uniform(0.02, 0.05, N)
        prior[:, 3] = 0.0
        pts = triangulate_tracks(undistort_graph(g, prior), tr, pinhole_K(prior), R1, t1, max_error=20.0)
        out[f"ba_radial_{seed}"] = _ba_digest(bundle_adjust(g, tr, pts, prior, R1, t1, camera_model="SIMPLE_RADIAL", loss_scale=loss,
                                                            max_iterations=100, function_tolerance=1e-12))
        if seed == 2:
            out["ba_radial_gauge"] = _ba_digest(bundle_adjust(g, tr, pts, prior, R1, t1, camera_model="SIMPLE_RADIAL",
                                                              fixed_poses=(0, 3, 5), fixed_tx=(1, 6), fixed_intrinsics=(2, 3),
                                                              max_iterations=30))

    pairs, g, tr, K, R, t = graph(11, 10, 1500, 1, 0.2, None)
    out["reconstruct_pinhole_11"] = _rec_digest(reconstruct(pairs, g, tr, K))
    for seed, N, spread in ((11, 10, False), (40, 30, True)):
        pairs, g, tr, intr, R, t = graph(seed, N, 1500, 1, 0.0, (-0.05, 0.05), spread)
        rng = np.random.default_rng(seed)
        prior = intr.cpu().numpy().copy()
        prior[:, 0] *= 1 + rng.uniform(-0.03, 0.03, N)
        prior[:, 3] = 0.0
        out[f"reconstruct_radial_{seed}"] = _rec_digest(reconstruct(pairs, g, tr, None, intrinsics=prior, refine_intrinsics=True))
    return out


if __name__ == "__main__":
    path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "ba_digests.json")
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    d = digests()
    with open(path, "w") as f:
        json.dump(d, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(d, indent=1, sort_keys=True))
