"""Writes tests/golden/triangulate_before_images.npz: what `triangulate_tracks` returns (X, ok, num_inliers, error, inlier) on two
seeded `planted_cameras` scenes, keyed "<scene>_<field>".  The committed file was made on an H100 by the release before
`triangulate_tracks` took the `images` argument (the commit "Bundle-adjust cameras and track points on the device"), so that
tests/test_absolute_pose_gpu.py pins `images=None` byte for byte to it.  Run from the repository root with a built library:

    python tests/golden/make_golden_triangulate.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from roma_b200 import build_tracks, consolidate_matches, synthetic, triangulate_tracks, verify_matches  # noqa: E402

# (seed, N, points, cell_size, outlier_frac) as in tests/test_absolute_pose_gpu.py
SCENES = {"a": (12, 6, 400, 1, 0.2), "b": (13, 5, 400, 4, 0.0)}


def main():
    out = {}
    for tag, (seed, N, points, cs, of) in SCENES.items():
        pairs, m, c, sizes, views, K, R, t, X = synthetic.planted_cameras(seed, N, points, size=(384, 512), cell_size=cs,
                                                                          outlier_frac=of, device="cuda")
        g = consolidate_matches(pairs, m, c, sizes, cell_size=cs)
        if of > 0:
            g = verify_matches(pairs, g, threshold={1: 2.0, 4: 3.0}[cs])[0]
        p = triangulate_tracks(g, build_tracks(pairs, g), K, R, t)
        for f in ("X", "ok", "num_inliers", "error", "inlier"):
            out[f"{tag}_{f}"] = getattr(p, f).cpu().numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "triangulate_before_images.npz"), **out)


if __name__ == "__main__":
    main()
