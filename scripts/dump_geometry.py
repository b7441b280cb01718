"""Outputs of the device pose and homography estimators on fixed seeded inputs, so that two versions of the code can be compared
bit for bit: 64 ragged pairs of 2 000 to 10 000 points with 20 to 90 % outliers (`synthetic.two_view_scene` / `planar_scene`),
`max_iters` beyond one round, homographies by RANSAC and by least squares (method 0), and fundamental matrices by MAGSAC++.

    python scripts/dump_geometry.py --out FILE.npz

Writes R, t, ok and the concatenated masks of `estimate_pose_batched`, H, ok and masks of `find_homography_batched` per
method, and F, ok and masks of `find_fundamental_batched`, to one .npz; compare two such files array by array with np.array_equal.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    import numpy as np
    from roma_b200 import geometry, synthetic

    rng = np.random.default_rng(0)
    B = 64
    ns = rng.integers(2000, 10001, size=B)
    fracs = rng.uniform(0.2, 0.9, size=B)
    out = {"n": ns}
    scenes = [synthetic.two_view_scene(1000 + b, int(ns[b]), float(fracs[b])) for b in range(B)]
    K0, K1 = np.stack([s["K0"] for s in scenes]), np.stack([s["K1"] for s in scenes])
    R, t, ok, masks = geometry.estimate_pose_batched([s["kpts0"] for s in scenes], [s["kpts1"] for s in scenes], K0, K1, 0.5 / 2400,
                                                     max_iters=3000, seed=7)
    out.update(pose_R=R, pose_t=t, pose_ok=ok, pose_mask=np.concatenate(masks))
    planes = [synthetic.planar_scene(2000 + b, int(ns[b]), float(fracs[b])) for b in range(B)]
    for method in (geometry.RANSAC, 0):
        H, ok, masks = geometry.find_homography_batched([p["src"] for p in planes], [p["dst"] for p in planes], method, 3.0, 5000,
                                                        0.99999, seed=7)
        out.update({f"homog{method}_H": H, f"homog{method}_ok": ok, f"homog{method}_mask": np.concatenate(masks)})
    F, ok, masks = geometry.find_fundamental_batched([s["kpts0"] for s in scenes], [s["kpts1"] for s in scenes], geometry.USAC_MAGSAC,
                                                     0.2, 0.999999, 10000, seed=7)
    out.update(fund_F=F, fund_ok=ok, fund_mask=np.concatenate(masks))
    np.savez(args.out, **out)
    print({k: v.shape for k, v in out.items()}, "pose ok", int(out["pose_ok"].sum()), "homography ok", int(out["homog8_ok"].sum()),
          "fundamental ok", int(out["fund_ok"].sum()))


if __name__ == "__main__":
    main()
