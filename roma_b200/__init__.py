"""roma_b200 — H100-native implementation of RoMa's dense `match()` / `sample()` path.

Drop-in for `romatch`'s public surface on that path (`romatch/__init__.py:2`):

    from roma_b200 import roma_outdoor
    model = roma_outdoor(device="cuda", weights=..., dinov2_weights=...)
    warp, certainty = model.match(im_A, im_B)
    matches, conf = model.sample(warp[0], certainty[0])
"""
DEBUG_MODE = False
RANK = 0
GLOBAL_STEP = 0
STEP_SIZE = 1
LOCAL_RANK = -1


def __getattr__(name):
    # factories import torch + the CUDA library lazily so that `import roma_b200.arch` stays light
    if name in ("roma_outdoor", "roma_indoor", "tiny_roma_v1_outdoor", "roma_model"):
        from . import model_zoo
        return getattr(model_zoo, name)
    if name == "decode_jpeg":
        from .jpeg import decode_jpeg
        return decode_jpeg
    if name in ("estimate_pose", "estimate_pose_batched", "find_homography", "find_homography_batched", "RANSAC", "find_fundamental",
                "find_fundamental_batched", "USAC_MAGSAC", "estimate_absolute_pose", "estimate_absolute_pose_batched"):
        from . import geometry
        return getattr(geometry, name)
    if name in ("consolidate_matches", "MatchGraph"):
        from . import match_graph
        return getattr(match_graph, name)
    if name in ("build_tracks", "Tracks"):
        from . import tracks
        return getattr(tracks, name)
    if name in ("verify_matches", "PairGeometry"):
        from . import verify
        return getattr(verify, name)
    if name in ("triangulate_tracks", "Points3D"):
        from . import triangulate
        return getattr(triangulate, name)
    if name in ("register_images", "Registration"):
        from . import register
        return getattr(register, name)
    if name in ("default_intrinsics", "pinhole_K", "undistort_keypoints", "undistort_graph"):
        from . import camera
        return getattr(camera, name)
    if name in ("bundle_adjust", "BundleResult"):
        from . import bundle
        return getattr(bundle, name)
    if name in ("initialize_reconstruction", "TwoViewInit", "reconstruct", "Reconstruction", "write_colmap_text"):
        from . import mapper
        return getattr(mapper, name)
    if name in ("triangulate_warps", "fuse_depth_maps", "write_ply", "DepthMaps", "DenseCloud"):
        from . import dense
        return getattr(dense, name)
    if name in ("select_pairs", "RetrievalPairs"):
        from . import retrieval
        return getattr(retrieval, name)
    if name in ("warp_kpts", "get_gt_warp", "dense_geometric_dist"):
        from . import depth_warp
        return getattr(depth_warp, name)
    raise AttributeError(name)
