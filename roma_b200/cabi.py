"""ctypes binding of libromab200.so — the thin shim between PyTorch (device memory, streams) and the C ABI.

The argument structs are generated from `include/romab200.h` itself at import time, so the Python side
cannot drift from the header.  Every pointer field takes a tensor (or None), never a raw address: an operand that starts
inside a buffer is passed as a view (`packing.at`), so its dtype, device, layout and extent are checked against what the call
describes before the library sees it.  `call` passes the tensors' addresses and the current CUDA stream; a non-zero return
code becomes a `RuntimeError` carrying `romab200_last_error()`.
There is no fallback: if the library is missing or the device is not an H100 (sm_90), calls fail loudly.
"""
from __future__ import annotations

import ctypes
import os
import re
from typing import Dict

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(HERE), "include", "romab200.h")
LIB_PATH = os.path.join(HERE, "lib", "libromab200.so")

RB_F32, RB_F16, RB_BF16, RB_F16S, RB_F64 = 0, 1, 2, 3, 4
ACT_NONE, ACT_RELU, ACT_GELU = 0, 1, 2
ROWMAP_NONE, ROWMAP_PAD_KEEP, ROWMAP_PAD_TO_COMPACT, ROWMAP_SEGMENT = 0, 1, 2, 3
EPI_LINEAR, EPI_COSKERNEL = 0, 1
BACKEND_AUTO, BACKEND_SIMT, BACKEND_TCGEN05 = 0, 1, 2
SAMPLE_IDENTITY, SAMPLE_THRESHOLD, SAMPLE_BALANCE = 0, 1, 2

DTYPE_CODE = {torch.float32: RB_F32, torch.float16: RB_F16, torch.bfloat16: RB_BF16}

_CTYPES = {
    "int32_t": ctypes.c_int32, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64, "float": ctypes.c_float, "double": ctypes.c_double,
}


def _parse_header(path: str):
    """Returns ({struct_name: [(field, ctype)]}, [function names]) parsed from the C header."""
    text = open(path).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    structs: Dict[str, list] = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", text, flags=re.S):
        fields = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            m = re.match(r"(const\s+)?(\w+)\s*(\*?)\s*(.*)$", decl, flags=re.S)
            base, ptr, names = m.group(2), m.group(3), m.group(4)
            first = True
            for part in names.split(","):
                part = part.strip()
                is_ptr = bool(ptr) if first else part.startswith("*")
                first = False
                part = part.lstrip("*").strip()
                arr = re.match(r"(\w+)\[(\d+)\]$", part)
                if is_ptr:
                    fields.append((part, ctypes.c_void_p))
                elif arr:
                    fields.append((arr.group(1), _CTYPES[base] * int(arr.group(2))))
                else:
                    fields.append((part, _CTYPES[base]))
        structs[name] = fields
    funcs = re.findall(r"\b(romab200_\w+)\s*\(", text)
    return structs, sorted(set(funcs))


STRUCT_FIELDS, FUNCTIONS = _parse_header(HEADER)
# integer constants of the header that the host side sizes buffers with
(RB_MG_TILE, RB_MG_PAIR_SMEM, RB_TRACKS_TILE, RB_TRACKS_BAD_ID, RB_TRACKS_WALK, RB_VERIFY_TILE, RB_VERIFY_BAD_ID, RB_VERIFY_PAIR_BYTES,
 RB_VERIFY_SLICE_BYTES, RB_VERIFY_POINT_BYTES, RB_VERIFY_CHUNK_BYTES, RB_TRI_GN_ITERS, RB_TRI_CAM, RB_TRI_BAD_ID) = (
    int(re.search(rf"#define\s+{name}\s+(\d+)", open(HEADER).read()).group(1))
    for name in ("RB_MG_TILE", "RB_MG_PAIR_SMEM", "RB_TRACKS_TILE", "RB_TRACKS_BAD_ID", "RB_TRACKS_WALK", "RB_VERIFY_TILE", "RB_VERIFY_BAD_ID",
                 "RB_VERIFY_PAIR_BYTES", "RB_VERIFY_SLICE_BYTES", "RB_VERIFY_POINT_BYTES", "RB_VERIFY_CHUNK_BYTES", "RB_TRI_GN_ITERS",
                 "RB_TRI_CAM", "RB_TRI_BAD_ID"))
RB_TRI_CTR = int(re.search(r"#define\s+RB_TRI_CTR\s+0x([0-9a-fA-F]+)u", open(HEADER).read()).group(1), 16)
(RB_BA_BAD_ID, RB_BA_REPEATED, RB_BA_CAM, RB_BA_TRACK, RB_BA_RESULT, RB_BA_NB, RB_BA_ELEMENT_BYTES, RB_BA_TRACK_BYTES, RB_BA_IMAGE_BYTES,
 RB_BA_FREE_BYTES, RB_BA_ONCE_BYTES, RB_BA_CAM1, RB_BA_ELEMENT_BYTES1, RB_BA_IMAGE_BYTES1, RB_BA_FREE_BYTES1) = (
    int(re.search(rf"#define\s+{name}\s+(\d+)", open(HEADER).read()).group(1))
    for name in ("RB_BA_BAD_ID", "RB_BA_REPEATED", "RB_BA_CAM", "RB_BA_TRACK", "RB_BA_RESULT", "RB_BA_NB", "RB_BA_ELEMENT_BYTES",
                 "RB_BA_TRACK_BYTES", "RB_BA_IMAGE_BYTES", "RB_BA_FREE_BYTES", "RB_BA_ONCE_BYTES", "RB_BA_CAM1", "RB_BA_ELEMENT_BYTES1",
                 "RB_BA_IMAGE_BYTES1", "RB_BA_FREE_BYTES1"))
(RB_ABS_ROUND, RB_ABS_MAX_SOL, RB_ABS_MAX_SPLITS, RB_ABS_SLICE, RB_ABS_STATE, RB_ABS_MAX_BATCH, RB_REG_BAD_ID, RB_REG_ITEM_BYTES, RB_REG_SLICE_BYTES,
 RB_REG_POINT_BYTES, RB_REG_CHUNK_BYTES) = (
    int(re.search(rf"#define\s+{name}\s+(\d+)", open(HEADER).read()).group(1))
    for name in ("RB_ABS_ROUND", "RB_ABS_MAX_SOL", "RB_ABS_MAX_SPLITS", "RB_ABS_SLICE", "RB_ABS_STATE", "RB_ABS_MAX_BATCH", "RB_REG_BAD_ID", "RB_REG_ITEM_BYTES",
                 "RB_REG_SLICE_BYTES", "RB_REG_POINT_BYTES", "RB_REG_CHUNK_BYTES"))
RB_DENSE_CAM, RB_DENSE_REASONS, RB_DENSE_MAX_CTAS, RB_DENSE_TILE = (
    int(re.search(rf"#define\s+{name}\s+(\d+)", open(HEADER).read()).group(1))
    for name in ("RB_DENSE_CAM", "RB_DENSE_REASONS", "RB_DENSE_MAX_CTAS", "RB_DENSE_TILE"))
STRUCTS = {name: type(name, (ctypes.Structure,), {"_fields_": fields}) for name, fields in STRUCT_FIELDS.items()}
_PTR_FIELDS = {name: {f for f, t in fields if t is ctypes.c_void_p} for name, fields in STRUCT_FIELDS.items()}

_lib = None


def load_library(path: str = LIB_PATH) -> ctypes.CDLL:
    """dlopen the in-tree library and type its entry points.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise RuntimeError(f"{path} not found: build it with `python -m roma_b200.build` "
                           "(there is no CPU or PyTorch fallback for the CUDA path)")
    lib = ctypes.CDLL(path)
    lib.romab200_last_error.restype = ctypes.c_char_p
    lib.romab200_abi_version.restype = ctypes.c_int
    lib.romab200_device_ok.restype = ctypes.c_int
    lib.romab200_launch_count.restype = ctypes.c_ulonglong
    for fn in FUNCTIONS:
        getattr(lib, fn)            # AttributeError if the header declares a symbol the library lacks
    _lib = lib
    return lib


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


launch_count = 0      # number of C-ABI calls made (bench.py reports kernel launches from it)

# ---- argument validation: the C ABI takes raw pointers, so a tensor of the wrong dtype / device / layout would be silent garbage.
# For every struct: tensor field -> the field that carries its dtype code (or a fixed torch dtype).
_CODE_DTYPE = {RB_F32: torch.float32, RB_F16: torch.float16, RB_BF16: torch.bfloat16, RB_F16S: torch.float16, RB_F64: torch.float64}
_F32 = torch.float32
_F64 = torch.float64
_FIELD_DTYPES = {
    "rb_gemm_args": {"A": "dtype_ab", "B": "dtype_ab", "A_lo": torch.float16, "B_lo": torch.float16, "C": "dtype_c", "C_lo": torch.float16,
                     "R": "dtype_r", "bias": _F32, "col_scale": _F32, "norm_a": _F32, "norm_b": _F32},
    "rb_layernorm_args": {"x": "dtype_x", "y": "dtype_y", "y_lo": torch.float16, "gamma": _F32, "beta": _F32},
    "rb_softmax_args": {"s": "dtype", "out_hi": torch.float16, "out_lo": torch.float16},
    "rb_flash_attn_args": {"qkv": "dtype", "out": "dtype", "qkv_lo": torch.float16, "out_lo": torch.float16},
    "rb_rownorm_args": {"x": "dtype", "out": _F32},
    "rb_copy2d_args": {"src": "dtype_src", "dst": "dtype_dst", "row_scale": _F32},
    "rb_gather_rows_args": {"src_index": torch.int32, "dst_index": torch.int32},
    "rb_split_pair_args": {"x": _F32, "hi": torch.float16, "lo": torch.float16, "row_norm": _F32},
    "rb_conv_first_args": {"image": _F32, "out": "dtype_out", "out_lo": torch.float16, "weight": _F32, "bias": _F32},
    "rb_maxpool_args": {"in": "dtype", "out": "dtype", "in_lo": torch.float16, "out_lo": torch.float16},
    "rb_im2col_args": {"image": _F32, "out": "dtype_out"},
    "rb_tokens_args": {"patch": _F32, "cls": _F32, "pos": _F32, "tokens": _F32},
    "rb_gp_solve_args": {"W": _F32},
    "rb_cls_args": {"logits": "dtype", "state": _F32},
    "rb_refiner_prologue_args": {"feat": "dtype", "state": _F32, "d": "dtype", "emb_weight": _F32, "emb_bias": _F32, "grid_x": _F32, "grid_y": _F32,
                                 "win_x": _F32, "win_y": _F32, "tile_done": torch.uint8, "corr_table": _F32},
    "rb_local_corr_args": {"f0": "dtype_f", "f1": "dtype_f", "flow": _F32, "out": "dtype_out", "win_x": _F32, "win_y": _F32},
    "rb_local_corr_warp_args": {"f0": _F32, "f1": _F32, "warp": _F32, "out": _F32},
    "rb_dwconv_args": {"in": "dtype", "weight": _F32, "bias": _F32, "out_lo": torch.float16},
    "rb_refiner_block_small_args": {"in": "dtype", "out": "dtype", "dw_weight": _F32, "dw_bias": _F32, "pw_weight_host": _F32, "pw_bias_host": _F32},
    "rb_refiner_block_c144_args": {"in": "dtype", "out": "dtype", "dw_weight": _F32, "dw_bias": _F32, "pw_weight": "dtype", "pw_bias": _F32},
    "rb_refiner_block_c144_split_args": {"in": _F32, "out": _F32, "dw_weight": _F32, "dw_bias": _F32, "pw_weight": torch.float16,
                                         "pw_weight_lo": torch.float16, "pw_bias": _F32},
    "rb_refiner_tail_args": {"d": "dtype", "weight": _F32, "bias": _F32, "state": _F32, "delta_out": _F32},
    "rb_resize_args": {"in": _F32, "out": _F32},
    "rb_match_epilogue_args": {"state": _F32, "coarse_state": _F32, "warp": _F32, "cert": _F32, "grid_x": _F32, "grid_y": _F32},
    "rb_kde_args": {"x": _F32, "density": _F32, "workspace": _F32},
    "rb_preprocess_args": {"in": torch.uint8, "tmp": torch.uint8, "out_u8": torch.uint8, "out": _F32, "bounds_x": torch.int32, "kk_x": torch.int32,
                           "bounds_y": torch.int32, "kk_y": torch.int32},
    "rb_sample_args": {"values": _F32, "out_idx": torch.int32, "out_weights": _F32, "keys": _F32, "scratch": torch.int32, "seed_dev": torch.int64},
    "rb_sample_gather_args": {"matches": _F32, "certainty": _F32, "idx": torch.int32, "out_matches": _F32, "out_certainty": _F32},
    "rb_tiny_conv_args": {"in": _F32, "out": _F32, "weight": _F32, "bias": _F32, "col_scale": _F32, "R": _F32},
    "rb_tiny_gray_args": {"in": _F32, "out": _F32},
    "rb_tiny_avgpool_args": {"in": _F32, "out": _F32},
    "rb_tiny_add3_args": {"a": _F32, "b": _F32, "c": _F32, "out": _F32},
    "rb_tiny_pos_embed_args": {"f0": _F32, "f1": _F32, "state": _F32, "grid_x": _F32, "grid_y": _F32, "grid_lr_x": _F32, "grid_lr_y": _F32},
    "rb_tiny_warp_concat_args": {"f0": _F32, "f1": _F32, "state": _F32, "out": _F32},
    "rb_tiny_epilogue_args": {"state": _F32, "warp": _F32, "cert": _F32, "grid_x": _F32, "grid_y": _F32},
    "rb_keypoints_sample_args": {"x": _F32, "warp": _F32, "cert": _F32, "x_to_B": _F32, "cert_out": _F32},
    "rb_keypoints_mnn_args": {"x_A_to_B": _F32, "cert_A": _F32, "x_B": _F32, "workspace": _F32, "offsets": torch.int64, "inds_A": torch.int64,
                              "inds_B": torch.int64},
    "rb_jpeg_args": {"stream": torch.uint8, "desc": torch.int64, "tables": torch.int32, "comp": torch.uint8, "chunks": torch.int32,
                     "istart": torch.int32, "exits": torch.int64, "counts": torch.int32, "coef": torch.int16, "state": torch.int32,
                     "flags": torch.int32, "planes": torch.uint8, "out": torch.uint8},
    "rb_pose_args": {"x0": _F64, "x1": _F64, "offsets": torch.int64, "K": _F64, "xn": _F64, "sample": torch.int32, "E": _F64, "nsol": torch.int32,
                     "counts": torch.int32, "state": torch.int32, "best_E": _F64, "running": torch.int32, "R": _F64, "t": _F64, "ok": torch.uint8,
                     "mask": torch.uint8},
    "rb_homography_args": {"src": _F32, "dst": _F32, "offsets": torch.int64, "sample": torch.int32, "attempts": torch.int32, "status": torch.int32,
                           "H": _F64, "counts": torch.int32, "state": torch.int32, "best_H": _F64, "running": torch.int32, "out_H": _F64,
                           "ok": torch.uint8, "mask": torch.uint8},
    "rb_fund_args": {"x0": _F64, "x1": _F64, "offsets": torch.int64, "table": _F64, "norm": _F64, "xn": _F64, "sample": torch.int32,
                     "nmod": torch.int32, "F": _F64, "counts": torch.int32, "losses": _F64, "state": torch.int32, "best_F": _F64,
                     "best_loss": _F64, "running": torch.int32, "out_F": _F64, "ok": torch.uint8, "mask": torch.uint8},
    "rb_match_graph_keypoints_args": {"pairs": torch.int64, "matches": _F32, "certainty": _F32, "image_sizes": torch.int32, "cell_start": torch.int64,
                                      "tile_start": torch.int64, "grid_bits": torch.int32, "grid_g": torch.int64, "tile_scan": torch.int64,
                                      "kp_offsets": torch.int64, "keypoints": _F32, "kp_scores": _F32, "sid": torch.int32},
    "rb_match_graph_pairs_args": {"sid": torch.int32, "certainty": _F32, "scratch": torch.uint8, "match_offsets": torch.int64,
                                  "matches": torch.int32, "match_scores": _F32},
    "rb_tracks_args": {"pairs": torch.int64, "kp_offsets": torch.int64, "match_offsets": torch.int64, "matches": torch.int32, "match_scores": _F32,
                       "parent": torch.int32, "size": torch.int32, "tile_scan": torch.int64, "info": torch.int64, "kp_track": torch.int32,
                       "keys": torch.int64, "keys_alt": torch.int64, "hist": torch.int32, "track_offsets": torch.int64, "elements": torch.int32},
    "rb_verify_args": {"pairs": torch.int64, "kp_offsets": torch.int64, "keypoints": _F32, "match_offsets": torch.int64, "matches": torch.int32,
                       "match_scores": _F32, "info": torch.int64, "x0": _F64, "x1": _F64, "chunk_offsets": torch.int64, "ok": torch.uint8,
                       "mask": torch.uint8, "num_inliers": torch.int64, "accepted": torch.uint8, "tile_scan": torch.int64,
                       "out_offsets": torch.int64, "out_matches": torch.int32, "out_scores": _F32, "pair_list": torch.int32},
    "rb_tri_args": {"track_offsets": torch.int64, "elements": torch.int32, "kp_offsets": torch.int64, "keypoints": _F32, "cameras": _F64,
                    "info": torch.int64, "X": _F64, "ok": torch.uint8, "num_inliers": torch.int32, "error": _F64, "inlier": torch.uint8},
    "rb_ba_args": {"track_offsets": torch.int64, "elements": torch.int32, "kp_offsets": torch.int64, "keypoints": _F32, "track_ok": torch.uint8,
                   "inlier": torch.uint8, "free_index": torch.int32, "free_cams": torch.int32, "fixed_tx": torch.uint8, "info": torch.int64,
                   "elem_track": torch.int32, "keys": torch.int64, "keys_alt": torch.int64, "hist": torch.int32, "obs_offsets": torch.int64,
                   "obs": torch.int32, "cams": _F64, "X": _F64, "cams_trial": _F64, "X_trial": _F64, "W": _F64, "track_sys": _F64,
                   "cam_sys": _F64, "S": _F64, "rhs": _F64, "cam_pred": _F64, "track_part": _F64, "result": _F64, "error": _F64,
                   "pin": torch.uint8},
    "rb_ba_groups_args": {"group_offsets": torch.int32, "group_members": torch.int32, "group_pin": torch.uint8, "S": _F64, "rhs": _F64,
                          "S_groups": _F64, "rhs_groups": _F64, "result": _F64},
    "rb_abspose_args": {"x": _F64, "X": _F64, "offsets": torch.int64, "K": _F64, "sample": torch.int32, "models": _F64, "nsol": torch.int32,
                        "counts": torch.int32, "state": torch.int32, "best": _F64, "running": torch.int32, "R": _F64, "t": _F64, "ok": torch.uint8,
                        "num_inliers": torch.int64, "mask": torch.uint8},
    "rb_register_args": {"track_offsets": torch.int64, "elements": torch.int32, "kp_offsets": torch.int64, "keypoints": _F32, "track_ok": torch.uint8,
                         "points": _F64, "info": torch.int64, "keys": torch.int64, "keys_alt": torch.int64, "hist": torch.int32,
                         "image_offsets": torch.int64, "elem": torch.int32, "track": torch.int32, "images": torch.int32,
                         "out_offsets": torch.int64, "x": _F64, "X": _F64},
    "rb_undistort_args": {"kp_offsets": torch.int64, "keypoints": _F32, "intrinsics": _F64, "out": _F32, "clamped": torch.int64},
    "rb_twoview_args": {"offsets": torch.int64, "x0": _F64, "x1": _F64, "xn": _F64, "mask": torch.uint8, "K": _F64, "R": _F64, "t": _F64,
                        "ok": torch.uint8, "angle": _F64, "num_good": torch.int64, "median_angle": _F64, "forward": _F64},
    "rb_warp_kpts_args": {"depth0": "depth_dtype", "depth1": "depth_dtype", "T": _F64, "K0": _F64, "K1": _F64, "kpts": "kpts_dtype", "warped": _F64,
                          "valid": torch.uint8},
    "rb_gt_warp_args": {"depth0": "depth_dtype", "depth1": "depth_dtype", "T": _F64, "K0": _F64, "K1": _F64, "grid_x": _F32, "grid_y": _F32,
                        "x2": _F64, "prob": _F32},
    "rb_dense_geometric_dist_args": {"depth0": "depth_dtype", "depth1": "depth_dtype", "T": _F64, "K0": _F64, "K1": _F64, "dense_matches": _F32,
                                     "gd": _F64, "prob": _F32, "partial_sum": _F64, "partial_cnt": torch.int32, "pair_sum": _F64,
                                     "pair_cnt": torch.int64, "pck": _F32, "epe": _F64},
    "rb_dense_tri_args": {"pairs": torch.int64, "warp": _F32, "certainty": _F32, "image_sizes": torch.int32, "cameras": _F64,
                          "registered": torch.uint8, "images": torch.int32, "depth": _F32, "score": _F32, "source": torch.int64,
                          "elem_depth": _F32, "partial": torch.int32, "pair_counts": torch.int64},
    "rb_dense_fuse_args": {"image_sizes": torch.int32, "cameras": _F64, "registered": torch.uint8, "nbr_offsets": torch.int64,
                           "nbrs": torch.int32, "depth": _F32, "score": _F32, "colors": torch.uint8, "color_offsets": torch.int64,
                           "color_sizes": torch.int32, "tile_scan": torch.int64, "points": _F64, "rgb": torch.uint8, "image": torch.int32,
                           "pixel": torch.int64, "num_views": torch.int32, "point_score": _F32},
}
# tensor fields that the call describes with explicit element strides, so they may be non-contiguous views
_STRIDED_FIELDS = {"rb_keypoints_sample_args": {"warp", "cert"}, "rb_dense_geometric_dist_args": {"dense_matches"}}
# pointer fields the library reads on the host (the refiner block passes these weights as kernel parameters): CPU tensors
_HOST_FIELDS = {"rb_refiner_block_small_args": {"pw_weight_host", "pw_bias_host"}}


def _gemm_min_elems(kw):
    """(field, minimum number of elements) of the GEMM operands for the given geometry."""
    b0, b1 = kw.get("batch0", 1) or 1, kw.get("batch1", 1) or 1
    M, N, K, nt = kw["M"], kw["N"], kw["K"], kw.get("ntaps", 1) or 1
    offa = (b0 - 1) * kw.get("sa0", 0) + (b1 - 1) * kw.get("sa1", 0)
    offb = (b0 - 1) * kw.get("sb0", 0) + (b1 - 1) * kw.get("sb1", 0)
    offc = (b0 - 1) * kw.get("sc0", 0) + (b1 - 1) * kw.get("sc1", 0)
    a = offa + ((kw.get("a_rows") or M) - 1) * kw["lda"] + K // nt
    b = offb + ((K - 1) * kw["ldb"] + N if kw.get("trans_b", 0) else (N - 1) * kw["ldb"] + K)
    rows_out = M
    if kw.get("rowmap", 0) == ROWMAP_PAD_TO_COMPACT:
        rows_out = M // (kw["pad_h"] * kw["pad_w"]) * (kw["pad_h"] - 2) * (kw["pad_w"] - 2)
    elif kw.get("rowmap", 0) == ROWMAP_SEGMENT:
        rows_out = (M - 1) // kw["seg_in"] * kw["seg_out"] + (M - 1) % kw["seg_in"] + kw.get("seg_off", 0) + 1
    c = offc + (rows_out - 1) * kw["ldc"] + N
    return {"A": a, "A_lo": a, "B": b, "B_lo": b, "C": c, "C_lo": c}


def _copy2d_min_elems(kw):
    return {"src": (kw["rows"] - 1) * kw["lds"] + kw["cols"], "dst": (kw["rows"] - 1) * kw["ldd"] + kw["cols"]}


def _gather_rows_min_elems(kw):
    """The row geometry is in bytes; converted to elements of the tensor passed."""
    out = {}
    for k, rows, ld in (("src", "src_rows", "ld_src"), ("dst", "dst_rows", "ld_dst")):
        if isinstance(kw.get(k), torch.Tensor):
            out[k] = -(-((kw[rows] - 1) * kw[ld] + kw["row_bytes"]) // kw[k].element_size())
    return out


def _sample_min_elems(kw):
    b, n, k, rep = max(kw.get("batch", 1), 1), kw["n"], kw["k"], max(kw.get("repeats", 0), 1)
    return {"values": ((b - 1) // rep) * (kw.get("stride") or n) + n, "keys": b * n, "scratch": b * 2056, "out_idx": b * k, "out_weights": b * k,
            "seed_dev": (b - 1) * kw.get("seed_stride", 0) + 1}


def _sample_gather_min_elems(kw):
    items, k, rows = kw["items"], kw["k"], ((kw["items"] - 1) // max(kw.get("repeats", 0), 1) + 1) * kw["n"]
    return {"matches": 4 * rows, "certainty": rows, "idx": items * k, "out_matches": 4 * items * k, "out_certainty": items * k}


def _match_graph_keypoints_min_elems(kw):
    sides, img = kw["num_pairs"] * kw["n"], kw["num_images"] + 1
    return {"pairs": 2 * kw["num_pairs"], "matches": 4 * sides, "certainty": sides, "image_sizes": 2 * kw["num_images"], "cell_start": img,
            "tile_start": img, "grid_bits": kw["grid_cells"], "grid_g": kw["grid_cells"], "tile_scan": kw["grid_tiles"] + 1, "kp_offsets": img,
            "keypoints": 2 * kw["kp_capacity"], "kp_scores": kw["kp_capacity"], "sid": 2 * sides}


def _match_graph_pairs_min_elems(kw):
    sides, cap = kw["num_pairs"] * kw["n"], kw.get("match_capacity", 0)
    return {"sid": 2 * sides, "certainty": sides, "scratch": kw.get("scratch_bytes", 0), "match_offsets": kw["num_pairs"] + 1,
            "matches": 2 * cap, "match_scores": cap}


def _tracks_min_elems(kw):
    K, kept, tile = kw["num_rows"], kw.get("num_kept", 0), RB_TRACKS_TILE
    return {"pairs": 2 * kw["num_pairs"], "kp_offsets": kw["num_images"] + 1, "match_offsets": kw["num_pairs"] + 1, "matches": 2 * kw["num_matches"],
            "match_scores": kw["num_matches"], "parent": K, "size": K, "tile_scan": (K + tile - 1) // tile + 1, "info": 5, "kp_track": K,
            "keys": kept, "keys_alt": kept, "hist": 256 * ((kept + tile - 1) // tile) + 1, "track_offsets": kept // 2 + 1, "elements": 2 * kept}


def _verify_min_elems(kw):
    P, M, kept, tiles = kw["num_pairs"], kw["num_matches"], kw.get("num_kept", 0), (kw["num_matches"] + RB_VERIFY_TILE - 1) // RB_VERIFY_TILE
    out = {"pairs": 2 * P, "kp_offsets": kw["num_images"] + 1, "keypoints": 2 * kw["num_rows"], "match_offsets": P + 1, "matches": 2 * M,
           "match_scores": M, "info": 2, "ok": P, "mask": M, "num_inliers": P, "accepted": P, "tile_scan": tiles + 1, "out_offsets": P + 1,
           "out_matches": 2 * kept, "out_scores": kept}
    if "chunk_offsets" in kw:
        out["chunk_offsets"] = kw["pair_end"] - kw["pair_begin"] + 1
    if kw.get("pair_list") is not None:
        out["pair_list"] = kw["pair_end"]
    return out


def _tri_min_elems(kw):
    T, N, E = kw["num_tracks"], kw["num_images"], kw["num_elements"]
    return {"track_offsets": T + 1, "elements": 2 * E, "kp_offsets": N + 1, "keypoints": 2 * kw["num_rows"], "cameras": N * RB_TRI_CAM,
            "info": 1, "X": 3 * T, "ok": T, "num_inliers": T, "error": T, "inlier": E}


def _ba_min_elems(kw):
    T, N, F, E = kw["num_tracks"], kw["num_images"], kw.get("num_free", 0), kw["num_elements"]
    nc, cam = (8, RB_BA_CAM1) if kw.get("camera_model", 0) == 1 else (6, RB_BA_CAM)
    n = nc * F
    return {"track_offsets": T + 1, "elements": 2 * E, "kp_offsets": N + 1, "keypoints": 2 * kw["num_rows"], "track_ok": T, "inlier": E,
            "free_index": N, "free_cams": F, "fixed_tx": F, "info": 2, "elem_track": E, "keys": E, "keys_alt": E,
            "hist": 256 * ((E + RB_TRACKS_TILE - 1) // RB_TRACKS_TILE) + 1, "obs_offsets": N + 1, "obs": E, "cams": N * cam,
            "X": 3 * T, "cams_trial": N * cam, "X_trial": 3 * T, "W": 3 * nc * E, "track_sys": T * RB_BA_TRACK, "cam_sys": 2 * nc * F,
            "S": n * n, "rhs": n, "cam_pred": N, "track_part": 3 * T, "result": RB_BA_RESULT, "error": T, "pin": 8 * F}


def _ba_groups_min_elems(kw):
    F, G = kw["num_free"], kw["num_groups"]
    ng = 6 * F + 2 * G
    return {"group_offsets": G + 1, "group_members": F, "group_pin": 2 * G, "S": 64 * F * F, "rhs": 8 * F, "S_groups": ng * ng,
            "rhs_groups": ng, "result": RB_BA_RESULT}


def abspose_splits(max_n) -> int:
    """Score slices of an absolute-pose launch whose largest item has max_n points (include/romab200.h)."""
    return max(1, min(RB_ABS_MAX_SPLITS, -(-int(max_n) // RB_ABS_SLICE)))


def _abspose_min_elems(kw):
    B, total = kw["batch"], kw["x"].numel() // 2
    splits = abspose_splits(kw["max_n"])
    return {"x": 2 * total, "X": 3 * total, "offsets": B + 1, "K": 9 * B, "sample": 3 * B * RB_ABS_ROUND, "models": 12 * B * RB_ABS_ROUND * RB_ABS_MAX_SOL,
            "nsol": B * RB_ABS_ROUND, "counts": B * splits * RB_ABS_MAX_SOL * RB_ABS_ROUND,
            "state": B * RB_ABS_STATE, "best": 12 * B, "running": 1, "R": 9 * B, "t": 3 * B, "ok": B, "num_inliers": B, "mask": total}


def _register_min_elems(kw):
    T, N, E = kw["num_tracks"], kw["num_images"], kw["num_elements"]
    out = {"track_offsets": T + 1, "elements": 2 * E, "kp_offsets": N + 1, "keypoints": 2 * kw["num_rows"], "track_ok": T, "points": 3 * T,
           "info": 1, "keys": E, "keys_alt": E, "hist": 256 * ((E + RB_TRACKS_TILE - 1) // RB_TRACKS_TILE) + 1, "image_offsets": N + 1,
           "elem": E, "track": E}
    if kw.get("num_list"):
        total = kw["x"].numel() // 2
        out.update(images=kw["num_list"], out_offsets=kw["num_list"] + 1, X=3 * total)
    return out


def _undistort_min_elems(kw):
    return {"kp_offsets": kw["num_images"] + 1, "keypoints": 2 * kw["num_rows"], "intrinsics": 4 * kw["num_images"], "out": 2 * kw["num_rows"],
            "clamped": 1}


def _twoview_min_elems(kw):
    B, total = kw["batch"], kw["mask"].numel()
    return {"offsets": B + 1, "x0": 2 * total, "x1": 2 * total, "xn": 4 * total, "K": 18 * B, "R": 9 * B, "t": 3 * B, "ok": B,
            "angle": total, "num_good": B, "median_angle": B, "forward": B}


def _dense_tri_min_elems(kw):
    P, N, C, n = kw["num_pairs"], kw["num_images"], kw["chunk"], kw["H"] * kw["W"]
    return {"pairs": 2 * P, "warp": 8 * C * n, "certainty": 2 * C * n, "image_sizes": 2 * N, "cameras": N * RB_DENSE_CAM, "registered": N,
            "images": kw["num_list"], "depth": N * n, "score": N * n, "source": N * n, "elem_depth": 2 * C * n,
            "partial": 2 * C * RB_DENSE_MAX_CTAS * RB_DENSE_REASONS, "pair_counts": P * RB_DENSE_REASONS}


def _dense_fuse_min_elems(kw):
    N, n, M = kw["num_images"], kw["H"] * kw["W"], kw.get("num_points", 0)
    out = {"image_sizes": 2 * N, "cameras": N * RB_DENSE_CAM, "registered": N, "nbr_offsets": N + 1, "depth": N * n, "score": N * n,
           "color_offsets": N + 1, "color_sizes": 2 * N, "tile_scan": N * (-(-n // RB_DENSE_TILE)) + 1, "points": 3 * M, "rgb": 3 * M,
           "image": M, "pixel": M, "num_views": M, "point_score": M}
    if kw.get("colors") is not None:
        out["colors"] = kw["color_bytes"]
    return out


# struct -> function of the call's arguments giving {field: minimum number of elements} for the described geometry
_MIN_ELEMS = {"rb_gemm_args": _gemm_min_elems, "rb_copy2d_args": _copy2d_min_elems, "rb_gather_rows_args": _gather_rows_min_elems,
              "rb_sample_args": _sample_min_elems, "rb_sample_gather_args": _sample_gather_min_elems,
              "rb_match_graph_keypoints_args": _match_graph_keypoints_min_elems, "rb_match_graph_pairs_args": _match_graph_pairs_min_elems,
              "rb_tracks_args": _tracks_min_elems, "rb_verify_args": _verify_min_elems, "rb_tri_args": _tri_min_elems,
              "rb_ba_args": _ba_min_elems, "rb_ba_groups_args": _ba_groups_min_elems, "rb_abspose_args": _abspose_min_elems,
              "rb_register_args": _register_min_elems,
              "rb_twoview_args": _twoview_min_elems, "rb_undistort_args": _undistort_min_elems,
              "rb_dense_tri_args": _dense_tri_min_elems, "rb_dense_fuse_args": _dense_fuse_min_elems}


def _validate(fn_name, struct_name, kw):
    table = _FIELD_DTYPES.get(struct_name, {})
    cur = torch.cuda.current_device() if torch.cuda.is_available() else None
    mins = _MIN_ELEMS[struct_name](kw) if struct_name in _MIN_ELEMS else {}
    strided = _STRIDED_FIELDS.get(struct_name, ())
    host = _HOST_FIELDS.get(struct_name, ())
    for k, v in kw.items():
        if not isinstance(v, torch.Tensor):
            if v is not None and k in _PTR_FIELDS[struct_name]:
                raise TypeError(f"{fn_name}: pointer field `{k}` takes a tensor or None, not {type(v).__name__} "
                                "(pass an operand that starts inside a buffer as a view, packing.at)")
            continue
        if k in host:
            if v.device.type != "cpu":
                raise RuntimeError(f"{fn_name}: argument `{k}` is read on the host, it must be a CPU tensor (got one on {v.device})")
        elif not v.is_cuda or (cur is not None and v.device.index != cur):
            raise RuntimeError(f"{fn_name}: argument `{k}` lives on {v.device}, expected the current CUDA device cuda:{cur}")
        if k not in strided and not v.is_contiguous():
            raise RuntimeError(f"{fn_name}: argument `{k}` is not contiguous (shape {tuple(v.shape)}, strides {v.stride()})")
        want = table.get(k)
        if isinstance(want, str):
            want = _CODE_DTYPE.get(kw.get(want))
        if want is not None and v.dtype != want:
            raise RuntimeError(f"{fn_name}: argument `{k}` has dtype {v.dtype}, the call describes it as {want}")
        if k in mins and v.numel() < mins[k]:
            raise RuntimeError(f"{fn_name}: argument `{k}` holds {v.numel()} elements, the described geometry needs {mins[k]}")


def call(fn_name: str, struct_name: str, **kw) -> None:
    """Fill `struct_name` from keyword arguments (a pointer field takes a tensor, passed as its address, or None) and call `fn_name`."""
    global launch_count
    lib = load_library()
    args = STRUCTS[struct_name]()
    valid = {f for f, _ in STRUCT_FIELDS[struct_name]}
    for k in kw:
        if k not in valid:
            raise TypeError(f"{struct_name} has no field {k}")
    _validate(fn_name, struct_name, kw)
    for k, v in kw.items():
        if k in _PTR_FIELDS[struct_name]:
            setattr(args, k, None if v is None else v.data_ptr())
        elif isinstance(v, (list, tuple)):
            arr = getattr(args, k)
            for i, x in enumerate(v):
                arr[i] = x
        else:
            setattr(args, k, v)
    rc = getattr(lib, fn_name)(ctypes.byref(args), _stream())
    launch_count += 1
    if rc != 0:
        raise RuntimeError(f"{fn_name} failed: {lib.romab200_last_error().decode()}")


def prologue_tiles(radius: int, h: int, w: int) -> int:
    """Tiles per map of the tile-cooperative refiner prologue (`tile_done` bytes per decoder item; include/romab200.h)."""
    ty = 2 if radius == 7 else 4
    return ((h + ty - 1) // ty) * ((w + 7) // 8)


def kernel_launches() -> int:
    """Kernels launched by libromab200 in this process so far."""
    return int(load_library().romab200_launch_count())


def device_ok() -> bool:
    return bool(load_library().romab200_device_ok())
