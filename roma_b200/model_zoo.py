"""Model factories with the reference's signatures (`romatch/models/model_zoo/__init__.py:18-94`,
`roma_models.py:32-205`).

`roma_outdoor` / `roma_indoor` build the same graph (only the checkpoint URL differs in the reference).
Weights are state dicts in the reference's key layout; with `weights=None` the reference downloads them
via `torch.hub` and so does this factory (there is no bundled checkpoint).  `amp_dtype` selects the
arithmetic regime exactly as on the reference's CUDA path: float16 (default) / bfloat16 = 16-bit tensor-core
operands with fp32 accumulation, float32 = the fp32 parity mode (fp32-class GEMMs on the tensor cores from split-fp16
operand pairs; `fp32_backend` below selects the CUDA-core cross-check instead).
"""
from __future__ import annotations

from typing import Union

import torch

from .engine import Engine
from .matcher import RegressionMatcher

weight_urls = {
    "romatch": {
        "outdoor": "https://github.com/Parskatt/storage/releases/download/roma/roma_outdoor.pth",
        "indoor": "https://github.com/Parskatt/storage/releases/download/roma/roma_indoor.pth",
    },
    "tiny_roma_v1": {
        "outdoor": "https://github.com/Parskatt/storage/releases/download/roma/tiny_roma_v1_outdoor.pth",
    },
    "dinov2": "https://dl.fbaipublicfiles.com/dinov2/dinov2_vitl14/dinov2_vitl14_pretrain.pth",
}

_PRECISION = {torch.float16: "fp16", torch.bfloat16: "bf16", torch.float32: "fp32"}
# GEMM back-end of the amp_dtype=float32 parity mode: "tcgen05" (default; the name of the tensor-core back-end, wgmma on
# sm_90a) = split-fp16 operand pairs on the tensor cores
# (fp32-class results); "simt" = CUDA-core FFMA GEMMs, kept as the slow cross-check.  Also settable with the environment
# variable ROMA_B200_FP32_BACKEND (the factories keep the reference's signatures, so this is not a keyword argument).
fp32_backend = None


def roma_model(resolution, upsample_preds, device=None, weights=None, dinov2_weights=None,
               amp_dtype: torch.dtype = torch.float16, use_custom_corr=True, symmetric=True, upsample_res=None,
               sample_thresh=0.05, sample_mode="threshold_balanced", attenuate_cert=True, **kwargs):
    """Counterpart of `roma_models.roma_model`; `use_custom_corr` is accepted and ignored — the local
    correlation is always this package's fused kernel."""
    if isinstance(resolution, int):
        resolution = (resolution, resolution)
    if isinstance(upsample_res, int):
        upsample_res = (upsample_res, upsample_res)
    assert resolution[0] % 14 == 0, "Needs to be multiple of 14 for backbone"
    assert resolution[1] % 14 == 0, "Needs to be multiple of 14 for backbone"
    if amp_dtype not in _PRECISION:
        raise ValueError(f"unsupported amp_dtype {amp_dtype}")
    precision = _PRECISION[amp_dtype]
    if precision == "fp32":
        import os
        backend = fp32_backend or os.environ.get("ROMA_B200_FP32_BACKEND", "tcgen05")
        if backend not in ("tcgen05", "simt"):
            raise ValueError(f"fp32 back-end must be 'tcgen05' or 'simt', got {backend!r}")
        precision = "fp32" if backend == "tcgen05" else "fp32_simt"
    engine = Engine(weights, dinov2_weights, device, precision=precision)
    h, w = resolution
    return RegressionMatcher(engine, h=h, w=w, upsample_preds=upsample_preds, upsample_res=upsample_res,
                             symmetric=symmetric, attenuate_cert=attenuate_cert, sample_mode=sample_mode,
                             sample_thresh=sample_thresh, **kwargs)


def _roma(kind, device, weights, dinov2_weights, coarse_res, upsample_res, amp_dtype, symmetric, use_custom_corr,
          upsample_preds):
    if weights is None:
        weights = torch.hub.load_state_dict_from_url(weight_urls["romatch"][kind], map_location="cpu")
    if dinov2_weights is None:
        dinov2_weights = torch.hub.load_state_dict_from_url(weight_urls["dinov2"], map_location="cpu")
    return roma_model(resolution=coarse_res, upsample_preds=upsample_preds, weights=weights,
                      dinov2_weights=dinov2_weights, device=device, amp_dtype=amp_dtype, symmetric=symmetric,
                      use_custom_corr=use_custom_corr, upsample_res=upsample_res)


def roma_outdoor(device, weights=None, dinov2_weights=None, coarse_res: Union[int, tuple] = 560,
                 upsample_res: Union[int, tuple] = 864, amp_dtype: torch.dtype = torch.float16, symmetric=True,
                 use_custom_corr=True, upsample_preds=True):
    return _roma("outdoor", device, weights, dinov2_weights, coarse_res, upsample_res, amp_dtype, symmetric,
                 use_custom_corr, upsample_preds)


def roma_indoor(device, weights=None, dinov2_weights=None, coarse_res: Union[int, tuple] = 560,
                upsample_res: Union[int, tuple] = 864, amp_dtype: torch.dtype = torch.float16, symmetric=True,
                use_custom_corr=True, upsample_preds=True):
    return _roma("indoor", device, weights, dinov2_weights, coarse_res, upsample_res, amp_dtype, symmetric,
                 use_custom_corr, upsample_preds)


def tiny_roma_v1_outdoor(device, weights=None, xfeat=None):
    """TinyRoMa (`model_zoo/__init__.py:18-28`, `roma_models.py:21-29`).  Like the reference, `weights=None` downloads the
    checkpoint and `xfeat=None` loads XFeat through torch.hub ("verlab/accelerated_features"); the engine reads the backbone's
    layer structure from that module and its weights from the checkpoint's `xfeat.0.*` entries."""
    if torch.device(device).type != "cuda":
        raise RuntimeError(f"roma_b200 runs on a CUDA device only (there is no CPU fallback); got device={device!r}")
    if weights is None:
        weights = torch.hub.load_state_dict_from_url(weight_urls["tiny_roma_v1"]["outdoor"], map_location="cpu")
    if xfeat is None:
        xfeat = torch.hub.load("verlab/accelerated_features", "XFeat", pretrained=True, top_k=4096).net
    from .tiny import TinyRoMa
    return TinyRoMa(xfeat, weights, device)
