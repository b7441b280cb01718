"""Host side of `match_keypoints`: which inputs go to the device kernels, and the exact-difference distance those kernels use
checked against the reference's golden matches on the CPU."""
import os

import numpy as np
import torch
import torch.nn.functional as F

from roma_b200 import cabi
from roma_b200.matcher import RegressionMatcher, _keypoints_on_device

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "helpers.npz"))


def _golden_inputs():
    W = G["warp"].shape[1] // 2
    return (torch.from_numpy(G["x_A"]), torch.from_numpy(G["x_B"]), torch.from_numpy(G["warp"])[:, :W],
            torch.from_numpy(G["certainty"])[:, :W])


def test_cpu_tensors_never_reach_the_c_abi(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("CPU tensors must not reach the C ABI")
    monkeypatch.setattr(cabi, "call", refuse)
    x_A, x_B, warp, cert = _golden_inputs()
    assert not _keypoints_on_device(x_A, x_B, warp, cert)
    m = RegressionMatcher.__new__(RegressionMatcher)
    ia, ib = m.match_keypoints(x_A, x_B, warp, cert, return_inds=True, max_dist=0.005, cert_th=0.2)
    assert torch.equal(ia, torch.from_numpy(G["kp_inds_A"])) and torch.equal(ib, torch.from_numpy(G["kp_inds_B"]))


def test_exact_difference_distance_reproduces_the_golden_matches():
    """The device path's distance, sqrt(dx*dx + dy*dy) with every operation in float32, selects exactly the pairs the reference's
    cdist statement selected on these vectors."""
    x_A, x_B, warp, cert = _golden_inputs()
    a = F.grid_sample(warp[..., -2:].permute(2, 0, 1)[None], x_A[None, None], align_corners=False)[0, :, 0].mT.numpy()
    c = F.grid_sample(cert[None, None], x_A[None, None], align_corners=False)[0, 0, 0].numpy()
    b = x_B.numpy()
    dx = a[:, None, 0] - b[None, :, 0]
    dy = a[:, None, 1] - b[None, :, 1]
    D = np.sqrt(dx * dx + dy * dy)
    assert D.dtype == np.float32
    mask = (D == D.min(axis=1, keepdims=True)) & (D == D.min(axis=0, keepdims=True)) & (c[:, None] > np.float32(0.2)) & (D < np.float32(0.005))
    ia, ib = np.nonzero(mask)
    assert np.array_equal(ia, G["kp_inds_A"]) and np.array_equal(ib, G["kp_inds_B"])
