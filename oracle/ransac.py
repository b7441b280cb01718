"""The RANSAC pieces that the pose and homography restatements (oracle/pose_ransac.py, oracle/homography_ransac.py) share, for
the tests only: the Philox4x32-10 sample stream, the distinct-index draw and OpenCV's RANSACUpdateNumIters."""
from __future__ import annotations

import math

import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """Philox4x32-10 (Salmon et al. 2011) of counters ctr [..., 4] (uint32) under key (k0, k1); returns [..., 4] uint32."""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & M32]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return np.stack(c, axis=-1).astype(np.uint32)


def draw_distinct(m, n, seed, ctr_of):
    """m distinct indices in [0, n): the words of philox4x32_10(ctr_of(sub)) under key (seed lo, seed hi) for sub = 0, 1, ... in
    order, index (w * n) >> 32, repeats skipped.  ctr_of(sub) gives the four counter words of sub-draw `sub`."""
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    out, sub = [], 0
    while len(out) < m:
        for w in philox4x32_10(np.array(ctr_of(sub), dtype=np.uint64), key):
            v = (int(w) * n) >> 32
            if v not in out and len(out) < m:
                out.append(v)
        sub += 1
    return out


def ransac_update_num_iters(p, ep, max_iters, model_points):
    """cv::RANSACUpdateNumIters with (1 - ep)^model_points as products from the left, as the device computes it."""
    p = min(max(p, 0.0), 1.0)
    ep = min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, 2.2250738585072014e-308)
    q = 1.0 - ep
    pw = q
    for _ in range(model_points - 1):
        pw = pw * q
    denom = 1.0 - pw
    if denom < 2.2250738585072014e-308:
        return 0
    num, denom = math.log(num), math.log(denom)
    return max_iters if denom >= 0 or -num >= max_iters * (-denom) else int(np.rint(num / denom))
