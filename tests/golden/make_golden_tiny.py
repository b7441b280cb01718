"""Generate the TinyRoMa golden fixtures (`tiny_*.npz`) FROM THE UNMODIFIED REFERENCE.

    PYTHONPATH=<reference tree> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_tiny.py

The reference's `tiny_roma_v1_model(weights, xfeat=...)` (roma_models.py:21-29) is built on CPU (fp32) around the stand-in
backbone `roma_b200.synthetic.xfeat_standin()` with the seeded checkpoint `synthetic.make_tiny_weights(0, xfeat)`, which loads
strictly, and run through `match()` on seeded uniform [0, 1) tensors / seeded PIL images.  Stage tensors are captured by wrapping the
model instance's own `forward_single`, `pos_embed` and `forward` (the reference source is not modified).

Seed rule: every fixture stores `gap`, the per-pixel difference between the best and the second-best correlation score of the
coarse match.  Starting from the seed given below, the first seed whose minimum gap is >= 1e-4 is used (and stored in `meta`), so
that an argmax decided by the summation order of a 64-term dot product cannot decide a test.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from roma_b200 import synthetic  # noqa: E402
from romatch.models.model_zoo.roma_models import tiny_roma_v1_model  # noqa: E402  (the reference)

MIN_GAP = 1e-4
# (channel step, pixel step) of the stored stage tensors x[:, ::cs, ::ss, ::ss]; stored beside each as `<key>__step`
STAGE_STEPS = {"x2": (4, 2), "feats": (8, 2), "pos_embed": (1, 1), "corresps8": (1, 1), "corresps4": (1, 1)}


def checksum(t):
    t = t.double()
    return np.array([t.sum().item(), t.abs().sum().item(), (t * t).sum().item()])


def images(seed, shape0, shape1):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(*shape0, generator=g), torch.rand(*shape1, generator=g)


def model(exact=False):
    xf = synthetic.xfeat_standin()
    m = tiny_roma_v1_model(weights=synthetic.make_tiny_weights(0, synthetic.xfeat_standin()), xfeat=xf, exact_softmax=exact)
    trace = {}
    fs, pe, fw = m.forward_single, m.pos_embed, m.forward

    def forward_single(x):
        out = fs(x)
        trace.setdefault("x2", []).append(out[0])
        trace.setdefault("feats", []).append(out[1])
        return out

    def pos_embed(cv):
        B, H1, W1, H0, W0 = cv.shape
        top2 = cv.reshape(B, H1 * W1, H0, W0).topk(2, dim=1).values
        trace["gap"] = (top2[:, 0] - top2[:, 1])
        out = pe(cv)
        trace["pos_embed"] = out
        return out

    def forward(batch):
        out = fw(batch)
        trace["corresps8"] = torch.cat((out[8]["flow"], out[8]["certainty"]), 1)
        trace["corresps4"] = torch.cat((out[4]["flow"], out[4]["certainty"]), 1)
        return out
    m.forward_single, m.pos_embed, m.forward = forward_single, pos_embed, forward
    return m, trace


def run(name, shape0, shape1, seed, exact=False, step=1, stages=False, pil=False):
    while True:
        m, trace = model(exact)
        if pil:
            a, b = synthetic.make_pil_pair(seed)
            warp, cert = m.match(a, b)
            warp, cert = warp[None], cert[None]
        else:
            A, B = images(seed, shape0, shape1)
            warp, cert = m.match(A, B)
        if trace["gap"].min().item() >= MIN_GAP:
            break
        print(name, "seed", seed, "min gap", trace["gap"].min().item(), "-> next seed")
        seed += 1
    out = dict(warp=warp[:, ::step, ::step].numpy(), certainty=cert[:, ::step, ::step].numpy(), warp_checksum=checksum(warp),
               certainty_checksum=checksum(cert), gap=trace["gap"].numpy(),
               meta=np.array([seed, int(exact), step, int(pil)]))
    if not pil:
        out["shape0"], out["shape1"] = np.array(shape0), np.array(shape1)
    np.savez_compressed(os.path.join(HERE, f"{name}.npz"), **out)
    if stages:
        st = {"x2": torch.cat(trace["x2"]), "feats": torch.cat(trace["feats"]), "pos_embed": trace["pos_embed"],
              "corresps8": trace["corresps8"], "corresps4": trace["corresps4"]}
        arrs = {}
        for k, v in st.items():
            cs, ss = STAGE_STEPS[k]
            arrs[k], arrs[k + "__step"] = np.ascontiguousarray(v[:, ::cs, ::ss, ::ss].numpy()), np.array([cs, ss])
        np.savez_compressed(os.path.join(HERE, f"{name}_stages.npz"), **arrs)
    print(name, "seed", seed, {k: v.shape for k, v in out.items()}, "min gap", out["gap"].min())


if __name__ == "__main__":
    torch.set_num_threads(8)
    only = set(sys.argv[1:])
    jobs = [
        ("tiny_b2", (2, 3, 256, 320), (2, 3, 256, 320), 1, dict(stages=True, step=2)),
        ("tiny_unequal", (1, 3, 250, 330), (1, 3, 200, 290), 2, dict(step=2)),
        ("tiny_exact", (1, 3, 256, 320), (1, 3, 256, 320), 3, dict(exact=True, step=2)),
        ("tiny_pil", None, None, 3, dict(pil=True)),
        ("tiny_full", (1, 3, 560, 560), (1, 3, 560, 560), 4, dict(step=8)),
    ]
    for name, s0, s1, seed, kw in jobs:
        if not only or name in only:
            run(name, s0, s1, seed, **kw)
