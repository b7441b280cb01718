"""Golden DINOv2 tokens for the retrieval descriptor, FROM THE UNMODIFIED REFERENCE (`DinoVisionTransformer.forward_features`,
romatch/models/transformer/dinov2.py:222-238, built as in `CNNandDinov2`, romatch/models/encoders.py:29-50), on the CPU in fp32.

Run where the reference is importable (it is not needed by any test):

    PYTHONPATH=<reference tree> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_retrieval.py

The ViT-L/14 gets the seeded synthetic DINOv2 weights of `roma_b200.synthetic` (seed 0, strict load) and one seeded N(0,1) image of
42 x 56 pixels (`synthetic.make_pair(1, (42, 56), (42, 56), seed=4)[0]`, a 3 x 4 patch grid, so the positional embedding is
resized).  retrieval_dinov2.npz holds the image and the outputs `x_norm_clstoken` [1, 1024] and `x_norm_patchtokens` [1, 12, 1024]:
the inputs of the global descriptor (include/romab200.h, "Retrieval").
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
from romatch.models.transformer import vit_large  # noqa: E402  (the reference)

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from roma_b200 import synthetic  # noqa: E402


def main():
    _, dw = synthetic.make_weights(0)
    vit = vit_large(img_size=518, patch_size=14, init_values=1.0, ffn_layer="mlp", block_chunks=0).eval()
    vit.load_state_dict(dw, strict=True)
    image = synthetic.make_pair(1, (42, 56), (42, 56), seed=4)[0]
    with torch.no_grad():
        out = vit.forward_features(image)
    np.savez_compressed(os.path.join(HERE, "retrieval_dinov2.npz"), image=image.numpy(),
                        x_norm_clstoken=out["x_norm_clstoken"].numpy(), x_norm_patchtokens=out["x_norm_patchtokens"].numpy())


if __name__ == "__main__":
    main()
