import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    try:                                   # references must be true fp32 (cuDNN/cuBLAS default to TF32 for convs)
        import torch
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    except Exception:
        pass
    config.addinivalue_line("markers", "gpu: needs a CUDA device, an H100 (run with -m gpu)")
    config.addinivalue_line("markers", "slow: takes more than ~30 s on 8 CPU cores")


@pytest.fixture(scope="session")
def weights():
    """Seeded synthetic weights (seed 0) in the reference's state-dict layout."""
    from roma_b200 import synthetic
    return synthetic.make_weights(0)


def load_golden(name):
    import numpy as np
    path = os.path.join(ROOT, "tests", "golden", f"{name}.npz")
    return dict(np.load(path))
