import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "dinov3-jax_b200"), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) GPU; run with -m gpu on a GPU machine")


@pytest.fixture(scope="session")
def native():
    """The C-ABI library bound to cuda:0 — GPU tests fail loudly (no fallback) when it is missing."""
    import torch
    from dinov3_jax import _native
    assert torch.cuda.is_available(), "GPU test selected without a GPU"
    _native.init(0)
    return _native


GOLDEN = os.path.join(ROOT, "tests", "golden")


def reference_vectors():
    """The golden vectors of tests/golden/make_golden.py as one dict (stored in parts of under 1 MB each)."""
    import glob

    import numpy as np
    out = {}
    for p in sorted(glob.glob(os.path.join(GOLDEN, "reference_vectors_*.npz"))):
        with np.load(p) as z:
            out.update({k: z[k] for k in z.files})
    return out
