import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")
    config.addinivalue_line("markers", "gpu_unverified: GPU test of a kernel that has not run on an H100 yet (skipped without a "
                                       "GPU; NOT selected by -m gpu; run with -m gpu_unverified, then re-mark as gpu)")


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def spec():
    from spann3r_b200 import synth
    return synth.load_spec()


_SD_CACHE = {}


def get_state_dict(sharpen: bool):
    """Synthetic checkpoint (CPU fp32), cached per session."""
    from spann3r_b200 import synth
    if sharpen not in _SD_CACHE:
        _SD_CACHE[sharpen] = synth.make_state_dict(seed=0, sharpen=sharpen)
    return _SD_CACHE[sharpen]


def rel_l2(a, b):
    import torch
    a = torch.as_tensor(a).double()
    b = torch.as_tensor(b).double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))
