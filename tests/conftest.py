import os
import sys

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a) GPU")
    import torch
    from oracle.sta_oracle import usable_cpus
    torch.set_num_threads(usable_cpus())  # the oracle runs on the host: do not oversubscribe a cgroup-limited box


@pytest.fixture(scope="session")
def state_dict():
    """Deterministic synthetic checkpoint (oracle/sta_oracle.py::make_state_dict(0)); ~6 s, 1.75 GB."""
    from oracle.sta_oracle import make_state_dict
    return make_state_dict(0)


@pytest.fixture(scope="session")
def cuda_model(state_dict):
    import torch
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    m = STA()
    m.load_state_dict(state_dict, strict=True)
    m.eval()
    m._ready(torch.empty(1, device="cuda"))
    return m


@pytest.fixture(scope="session")
def cuda_model_x3(state_dict):
    """The same model in the split-precision parity mode (include/sta_b200.h STA_PRECISION_X3)."""
    import torch
    from vista_slam_b200.sta_model.sta_model import SymmetricTwoViewAssociation as STA
    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    m = STA(precision="x3")
    m.load_state_dict(state_dict, strict=True)
    m.eval()
    m._ready(torch.empty(1, device="cuda"))
    return m
