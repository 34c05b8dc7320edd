import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with `-m gpu`)")


def _has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def pytest_collection_modifyitems(config, items):
    if _has_cuda():
        return
    skip = pytest.mark.skip(reason="no CUDA device in this container")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def stages():
    return np.load(os.path.join(GOLDEN, "stages.npz"))


@pytest.fixture(scope="session")
def oracle():
    from oracle import dsp_oracle
    return dsp_oracle


@pytest.fixture(scope="session")
def oracle_decoders(oracle):
    return {n: oracle.DecoderWeights.from_npz(os.path.join(GOLDEN, f"decoder_{n}.npz")) for n in ("cars", "chairs")}


@pytest.fixture(scope="session")
def cfg_kitti():
    return json.load(open(os.path.join(ROOT, "dsp_slam_b200", "configs", "config_kitti.json")))


@pytest.fixture(scope="session")
def cfg_redwood():
    return json.load(open(os.path.join(ROOT, "dsp_slam_b200", "configs", "config_redwood_01053.json")))


@pytest.fixture(scope="session", autouse=True)
def _build_lib():
    """The in-tree CUDA library must exist for both the CPU (symbol) and GPU tests."""
    import __graft_entry__ as g
    if not os.path.isfile(g.LIB):
        g.build()
