import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100)")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a host without a GPU skips the gpu-marked tests instead of failing in Engine(0)."""
    try:
        import torch
        have = torch.cuda.is_available()
    except Exception:
        have = False
    if have:
        return
    skip = pytest.mark.skip(reason="no CUDA device (gpu-marked test)")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def params():
    from dc_tts_b200.params import init_params
    return init_params(0, "perturbed")


@pytest.fixture(scope="session")
def engine(params):
    """One engine per test session with the 'perturbed' seed-0 weights committed."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from dc_tts_b200.engine import Engine, set_engine
    e = Engine(0)
    e.load_params(params)
    set_engine(e)
    return e


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


# (tensor_path, decode_mode): fp32 CUDA-core blocks + graph-per-frame decode; wgmma blocks + graph-per-frame decode;
# the product default: wgmma blocks + the persistent cluster decode kernel
KERNEL_SETS = {"fp32path": (0, 0), "tensorpath": (1, 0), "cluster": (1, 1)}


@pytest.fixture(params=list(KERNEL_SETS), ids=list(KERNEL_SETS))
def path(engine, request):
    """Runs a GPU test once per kernel set (include/dctts.h: dctts_set_tensor_path, dctts_set_option "decode_mode")."""
    tp, dm = KERNEL_SETS[request.param]
    engine.set_tensor_path(tp)
    engine.set_option("decode_mode", dm)
    yield request.param
    engine.set_tensor_path(1)
    engine.set_option("decode_mode", 1)
