import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _have_gpu() -> bool:
    try:
        import torch

        return bool(torch.cuda.is_available())
    except Exception:
        return os.path.exists("/dev/nvidia0")


def pytest_collection_modifyitems(config, items):
    """A plain `pytest tests` on a box without a CUDA device skips the gpu-marked tests.  With `-m gpu` (the H100 run) or
    FASTLLAMA_B200_STRICT_GPU=1 nothing is skipped: a missing device or library must FAIL there, never pass silently."""
    strict = os.environ.get("FASTLLAMA_B200_STRICT_GPU") == "1" or "gpu" in (config.getoption("-m") or "").replace("not gpu", "")
    if strict or _have_gpu():
        return
    skip = pytest.mark.skip(reason="no CUDA device (gpu tests run on an H100; set FASTLLAMA_B200_STRICT_GPU=1 to force)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    from oracle.pyoracle import Oracle, build_oracle

    build_oracle()
    return Oracle()


@pytest.fixture(scope="session")
def ref():
    """The reference's own lib/ggml.c (oracle/_ref), where it was built."""
    from oracle.pyoracle import RefGgml, build_oracle, have_ref

    build_oracle()
    if not have_ref():
        pytest.skip("oracle/_ref not built (no /root/reference at build time)")
    return RefGgml()


GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="session", params=[64, 256, 4096])
def golden_rowfns(request):
    import numpy as np

    return request.param, np.load(os.path.join(GOLDEN, f"rowfns_k{request.param}.npz"))
