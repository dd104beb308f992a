import os
import sys

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if REPO not in sys.path:
    sys.path.insert(0, REPO)
GOLDEN = os.path.join(REPO, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`pytest tests` on a machine without a CUDA device (or without the built library) skips the gpu-marked tests instead of
    failing them; `-m gpu` on an H100 runs them."""
    import torch
    lib = os.path.join(REPO, "audiodec_b200", "lib", "libaudiodec_b200.so")
    reason = None
    if not torch.cuda.is_available():
        reason = "no CUDA device"
    elif not os.path.exists(lib):
        reason = "libaudiodec_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')"
    if reason:
        skip = pytest.mark.skip(reason=reason)
        for item in items:
            if "gpu" in item.keywords:
                item.add_marker(skip)


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def symad_sd():
    from audiodec_b200 import synthetic as S
    return S.symad_state_dict(seed=0)


@pytest.fixture(scope="session")
def hifigan_sd():
    from audiodec_b200 import synthetic as S
    return S.hifigan_state_dict(seed=1)


@pytest.fixture(params=["f16", "tf32", "ffma"])
def conv_path(request, monkeypatch):
    """The conv engines behind the same C ABI: wgmma with fp16-split operands (default), wgmma 3xTF32 and the CUDA-core FFMA
    kernels.  The library reads ADEC_CONV_PATH when a handle is created."""
    monkeypatch.setenv("ADEC_CONV_PATH", request.param)
    return request.param
