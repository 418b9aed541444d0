import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# Test infrastructure: tests/test_ingest_pipeline_cpu.py re-runs the GPU reader tests in a SUBPROCESS against the mock
# library of tests/mock_cuda (the C++ host side built against a host-memory stand-in for the CUDA runtime, CPU stand-ins
# for the cvk_* launchers), so the ingest pipeline's host logic is exercised on machines without a GPU.  Only that
# subprocess sets this variable; the product (curvine_b200/) has no knob that loads anything but its own library.
MOCK_LIB = os.environ.get("CV_TEST_MOCK_CUDA_LIB", "")
if MOCK_LIB:
    from curvine_b200 import _lib as _cv_lib
    _cv_lib.LIB_PATH = MOCK_LIB


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def cuda():
    import torch
    if MOCK_LIB:  # "device memory" is host memory here: CPU tensors, no streams to wait for
        import types
        from curvine_b200 import _lib

        def device_sync(*a, **k):  # the stand-in runtime can run its streams asynchronously (MOCK_CUDA_ASYNC=1): wait for them like the real call
            _lib.lib().cudaDeviceSynchronize()
        torch.cuda.synchronize = device_sync
        torch.cuda.current_stream = lambda *a, **k: types.SimpleNamespace(cuda_stream=0, synchronize=device_sync)
        torch.cuda.current_device = lambda: 0
        return torch.device("cpu")
    if not torch.cuda.is_available():
        pytest.fail("this test is marked gpu but no CUDA device is visible")
    torch.cuda.set_device(0)
    from curvine_b200 import _lib
    _lib.check(_lib.lib().cvk_init(0), "cvk_init")
    return torch.device("cuda:0")
