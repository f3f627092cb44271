import importlib
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


@pytest.fixture(scope="session")
def pkg():
    """The product package (directory name starts with a digit, hence importlib)."""
    return importlib.import_module("3dssd_b200")


@pytest.fixture(scope="session")
def oracle_ops():
    from oracle import ops
    ops.build()
    return ops


@pytest.fixture(scope="session")
def cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="session")
def ref_ops(cuda):
    """Outputs of the reference's own kernels, replayed from tests/golden/ref_kernels.npz (oracle/ref_golden.py).
    With SSD3D_RECORD_REF=<path> the live kernels (oracle/_ref/libref_ops.so, `make -C oracle ref`) run instead
    and their outputs are written to <path> at the end of the session."""
    from oracle import ref_golden, ref_ops
    path = os.environ.get("SSD3D_RECORD_REF")
    if not path:
        yield ref_golden.Replay(os.path.join(ROOT, "tests", "golden", "ref_kernels.npz"))
        return
    if not ref_ops.available():
        pytest.fail("SSD3D_RECORD_REF is set but oracle/_ref/libref_ops.so is not built")
    rec = ref_golden.Recorder(ref_ops)
    yield rec
    rec.save(path)
