"""Helpers shared by the test modules: the float64 launch checks' bounds and recorders, their inputs, the per-feature
references and comparators, and the host-emulation build.  Pytest does not collect this package."""
import contextlib
import pkgutil

import pytest
import torch

# the submodules, not the package itself: it is already being imported here, and it asserts nothing
pytest.register_assert_rewrite(*(f"{__name__}.{m.name}" for m in pkgutil.iter_modules(__path__)))


@contextlib.contextmanager
def tf32(enabled):
    """Lets cuDNN convolutions and cuBLAS matmuls use TF32 (or not) inside the block; restores both settings on exit."""
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = enabled
    try:
        yield
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev


@pytest.fixture
def fp64_references():
    """Runs the test with TF32 off, so that fp32 cuDNN / cuBLAS references round like fp32 (TF32 errs by ~1e-3)."""
    with tf32(False):
        yield
