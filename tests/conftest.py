import os
import sys
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "deep-prove_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


@pytest.fixture(scope="session", autouse=True)
def _built():
    """Build the in-tree libraries once if they are missing (nvcc cross-compiles without a GPU)."""
    need = [os.path.join(ROOT, "deep-prove_b200", "libdeepprove_b200.so"),
            os.path.join(ROOT, "deep-prove_b200", "libdeepprove_host.so"),
            os.path.join(ROOT, "oracle", "libdp_oracle.so")]
    if not all(os.path.exists(p) for p in need):
        import __graft_entry__
        __graft_entry__.build()


@pytest.fixture(scope="session")
def gpu():
    import dpb200
    if dpb200.device_count() <= 0:
        pytest.fail("marked gpu but no CUDA device is visible (no CPU fallback exists)")
    dpb200.init(0)
    return dpb200
