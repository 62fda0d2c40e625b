import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")


@pytest.fixture(scope="session")
def cuda_device():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


@pytest.fixture(scope="session", autouse=True)
def _bounded_cpu_threads():
    """The oracle runs on the host CPU.  torch defaults to one intra-op thread per visible core, which on a shared /
    cgroup-limited box (the GPU boxes) oversubscribes and makes the oracle 10-100x slower: use the cores this process
    may actually run on, at most 32, divided among xdist workers."""
    import torch

    try:
        allowed = len(os.sched_getaffinity(0))
    except (AttributeError, OSError):
        allowed = os.cpu_count() or 1
    workers = max(1, int(os.environ.get("PYTEST_XDIST_WORKER_COUNT", "1")))
    torch.set_num_threads(max(1, min(allowed, 32) // workers))
    yield
