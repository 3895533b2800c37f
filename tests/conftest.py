import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a GPU machine)")


@pytest.fixture(scope="session")
def cuda():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda:0")


@pytest.fixture(scope="session")
def record():
    """Parity numbers worth quoting (DESIGN.md §4) are appended to gpurun_out/parity_numbers.txt when that directory
    exists (GPU box runs); a no-op elsewhere."""
    path = os.path.join(ROOT, "gpurun_out", "parity_numbers.txt")

    def rec(line):
        print(line)
        if os.path.isdir(os.path.dirname(path)):
            with open(path, "a") as f:
                f.write(line + "\n")
    return rec
