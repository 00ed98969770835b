import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# The oracle parallelises over <= 32 row blocks per GEMM: on a many-core GPU host more OpenMP threads only add
# contention (measured: 128 threads are ~10x slower than 32), and the strict parity tests run it at batch 64 / 256.
os.environ.setdefault("OMP_NUM_THREADS", str(max(1, min(32, os.cpu_count() or 1))))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90a); select with -m gpu")
