import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _usable_cpus():
    """affinity capped by the cgroup CPU quota: the reference oracle (OpenMP) must not run 128 threads on a 16-CPU lease"""
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        n = os.cpu_count() or 1
    try:
        a, b = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if a != "max":
            n = max(1, min(n, int(float(a) / float(b) + 0.5)))
    except Exception:
        pass
    return n


os.environ.setdefault("OMP_NUM_THREADS", str(_usable_cpus()))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def ref():
    """compiled reference oracle (oracle/_ref); parity tests skip loudly if it did not travel"""
    from oracle import ref as r
    if not r.available():
        pytest.skip("oracle/_ref/libknowhere_ref.so not built")
    return r


@pytest.fixture(scope="session")
def kb():
    import knowhere_b200
    return knowhere_b200
