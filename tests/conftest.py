import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


def usable_cores():
    """Cores this process may really use: affinity capped by the cgroup quota (os.cpu_count() reports the host's cores in a
    container, and oversubscribed OpenMP loops crawl)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(float(q) / float(per) + 0.5)))
    except Exception:
        pass
    return max(1, n)


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.lib()
    # small test images: a few threads beat 64 (OpenMP fork/join per row loop)
    pyoracle.lib().orc_set_num_threads(min(8, usable_cores()))
    pyoracle.usable_cores = usable_cores
    return pyoracle


@pytest.fixture(scope="session")
def pair256():
    from denseflow_b200 import synth
    return synth.pair(256, 256, 0)
