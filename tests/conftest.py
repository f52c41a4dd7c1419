import os
import sys

# CPU test sessions share a small, quota-limited VM with their own worker subprocesses (2-rank gloo tests).  GNU OpenMP's
# default spin-waiting then turns any vCPU descheduling into a collapse: measured here, the same 20 conv fwd+bwd steps
# take 70 ms or 3,500 ms (and a 4 s trainer test 300 s) depending on what ran before, with 8 spinning threads per process
# burning the VM's CPU allowance.  Passive waiting and a modest team size keep the suite's run time bounded.  These must be
# set before torch (libgomp) is loaded; `setdefault` leaves explicit user settings alone; worker subprocesses inherit them.
os.environ.setdefault("OMP_WAIT_POLICY", "PASSIVE")
os.environ.setdefault("GOMP_SPINCOUNT", "0")
os.environ.setdefault("OMP_NUM_THREADS", "4")
os.environ.setdefault("MKL_NUM_THREADS", "4")

import pytest  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (H100); run with `pytest -m gpu` on the GPU box")


def pytest_collection_modifyitems(config, items):
    import torch

    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device on this box")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
