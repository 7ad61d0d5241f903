import os
import sys

import pytest

# scikit-learn's OpenMP reductions (the oracle's E-step) on a 100+-thread GPU host next to CUDA contexts: one test order
# segfaulted inside sklearn's ArgKmin with the default (all cores) thread count; a bounded pool is plenty for the
# oracle's small cases.  Must be set before numpy / scikit-learn are imported.
os.environ.setdefault("OMP_NUM_THREADS", "16")
os.environ.setdefault("OPENBLAS_NUM_THREADS", "16")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device: skip (instead of erroring in the backend fixture) where there is none."""
    try:
        import torch

        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (H100)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session")
def oracle():
    """The CPU oracle (test infrastructure); builds its C half on first use."""
    import subprocess

    so = os.path.join(ROOT, "oracle", "liboracle_c.so")
    if not os.path.exists(so):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")])
    from oracle import kmeans_oracle

    return kmeans_oracle
