"""dask_ml_b200 — a Hopper (H100, sm_90a) native engine for the dask_ml.cluster.KMeans hot path.

Same estimator API as ``dask_ml.cluster.KMeans`` (dask_ml/cluster/k_means.py:26-233); every
Lloyd iteration runs as hand-written CUDA behind the C ABI in ``include/bkm_b200.h``.
"""
from .chunked import ChunkedArray  # noqa: F401

__version__ = "0.1.0"
