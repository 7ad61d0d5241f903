"""Unsupervised clustering (dask_ml/cluster/__init__.py:3-5): KMeans, PartialMiniBatchKMeans and SpectralClustering.

Like the reference, the estimators are re-exported; ``dask_ml_b200.cluster.k_means`` is the module
(the reference's tests call ``k_means.k_init`` on it, tests/test_kmeans.py:136-147)."""
from .k_means import KMeans  # noqa: F401
from .minibatch import PartialMiniBatchKMeans  # noqa: F401
from .spectral import SpectralClustering  # noqa: F401
from . import k_means  # noqa: F401
