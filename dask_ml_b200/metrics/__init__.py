"""Distance operators on the KMeans path (dask_ml/metrics/pairwise.py:18-97), the kernel built on them (:131-139), and
the scoring metrics (dask_ml/metrics/classification.py, regression.py) and their scorers (scorer.py)."""
from .classification import accuracy_score, log_loss  # noqa: F401
from .pairwise import (  # noqa: F401
    euclidean_distances,
    pairwise_distances,
    pairwise_distances_argmin_min,
    pairwise_kernels,
    rbf_kernel,
)
from .regression import mean_absolute_error, mean_squared_error, r2_score  # noqa: F401
from .scorer import SCORERS, check_scoring, get_scorer  # noqa: F401
