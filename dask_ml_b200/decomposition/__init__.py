"""Matrix decomposition (dask_ml/decomposition/__init__.py): PCA and TruncatedSVD."""
from .pca import PCA  # noqa: F401
from .truncated_svd import TruncatedSVD  # noqa: F401
