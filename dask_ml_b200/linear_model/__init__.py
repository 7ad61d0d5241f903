"""Generalised linear models (dask_ml/linear_model/__init__.py): LogisticRegression, LinearRegression and
PoissonRegression."""
from .glm import LinearRegression, LogisticRegression, PoissonRegression  # noqa: F401
