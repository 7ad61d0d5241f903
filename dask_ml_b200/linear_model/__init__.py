"""Linear models (dask_ml/linear_model/__init__.py): LogisticRegression, LinearRegression and PoissonRegression, and the
block-wise SGD family PartialSGDClassifier, PartialSGDRegressor, PartialPerceptron,
PartialPassiveAggressiveClassifier and PartialPassiveAggressiveRegressor."""
from .glm import LinearRegression, LogisticRegression, PoissonRegression  # noqa: F401
from .passive_aggressive import (  # noqa: F401
    PartialPassiveAggressiveClassifier,
    PartialPassiveAggressiveRegressor,
)
from .perceptron import PartialPerceptron  # noqa: F401
from .stochastic_gradient import PartialSGDClassifier, PartialSGDRegressor  # noqa: F401
