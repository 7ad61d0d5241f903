"""Block-wise splitting of row-chunked arrays (dask_ml/model_selection/_split.py:24-202, 321-465)."""
from ._split import ShuffleSplit, train_test_split  # noqa: F401
