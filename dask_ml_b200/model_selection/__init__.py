"""Block-wise splitting of row-chunked arrays (dask_ml/model_selection/_split.py:24-465) and the hyper-parameter
searches over them (_search.py, methods.py)."""
from ._search import GridSearchCV, RandomizedSearchCV, check_cv, compute_n_splits  # noqa: F401
from ._split import KFold, ShuffleSplit, train_test_split  # noqa: F401
