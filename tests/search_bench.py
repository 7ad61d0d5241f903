"""Speed of a hyper-parameter search on one GPU (run on an H100: python tests/search_bench.py [--out FILE]).

``GridSearchCV(LogisticRegression(solver="lbfgs"), 8 values of C, cv=5)`` on 2^22 x 64 fp32 rows in blocks of 2^20 on
the device, against scikit-learn's ``GridSearchCV(cv=KFold(5))`` driving the same estimator on the host copy of the
rows (which indexes numpy, so every fold is copied on the host and uploaded again for every candidate).  Wall-clock
times of whole ``fit`` calls ending in a device synchronise, after one warm-up search on a small problem; the two are
alternated in the same process, and their per-split test scores are compared.  The card's name and power limit come
from the same run.  Fails without a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sklearn.model_selection as skms  # noqa: E402

from dask_ml_b200.datasets import make_classification  # noqa: E402
from dask_ml_b200.linear_model import LogisticRegression  # noqa: E402
from dask_ml_b200.model_selection import GridSearchCV  # noqa: E402
from nb_bench import _card  # noqa: E402

CS = list(np.logspace(-3, 2, 8))


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def _scores(cv_results, k):
    return np.stack([cv_results["split%d_test_score" % i] for i in range(k)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log2-rows", type=int, default=22)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("search_bench needs a CUDA device")

    est = LogisticRegression(solver="lbfgs")
    Xw, yw = make_classification(1 << 16, 64, chunks=1 << 14, device="cuda", dtype="float32", random_state=1)
    GridSearchCV(est, {"C": CS[:2]}, cv=5).fit(Xw, yw)                               # load modules, warm the passes
    skms.GridSearchCV(est, {"C": CS[:2]}, cv=skms.KFold(5)).fit(Xw.compute(), yw.compute())

    n = 1 << args.log2_rows
    X, y = make_classification(n, 64, chunks=1 << 20, device="cuda", dtype="float32", random_state=0)
    Xh, yh = X.compute(), y.compute()
    ours_t, theirs_t = [], []
    for _ in range(args.reps):
        t, ours = _timed(lambda: GridSearchCV(est, {"C": CS}, cv=5).fit(X, y))
        ours_t.append(t)
        t, theirs = _timed(lambda: skms.GridSearchCV(est, {"C": CS}, cv=skms.KFold(5)).fit(Xh, yh))
        theirs_t.append(t)
    diff = np.abs(_scores(ours.cv_results_, 5) - _scores(theirs.cv_results_, 5)).max()
    res = dict(card=_card(), rows=n, features=64, dtype="float32", candidates=len(CS), folds=5,
               device_search_s=min(ours_t), sklearn_search_s=min(theirs_t),
               speedup=min(theirs_t) / min(ours_t), all_device_s=ours_t, all_sklearn_s=theirs_t,
               max_split_score_diff=float(diff), best_C=float(ours.best_params_["C"]),
               sklearn_best_C=float(theirs.best_params_["C"]),
               mean_fit_s=float(ours.cv_results_["mean_fit_time"].mean()),
               mean_score_s=float(ours.cv_results_["mean_score_time"].mean()))
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
