"""Times one ``partial_fit`` block of the SGD family on the device against scikit-learn's ``partial_fit`` on the CPU for
the same block, and reports the host's row-order time separately.

    python tests/sgd_bench.py [--rows N] [--out FILE]

Workloads: N x 64 binary hinge; N x 64 with 20 classes; hashed CSR rows (2^20 features, about 100 nonzeros per row)
with 20 classes; and a dense shape on each side of the shared-memory / global-memory selection of the weights."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time
import warnings

import numpy as np
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sklearn import linear_model as sklm  # noqa: E402

from dask_ml_b200 import _lib  # noqa: E402
from dask_ml_b200.linear_model import PartialSGDClassifier  # noqa: E402

warnings.simplefilter("ignore")


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                     text=True).strip().splitlines()[0]
    except Exception:
        pl = "unknown"
    return name, pl


def _dense(n, d, k, seed):
    rng = np.random.RandomState(seed)
    return rng.standard_normal((n, d)), rng.randint(0, k, size=n)


def _hashed(n, nnz, k, seed):
    rng = np.random.RandomState(seed)
    cols = np.sort(np.stack([rng.choice(1 << 20, nnz, replace=False) for _ in range(min(n, 64))]), axis=1)
    cols = cols[np.arange(n) % cols.shape[0]]
    vals = rng.standard_normal((n, nnz)) / np.sqrt(nnz)
    A = sp.csr_matrix((vals.ravel(), cols.ravel(), np.arange(0, n * nnz + 1, nnz)), shape=(n, 1 << 20))
    return A, rng.randint(0, k, size=n)


def _time_device(X, y, k):
    est = PartialSGDClassifier(classes=np.arange(k), random_state=0)
    Xd = torch.from_numpy(X).cuda() if isinstance(X, np.ndarray) else X
    yd = torch.from_numpy(y).cuda()
    est.partial_fit(Xd, yd, classes=np.arange(k))          # first call: allocation and module load
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    est.partial_fit(Xd, yd)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, est


def _time_cpu(X, y, k):
    ref = sklm.SGDClassifier(random_state=0)
    ref.partial_fit(X, y, classes=np.arange(k))
    t0 = time.perf_counter()
    ref.partial_fit(X, y)
    return time.perf_counter() - t0, ref


def _order_time(n, P):
    lib = _lib.load()
    out = np.empty(n, dtype=np.int32)
    t0 = time.perf_counter()
    for s in range(P):
        lib.bkm_sgd_order(n, s + 1, out.ctypes.data_as(ctypes.c_void_p))
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.rows
    name, pl = _card()
    results = []
    cases = [
        ("dense %dx64 binary hinge" % n, lambda: _dense(n, 64, 2, 0), 2),
        ("dense %dx64 20 classes" % n, lambda: _dense(n, 64, 20, 1), 20),
        ("hashed CSR %dx2^20, 100 nnz/row, 20 classes" % (n // 4), lambda: _hashed(n // 4, 100, 20, 2), 20),
        ("dense %dx20000 binary (weights in shared memory)" % (n // 64), lambda: _dense(n // 64, 20000, 2, 3), 2),
        ("dense %dx30000 binary (weights in global memory)" % (n // 64), lambda: _dense(n // 64, 30000, 2, 4), 2),
    ]
    for label, make, k in cases:
        X, y = make()
        Xg = X if isinstance(X, np.ndarray) else torch.sparse_csr_tensor(
            torch.from_numpy(X.indptr.astype(np.int64)), torch.from_numpy(X.indices.astype(np.int64)),
            torch.from_numpy(X.data), size=X.shape).cuda()
        t_dev, est = _time_device(Xg, y, k)
        t_cpu, ref = _time_cpu(X, y, k)
        P = 1 if k == 2 else k
        rec = {"workload": label, "device_s": round(t_dev, 4), "sklearn_cpu_s": round(t_cpu, 4),
               "host_order_s": round(_order_time(X.shape[0], P), 4),
               "bit_identical": bool(np.array_equal(est.coef_, ref.coef_))}
        print(json.dumps(rec), flush=True)
        results.append(rec)
    summary = {"card": name, "power_limit": pl, "results": results}
    print(json.dumps({"card": name, "power_limit": pl}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
