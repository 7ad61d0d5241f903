"""Worker of tests/test_distributed_search_cpu.py: one rank of a gloo group cutting its own host blocks into KFold
pieces and scoring a split of them."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ([40, 25, 31], [17, 50])          # the row blocks of rank 0 and rank 1
K = 5


def data():
    rng = np.random.RandomState(5)
    n = sum(SIZES[0]) + sum(SIZES[1])
    X = rng.standard_normal((n, 3))
    return X, (X[:, 0] + 0.3 * rng.standard_normal(n) > 0).astype(np.int64)


class SignOfFirstColumn(object):
    """A fitted classifier that needs no fit: predict is ``X[:, 0] > 0`` per block, so a 0-row block predicts 0 rows."""

    def predict(self, X):
        from dask_ml_b200 import ChunkedArray

        return ChunkedArray([(np.asarray(b)[:, 0] > 0).astype(np.int64) for b in X.blocks])


def worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.metrics import SCORERS
        from dask_ml_b200.model_selection import KFold
        from dask_ml_b200.model_selection._search import _splits

        X, y = data()
        lo = 0 if rank == 0 else sum(SIZES[0])
        hi = lo + sum(SIZES[rank])
        X, y = [ChunkedArray.from_array(a[lo:hi], (tuple(SIZES[rank]),)) for a in (X, y)]
        out = {}
        for shuffle in (False, True):
            folds = KFold(K, shuffle=shuffle, random_state=4).split(X)
            for f, (tr, te) in enumerate(folds):
                for part, idx in (("train", tr), ("test", te)):
                    out["%d_%d_%s" % (shuffle, f, part)] = idx.compute() + lo       # rank-local -> global
                    out["%d_%d_%s_chunks" % (shuffle, f, part)] = np.array(idx.chunks[0])
        scores = []
        for f, (X_tr, y_tr, X_te, y_te) in enumerate(_splits(KFold(K), X, y, None)):
            out["views_%d_test_chunks" % f] = np.array(X_te.chunks[0])
            out["views_%d_test" % f] = X_te.compute()
            scores.append(SCORERS["accuracy"](SignOfFirstColumn(), X_te, y_te))
        out["scores"] = np.array(scores)
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), **out)
    finally:
        dist.destroy_process_group()
