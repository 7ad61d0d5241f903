"""Worker of tests/test_distributed_split_cpu.py: one rank of a gloo group splitting its own host blocks and scoring
its own rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = ([300, 300, 150], [400, 77])          # the row blocks of rank 0 and rank 1


def data():
    rng = np.random.RandomState(3)
    n = sum(SIZES[0]) + sum(SIZES[1])
    X = rng.standard_normal((n, 4))
    y = rng.randint(0, 3, size=n)
    pred = np.where(rng.rand(n) < 0.7, y, 0)
    proba = rng.dirichlet(np.ones(3), size=n)
    target = 50.0 + X @ np.array([1.0, -2.0, 0.5, 3.0])
    return X, y, pred, proba, target, target + 0.2 * rng.standard_normal(n)


def worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    import torch.distributed as dist

    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from dask_ml_b200 import ChunkedArray
        from dask_ml_b200.metrics import accuracy_score, log_loss, mean_squared_error, r2_score
        from dask_ml_b200.model_selection import train_test_split

        arrays = data()
        lo = 0 if rank == 0 else sum(SIZES[0])
        hi = lo + sum(SIZES[rank])
        X, y, pred, proba, target, guess = [ChunkedArray.from_array(a[lo:hi], (tuple(SIZES[rank]),)) for a in arrays]
        parts = train_test_split(X, y, test_size=0.25, random_state=11)
        scores = [accuracy_score(y, pred), log_loss(y, proba), mean_squared_error(target, guess),
                  r2_score(target, guess)]
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), scores=np.array(scores),
                 **{"part%d" % i: p.compute() for i, p in enumerate(parts)},
                 **{"chunks%d" % i: np.array(p.chunks[0]) for i, p in enumerate(parts)})
    finally:
        dist.destroy_process_group()
