"""Worker for tests/test_gpu_spectral.py::test_multi_gpu_embedding_equals_single_gpu (launched by torch.distributed.run,
one rank per GPU, NCCL): SpectralClustering on uneven row shards, the full embedding and eigenvalues saved per rank."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch
from sklearn.base import BaseEstimator


class Rec(BaseEstimator):
    def __init__(self, n_clusters=2):
        self.n_clusters = n_clusters

    def fit(self, X, y=None):
        self.X_ = np.asarray(X)
        self.labels_ = np.zeros(len(self.X_), dtype=np.int32)
        return self


def data():
    rng = np.random.RandomState(12)
    cent = rng.uniform(-3, 3, size=(6, 16))
    return (cent[rng.randint(0, 6, size=40000)] + 0.5 * rng.standard_normal((40000, 16))).astype(np.float32)


def fit(X):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import SpectralClustering

    rec = Rec()
    sc = SpectralClustering(n_clusters=6, n_components=120, gamma=0.1, random_state=4, assign_labels=rec)
    sc.fit(ChunkedArray.from_array(X, 7000))
    return rec.X_, sc.eigenvalues_


def single_gpu():
    return fit(data())


def main(out_dir):
    import torch.distributed as dist

    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    try:
        X = data()
        bounds = (np.linspace(0, 1, world + 1) ** 1.3 * len(X)).astype(int)      # uneven shards
        U, S = fit(X[bounds[rank]:bounds[rank + 1]])
        np.savez(os.path.join(out_dir, "rank%d.npz" % rank), U=U, S=S)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main(sys.argv[1])
