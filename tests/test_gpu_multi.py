"""N-GPU result == 1-GPU result == oracle.  Needs >= 2 GPUs; run with -m gpu."""
import os
import subprocess
import sys

import numpy as np
import pytest

from _util import assert_labels_match

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_multi_gpu_equals_single_gpu_and_oracle(tmp_path, oracle):
    import torch

    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip("needs at least 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
           "--master-addr", "127.0.0.1", "--master-port", "29577",
           os.path.join(ROOT, "tests", "dist_gpu_worker.py"), str(tmp_path)]
    subprocess.run(cmd, check=True, timeout=600, cwd=ROOT)

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.cluster import KMeans

    rng = np.random.RandomState(11)
    n, d, k = 64000, 64, 256
    cent = rng.uniform(-10, 10, size=(90, d))
    X = (cent[rng.randint(0, 90, size=n)] + rng.standard_normal((n, d))).astype(np.float32)
    init = X[:k].copy()
    one = KMeans(k, init=init, max_iter=6, tol=1e-4).fit(ChunkedArray.from_array(X, 9000))
    lab, inertia, C, n_iter = oracle.kmeans_single_lloyd(oracle.to_blocks(X, 9000), k, init=init, max_iter=6, tol=1e-4)
    labels = np.empty(n, dtype=np.int32)
    for r in range(world):
        g = np.load(tmp_path / ("rank%d.npz" % r))
        assert int(g["n_iter"]) == one.n_iter_ == n_iter
        np.testing.assert_allclose(g["centers"], one.cluster_centers_, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(g["centers"], C, rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(float(g["inertia"]), inertia, rtol=1e-6)
        labels[int(g["lo"]):int(g["hi"])] = g["labels"]
        # one node: the per-iteration collective ran over NVLink peer memory and is bit-exact in rank order
        assert bool(g["p2p_ready"]) or os.environ.get("BKM_P2P") == "0"
        assert int(g["p2p_bad"]) == 0
        if r:
            np.testing.assert_array_equal(g["centers_b"], np.load(tmp_path / "rank0.npz")["centers_b"])
    assert_labels_match(labels, np.concatenate(lab), X, C, rtol=1e-6)
    assert_labels_match(labels, one.labels_.compute(), X, C, rtol=1e-6)
