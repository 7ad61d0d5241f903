"""KFold and a scorer across two ``gloo`` ranks, each holding its own host blocks: the folds are windows of the global
rows in rank order, so the pieces of the two ranks together are those of one process holding all five blocks; a rank
none of whose rows is in a test window holds one 0-row block there; and a scorer returns the global score on every
rank."""
import os
import socket
import sys

import numpy as np
import pytest
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dist_search_worker as dw  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.timeout(600)
def test_two_ranks_fold_like_one_process_and_score_globally(tmp_path):
    mp.start_processes(dw.worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in (0, 1)]

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.metrics import accuracy_score
    from dask_ml_b200.model_selection import KFold

    X, y = dw.data()
    sizes = tuple(dw.SIZES[0] + dw.SIZES[1])
    one = ChunkedArray.from_array(X, (sizes,))
    nb0 = len(dw.SIZES[0])
    for shuffle in (False, True):
        for f, (tr, te) in enumerate(KFold(dw.K, shuffle=shuffle, random_state=4).split(one)):
            for part, idx in (("train", tr), ("test", te)):
                key = "%d_%d_%s" % (shuffle, f, part)
                np.testing.assert_array_equal(np.concatenate([r[0][key], r[1][key]]), idx.compute())
                both = [c for c in list(r[0][key + "_chunks"]) + list(r[1][key + "_chunks"]) if c]
                assert tuple(both) == idx.chunks[0]

    # n = 163, five windows of 33 / 33 / 33 / 32 / 32 rows: windows 0 and 1 lie on rank 0 (96 rows), 3 and 4 on rank 1
    assert tuple(r[1]["views_0_test_chunks"]) == (0,) and tuple(r[0]["views_4_test_chunks"]) == (0,)
    assert r[1]["views_0_test"].shape == (0, 3) and r[0]["views_1_test"].shape == (33, 3)
    starts = np.cumsum([0, 33, 33, 33, 32, 32])
    for f in range(dw.K):
        np.testing.assert_array_equal(np.concatenate([r[0]["views_%d_test" % f], r[1]["views_%d_test" % f]]),
                                      X[starts[f]:starts[f + 1]])
        rows = slice(starts[f], starts[f + 1])
        want = accuracy_score(y[rows], (X[rows, 0] > 0).astype(np.int64))
        np.testing.assert_allclose(r[0]["scores"][f], want, rtol=1e-15)
    np.testing.assert_array_equal(r[0]["scores"], r[1]["scores"])
