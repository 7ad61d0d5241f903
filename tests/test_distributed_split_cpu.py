"""train_test_split and the scoring metrics across two ``gloo`` ranks, each holding its own host blocks: the block seeds
are drawn for the blocks of all ranks in rank order, so the two ranks together give the split of one process holding all
five blocks, and every rank returns the global scores."""
import os
import socket
import sys

import numpy as np
import pytest
import sklearn.metrics as skm
import torch.multiprocessing as mp

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import dist_split_worker as dw  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.timeout(600)
def test_two_ranks_split_like_one_process_and_score_globally(tmp_path):
    mp.start_processes(dw.worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True, start_method="spawn")
    r = [np.load(tmp_path / ("rank%d.npz" % k)) for k in (0, 1)]

    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.model_selection import train_test_split

    X, y, pred, proba, target, guess = dw.data()
    sizes = dw.SIZES[0] + dw.SIZES[1]
    one = train_test_split(ChunkedArray.from_array(X, (tuple(sizes),)), ChunkedArray.from_array(y, (tuple(sizes),)),
                           test_size=0.25, random_state=11)
    nb0 = len(dw.SIZES[0])
    for i, part in enumerate(one):
        np.testing.assert_array_equal(np.concatenate([r[0]["part%d" % i], r[1]["part%d" % i]]), part.compute())
        assert tuple(r[0]["chunks%d" % i]) == part.chunks[0][:nb0]
        assert tuple(r[1]["chunks%d" % i]) == part.chunks[0][nb0:]
    want = [skm.accuracy_score(y, pred), skm.log_loss(y, proba), skm.mean_squared_error(target, guess),
            skm.r2_score(target, guess)]
    np.testing.assert_allclose(r[0]["scores"], want, rtol=1e-11)
    np.testing.assert_array_equal(r[0]["scores"], r[1]["scores"])
