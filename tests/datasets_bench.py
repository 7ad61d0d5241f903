"""Speed of the device generators on one GPU (run on an H100: python tests/datasets_bench.py [--out FILE]).

Workloads: make_classification 10M x 64 float32, make_regression 10M x 100 float64, make_counts 10M x 100 float64, in
blocks of 2^21 rows.  Per workload, the CUDA-event time of generating every block from drawn parameters
(``bkm_make_glm_chunk``, one launch per block; make_regression's host draw of ``coef``, a scikit-learn sample of the
first block's size, is timed separately) is alternated in the same process with the torch composition it replaces:
``torch.randn`` of the block, a matmul with the coefficients, then ``torch.bernoulli(sigmoid(z))``, ``+ bias`` or ``torch.poisson(exp(z))``.  Reports
achieved GB/s (the bytes of X and y written) against the 3.35 TB/s floor computed from the shapes, with the card's name
and power limit from the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import sklearn.datasets
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dask_ml_b200 import datasets as D  # noqa: E402
from nb_bench import PEAK_BW, _card, _time  # noqa: E402

BLOCK = 1 << 21


def run(name, n, d, dt, reps):
    ndt = np.float32 if dt == torch.float32 else np.float64
    sizes = D._normalize_chunks(BLOCK, n, d)
    rng = np.random.RandomState(0)
    if name == "make_regression":
        # the host half of make_regression (scikit-learn's first-block-sized sample for coef) is timed on its own
        t0 = time.perf_counter()
        _, _, coef = sklearn.datasets.make_regression(n_samples=sizes[0], n_features=d, coef=True, random_state=rng)
        host_ms = (time.perf_counter() - t0) * 1e3
        nz = np.flatnonzero(coef)
        info = np.column_stack([nz.astype(np.float64), coef[nz]])
        family = D._NORMAL
    else:
        host_ms = 0.0
        family = D._LOGISTIC if name == "make_classification" else D._POISSON
        info = D._informative(rng, d, 2, 1.0)
    key = D._draw_key(rng)
    gen = lambda: D._generate(sizes, d, ndt, family, info, key, "cuda")  # noqa: E731
    y_bytes = 8
    g = torch.Generator(device="cuda").manual_seed(0)
    beta = -torch.rand((d, 1), device="cuda", generator=g, dtype=dt) * (0.1 if name == "make_counts" else 1.0)

    def torched():
        out = []
        for r0 in range(0, n, BLOCK):
            m = min(BLOCK, n - r0)
            X = torch.randn((m, d), device="cuda", generator=g, dtype=dt)
            z = (X @ beta).squeeze(1).double()
            if name == "make_classification":
                y = torch.bernoulli(torch.sigmoid(z), generator=g).long()
            elif name == "make_regression":
                y = z + 0.0
            else:
                y = torch.poisson(torch.exp(z), generator=g).long()
            out.append((X, y))
        return out

    es = 4 if dt == torch.float32 else 8
    byts = n * (d * es + y_bytes)
    tf, tt = [], []
    for _ in range(3):
        tf.append(_time(gen, reps))
        tt.append(_time(torched, reps))
    t_f, t_t = min(tf), min(tt)
    X, y = gen()
    Xh = X.blocks[0][:4096].double().cpu().numpy()
    return dict(workload=name, n=n, d=d, dtype=str(dt).replace("torch.", ""), fused_ms=t_f, torch_ms=t_t,
                gbps=byts / t_f / 1e6, floor_ms=byts / PEAK_BW * 1e3, blocks=len(X.blocks), host_coef_ms=host_ms,
                x_mean=float(Xh.mean()), x_var=float(Xh.var()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--n", type=int, default=10_000_000)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "datasets_bench.py needs a GPU"
    rows = []
    for name, d, dt in (("make_classification", 64, torch.float32), ("make_regression", 100, torch.float64),
                        ("make_counts", 100, torch.float64)):
        r = run(name, a.n, d, dt, a.reps)
        rows.append(r)
        print("%-20s %9d x %3d %-8s fused %8.3f ms  torch %8.3f ms  %6.0f GB/s  floor %6.3f ms  host coef %7.1f ms"
              % (r["workload"], r["n"], r["d"], r["dtype"], r["fused_ms"], r["torch_ms"], r["gbps"], r["floor_ms"],
                 r["host_coef_ms"]),
              flush=True)
        torch.cuda.empty_cache()
    card = _card()
    print("card:", card)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
