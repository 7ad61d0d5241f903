"""Timing of TruncatedSVD on sparse CSR blocks on one H100 (not part of the suite).

The two workloads of tests/glm_sparse_bench.py, one CSR block each, float32 values:
  hashed   4M rows x 2^20 features, ~55 Zipf-distributed entries per row: k = 100, algorithm='randomized', n_iter=5
  onehot   10M rows x 1024 features (8 columns x 128 categories): k = 16, the exact regime

Per block it times, with CUDA events after a warm-up (median over --reps, alternated in the same process), the two panel
products at l = 110 (the subspace of k = 100) against a float64 torch composition of the same result:
bkm_csr_panel_chunk (X W) against torch.sparse.mm, and bkm_csc_panel_chunk (X^T P) against torch.sparse.mm on the
transpose from torch's CSC conversion (made outside the timing).  Outputs are compared at the timed sizes.  Each time is
set against its HBM floor: the CSR (or CSC) read once plus the panel written once, over 3.35 TB/s; the bytes of the
gathered panel rows (nnz l 8) are printed beside it.  Then the whole TruncatedSVD.fit per workload.  The card's name,
power limit and clock are read in the same run.

    python tests/svd_sparse_bench.py [--reps 10] [--small] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from glm_sparse_bench import HBM, card, hashed, onehot, timed  # noqa: E402

L = 110


def _rel(a, b):
    return float(torch.linalg.norm(a.double() - b.double()) / max(float(torch.linalg.norm(b.double())), 1e-300))


def bench_block(name, crow, col, val, n, d, k, algorithm, reps, fit_reps):
    from dask_ml_b200 import ChunkedArray
    from dask_ml_b200.decomposition import TruncatedSVD
    from dask_ml_b200.engine import CudaBackend

    be = CudaBackend()
    nnz = int(col.numel())
    es = val.element_size()
    blk = (crow, col, val, n)
    res = {"workload": name, "n": n, "d": d, "nnz": nnz, "l": L, "k": k, "algorithm": algorithm}
    csc = be.csr_transpose_chunk(blk, d)
    gen = torch.Generator(device="cuda").manual_seed(2)
    W = torch.randn((d, L), generator=gen, device="cuda", dtype=torch.float64)
    P = torch.randn((n, L), generator=gen, device="cuda", dtype=torch.float64)
    out = torch.empty((n, L), dtype=torch.float64, device="cuda")
    Z = torch.empty((d, L), dtype=torch.float64, device="cuda")
    X64 = torch.sparse_csr_tensor(crow, col, val.double(), size=(n, d))
    XT64 = X64.to_sparse_csc().t()                               # the CSR of X^T, built outside the timing
    box = {}

    def ours_row():
        be.csr_panel_chunk(blk, d, W, out=out)

    def torch_row():
        box["row"] = torch.sparse.mm(X64, W)

    def ours_col():
        be.csc_panel_chunk(csc, d, P, Z, first=True)

    def torch_col():
        box["col"] = torch.sparse.mm(XT64, P)

    t = timed([ours_row, torch_row], reps)
    res["row_panel_ms"], res["row_torch_ms"] = t
    res["row_rel_diff"] = _rel(out, box["row"])
    row_floor = (8 * (n + 1) + (8 + es) * nnz + 8 * n * L) / HBM * 1e3
    res["row_floor_ms"], res["row_gather_GB"] = row_floor, nnz * L * 8 / 1e9
    t = timed([ours_col, torch_col], reps)
    res["col_panel_ms"], res["col_torch_ms"] = t
    res["col_rel_diff"] = _rel(Z, box["col"])
    col_floor = (8 * (d + 1) + (4 + es) * nnz + 8 * d * L) / HBM * 1e3
    res["col_floor_ms"], res["col_gather_GB"] = col_floor, nnz * L * 8 / 1e9
    del X64, XT64, box, W, P, out, Z
    torch.cuda.empty_cache()

    X = ChunkedArray([torch.sparse_csr_tensor(crow, col, val, size=(n, d))])

    def fit():
        TruncatedSVD(n_components=k, algorithm=algorithm, n_iter=5, random_state=0).fit(X)

    res["fit_ms"] = timed([fit], fit_reps)[0]
    s = TruncatedSVD(n_components=k, algorithm=algorithm, n_iter=5, random_state=0).fit(X)
    res["singular_values_head"] = [float(v) for v in s.singular_values_[:3]]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--fit-reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--small", action="store_true", help="tiny sizes (a check of the script, not a measurement)")
    a = ap.parse_args()
    results = {"card": card()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    n1, n2 = (4_000_000, 10_000_000) if not a.small else (40_000, 100_000)
    crow, col, val = hashed(n1, 1 << 20, 60, gen)
    results["hashed"] = bench_block("hashed", crow, col, val, n1, 1 << 20, 100, "randomized", a.reps, a.fit_reps)
    del crow, col, val
    torch.cuda.empty_cache()
    crow, col, val = onehot(n2, 8, 128, gen)
    results["onehot"] = bench_block("onehot", crow, col, val, n2, 1024, 16, "tsqr", a.reps, a.fit_reps)
    results["card_after"] = card()
    print(json.dumps(results, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
